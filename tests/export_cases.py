"""TEST INFRASTRUCTURE ONLY.  Seeded inputs of the attention-probability export (merlot_attention_probs) and their float64
head-mean probabilities, restated from utils/transformer.py:98-120 as the kernel reads them: a padding query row has every
score 0 (a uniform row), a masked key scores -1e10, and with attention dropout the kept probabilities are scaled by 1/(1-p).

Every input is drawn on the CPU from a seeded generator, so one case is the same bits on every machine; `lse` is the
float64 log-sum-exp rounded to fp32, so the cases do not depend on the forward kernel."""
import hashlib

import torch

from tests import attn_dropout_oracle as AD

SEED = 2 ** 32 + 777  # non-zero high word of the Philox key
SITE = 11


def case(B, S, heads, seed, ragged=True, pair=(0, 0)):
    """(qkv bf16 [B*S, 3H], lse fp32 [B, heads, S], valid bool [B, S] or None) of one layer."""
    g = torch.Generator().manual_seed(seed)
    H = heads * 64
    qkv = torch.randn(B * S, 3 * H, generator=g).bfloat16()
    valid = None
    if ragged:
        lens = torch.randint(1, S + 1, (B,), generator=g)
        valid = torch.arange(S)[None] < lens[:, None]
        if S > 4:
            valid[-1, S // 3] = False  # a hole inside the last sequence
    s = scores(qkv, B, S, heads, valid, pair)
    return qkv, torch.logsumexp(s, -1).float(), valid


def scores(qkv, B, S, heads, valid, pair=(0, 0)):
    """float64 [B, heads, S, S] masked scores as the export kernel forms them."""
    x = qkv.double().reshape(B, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = torch.einsum("bhqd,bhkd->bhqk", x[0], x[1]) * 0.125
    vq = torch.ones(B, S, dtype=torch.bool) if valid is None else valid
    P, chunk = pair
    seg = torch.zeros(S, dtype=torch.int64)
    if chunk > 0:
        seg[P:] = 1 + (torch.arange(S - P) // chunk)
    ok = (seg[:, None] == seg[None]) | (seg == 0)[None] | (seg == 0)[:, None]
    keys = vq[:, None, None, :] & ok[None, None]
    s = torch.where(keys, s, torch.full_like(s, -1e10))
    return torch.where(vq[:, None, :, None], s, torch.zeros_like(s))


def head_mean(qkv, lse, B, S, heads, valid, pair=(0, 0), dropout=(0.0, 0, 0)):
    """float64 [B, S, S]: mean over heads of exp(score - lse), dropped as the kernels drop it when dropout[0] > 0."""
    pr = torch.exp(scores(qkv, B, S, heads, valid, pair) - lse.double()[..., None])
    p, seed, site = dropout
    if p > 0:
        pr = pr * torch.from_numpy(AD.attention_keep(seed, site, B, heads, S, p)).double() / (1.0 - p)
    return pr.mean(1)


def digest(t: torch.Tensor) -> str:
    """SHA-256 of a tensor's bytes (bit-identity checks against recorded outputs)."""
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


# (B, S, heads, ragged, pair): S across the 8-query CTA rows and the 256-key thread stride, ragged and full masks, one pair mask
SHAPES = [(2, 1, 1, False, (0, 0)), (2, 7, 2, True, (0, 0)), (1, 8, 2, True, (0, 0)), (2, 9, 2, True, (0, 0)),
          (2, 255, 2, True, (0, 0)), (1, 256, 3, False, (0, 0)), (2, 257, 2, True, (0, 0)), (2, 300, 2, True, (100, 40))]
