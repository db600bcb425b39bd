"""TEST INFRASTRUCTURE ONLY.  A float64 reference of one transformer stack as merlot_stack_forward / merlot_stack_backward
(merlot_b200/csrc/stack.cu) compute it, built from the oracle's primitives: O.layer_norm and O.gelu, the hidden-dropout mask
of oracle/dropout_mask.py, and tests/attn_dropout_oracle.py's attention_core (O.attention_core with its probabilities passed
through drop_probs, the attention-probability mask).

It takes the very bf16 weights and input the kernels read, the fused w_qkv [H, 3H] layout included, and rounds to bf16
exactly where stack.cu stores bf16 (x1, qkv, ctx, hmid, x2, act, hout and y), with a straight-through rounding so that
autograd differentiates the float64 arithmetic.  A comparison against it is then about the kernels' arithmetic, not about
the precision the stack stores activations in.

Per layer l (sites as in stack.cu): x1 = LN1(h); qkv = x1 Wqkv + b; ctx = attn(qkv) with the probabilities dropped at site
base + l; hmid = h + drop(ctx Wo + bo) at site base + 2l; x2 = LN2(hmid); act = gelu(x2 W1 + b1);
hout = hmid + drop(act W2 + b2) at site base + 2l + 1; and y = LN_final(h_last).

`wrong` selects a reference that is wrong in one way, for the tests that show their bars are tight enough:
  "sites_swapped"  the out-projection and FFN2 hidden-dropout sites exchanged;
  "attn_next_site" every layer's attention mask drawn at the next layer's site;
  "ln2_stats"      the middle layer's LN2 backward evaluated at LN1's statistics (the forward is unchanged).
"""
from __future__ import annotations

import torch

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O
from tests import attn_dropout_oracle as ADO

LAYER_PARAMS = ("ln1_gamma", "ln1_beta", "w_qkv", "b_qkv", "w_o", "b_o", "ln2_gamma", "ln2_beta", "w_1", "b_1", "w_2", "b_2")
WRONG = ("sites_swapped", "attn_next_site", "ln2_stats")


def _bf16(t: torch.Tensor) -> torch.Tensor:
    """bf16 rounding in the forward, identity in the backward."""
    return t + (t.to(torch.bfloat16).to(t.dtype) - t).detach()


def _ln(x, gamma, beta):
    return O.layer_norm(x, {"ln/gamma": gamma, "ln/beta": beta}, "ln")


def _stats(x):
    mean = x.mean(-1, keepdim=True)
    return mean, torch.rsqrt(((x - mean) ** 2).mean(-1, keepdim=True) + 1e-5)


class _LayerNormGradAt(torch.autograd.Function):
    """Value y (a LayerNorm output computed elsewhere); backward: the LayerNorm gradient formula of the kernels evaluated at
    the given statistics instead of those of x."""

    @staticmethod
    def forward(ctx, x, gamma, beta, y, mean, rstd):
        ctx.save_for_backward(x, gamma, mean, rstd)
        return y.clone()

    @staticmethod
    def backward(ctx, dy):
        x, gamma, mean, rstd = ctx.saved_tensors
        xh = (x - mean) * rstd
        gd = gamma * dy
        dx = rstd * (gd - gd.mean(-1, keepdim=True) - xh * (gd * xh).mean(-1, keepdim=True))
        return dx, (dy * xh).sum(0), dy.sum(0), None, None, None


def attention_mask(B: int, S: int, valid, pair=(0, 0), device="cpu"):
    """[B, S, S] float64 mask of merlot_attn_t: valid[q] & valid[k], and with pair_chunk_len > 0 only pairs that share a
    segment or have a vision token (t < pair_viz_len) on either side; None when every pair is valid."""
    if valid is None:
        return None
    v = valid.reshape(B, S).to(device=device, dtype=torch.bool)
    m = v[:, :, None] & v[:, None, :]
    P, chunk = pair
    if chunk > 0:
        t = torch.arange(S, device=device)
        seg = torch.where(t < P, torch.zeros_like(t), 1 + (t - P) // chunk)
        m &= (seg[:, None] == seg[None, :]) | (seg[:, None] == 0) | (seg[None, :] == 0)
    return m.double()


def hidden_keep(seed: int, site: int, rows: int, N: int, p: float, device) -> torch.Tensor:
    """float64 keep * scale of the hidden-dropout mask of a [rows, N] tensor at (seed, site)."""
    keep = torch.from_numpy(DM.counter_dropout_keep(seed, site, rows, N, p)).to(device)
    return keep.double() * float(DM.dropout_scale(p))


def stack_reference(layers, final_gamma, final_beta, h_in, dy, *, B, S, heads, valid=None, pair=(0, 0), hidden_p=0.0,
                    attn_p=0.0, seed=0, site_base=0, colsum_split=0, colsum_valid_q=False, wrong=None, device="cpu"):
    """layers: one dict per layer of the LAYER_PARAMS tensors (bf16 weights, fp32 vectors); h_in, dy: bf16 [B*S, H].
    Returns float64 tensors on `device`: y, colsum [B, S] and colsum2 (the queries >= colsum_split, when > 0), probs
    [layers, B, S, S] (head-mean, after dropout), dh_in, grads (one dict of g_<name> per layer) and d_final_gamma / _beta."""
    assert wrong is None or wrong in WRONG, wrong
    dd = dict(device=device, dtype=torch.float64)
    L = len(layers)
    M, H = h_in.shape
    P = [{k: v.to(**dd).requires_grad_(True) for k, v in lp.items()} for lp in layers]
    fg, fb = final_gamma.to(**dd).requires_grad_(True), final_beta.to(**dd).requires_grad_(True)
    h0 = h_in.to(**dd).requires_grad_(True)
    mask = attention_mask(B, S, valid, pair, device)
    qmask = torch.ones(B, S, **dd) if (valid is None or not colsum_valid_q) else valid.reshape(B, S).to(**dd)
    lo_q = (torch.arange(S, device=device) < colsum_split).double() if colsum_split > 0 else torch.ones(S, **dd)
    colsum, colsum2, probs_all = torch.zeros(B, S, **dd), torch.zeros(B, S, **dd), []
    s_attn, s_ffn = (1, 0) if wrong == "sites_swapped" else (0, 1)
    h = h0
    for l, p in enumerate(P):
        x1 = _bf16(_ln(h, p["ln1_gamma"], p["ln1_beta"]))
        qkv = _bf16(x1 @ p["w_qkv"] + p["b_qkv"])
        q, k, v = (qkv[:, i * H:(i + 1) * H].reshape(B, S, heads, 64).permute(0, 2, 1, 3) for i in range(3))
        asite = site_base + l + (1 if wrong == "attn_next_site" else 0)
        pr, c4 = ADO.attention_core(q, k, v, mask, lambda t: ADO.drop_probs(t, seed, asite, attn_p))
        with torch.no_grad():
            pm = pr.mean(1)  # [B, S(q), S(k)]
            probs_all.append(pm)
            w = (qmask * lo_q)[:, :, None]
            colsum += (pm * w).sum(1)
            colsum2 += (pm * (qmask * (1 - lo_q))[:, :, None]).sum(1)
        ctx = _bf16(c4.permute(0, 2, 1, 3).reshape(M, H))
        a = ctx @ p["w_o"] + p["b_o"]
        if hidden_p > 0:
            a = a * hidden_keep(seed, site_base + 2 * l + s_attn, M, H, hidden_p, device)
        hmid = _bf16(h + a)
        x2 = _ln(hmid, p["ln2_gamma"], p["ln2_beta"])
        if wrong == "ln2_stats" and l == min(1, L - 1):
            x2 = _LayerNormGradAt.apply(hmid, p["ln2_gamma"], p["ln2_beta"], x2.detach(), *(t.detach() for t in _stats(h)))
        act = _bf16(O.gelu(_bf16(x2) @ p["w_1"] + p["b_1"]))
        f = act @ p["w_2"] + p["b_2"]
        if hidden_p > 0:
            f = f * hidden_keep(seed, site_base + 2 * l + s_ffn, M, H, hidden_p, device)
        h = _bf16(hmid + f)
    y = _bf16(_ln(h, fg, fb))
    leaves = [h0, fg, fb] + [p[n] for p in P for n in LAYER_PARAMS]
    g = torch.autograd.grad(y, leaves, dy.to(**dd))
    grads = [{"g_" + n: g[3 + l * len(LAYER_PARAMS) + i] for i, n in enumerate(LAYER_PARAMS)} for l in range(L)]
    return dict(y=y.detach(), colsum=colsum, colsum2=colsum2 if colsum_split > 0 else None, probs=torch.stack(probs_all),
                dh_in=g[0], grads=grads, d_final_gamma=g[1], d_final_beta=g[2])
