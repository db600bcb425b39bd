"""Attention-probability dropout without a GPU: the restatement of the kernels' mask (tests/attn_dropout_oracle.py
`attention_keep`) against a per-element coding of its definition, its statistics, and the hook and transformer wrapper
through which the oracle drops the softmax probabilities (utils/transformer.py:114-115)."""
import math

import numpy as np
import pytest
import torch

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O
from tests import attn_dropout_oracle as AD

M32 = 0xFFFFFFFF


def _philox7(ctr, key):
    """Philox4x32-7 on Python integers, written independently of DM.philox4x32."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(7):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & M32, p1 & M32, ((p0 >> 32) ^ c3 ^ k1) & M32, p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
    return c0, c1, c2, c3


def _keep_loop(seed, site, B, heads, S, p):
    """The definition, one element at a time."""
    n16 = (S + 15) // 16
    th = DM.thresh16(p)
    out = np.zeros((B, heads, S, S), dtype=bool)
    for b in range(B):
        for h in range(heads):
            for q in range(S):
                for k in range(S):
                    blk = ((((b * heads + h) * n16 + q // 16) * 8 + q % 8) * n16 + k // 16) * 8 + k % 8
                    w = _philox7((blk & M32, blk >> 32, site, 0x4154544E), (seed & M32, seed >> 32))
                    out[b, h, q, k] = (w[2 * ((q >> 3) & 1) + ((k >> 3) & 1)] >> 16) >= th
    return out


@pytest.mark.parametrize("S", [1, 9, 17, 40])
def test_attention_keep_matches_the_definition(S):
    seed, site = 2 ** 33 + 17, 205
    got = AD.attention_keep(seed, site, 2, 3, S, 0.3)
    assert got.shape == (2, 3, S, S) and got.dtype == bool
    assert np.array_equal(got, _keep_loop(seed, site, 2, 3, S, 0.3))


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_attention_keep_rate(p):
    keep = AD.attention_keep(2 ** 40 + 3, 7, 2, 3, 300, p)
    q = 1.0 - DM.thresh16(p) / 65536.0
    assert abs(keep.mean() - q) < 5.0 * math.sqrt(q * (1.0 - q) / keep.size)


def _uncorrelated(a, b):
    a, b = a.ravel().astype(np.float64), b.ravel().astype(np.float64)
    assert not np.array_equal(a, b)
    assert abs(np.corrcoef(a, b)[0, 1]) < 5.0 / math.sqrt(a.size)


def test_attention_keep_streams_differ():
    """Heads, batch elements, sites and seeds s / s + 2^32 draw unrelated masks; so does hidden dropout (counter word "MERL"
    instead of "ATTN") at the same seed and site."""
    s, site, S, p = 11, 3, 96, 0.5
    k = AD.attention_keep(s, site, 2, 2, S, p)
    _uncorrelated(k[:, 0], k[:, 1])
    _uncorrelated(k[0], k[1])
    _uncorrelated(k, AD.attention_keep(s, site + 1, 2, 2, S, p))
    _uncorrelated(k, AD.attention_keep(s + 2 ** 32, site, 2, 2, S, p))
    # hidden dropout's mask of the same number of elements, at the same seed and site
    _uncorrelated(k, DM.counter_dropout_keep(s, site, 2 * 2 * S, S, p))


def test_attention_dropout_kernel_sites():  # merlot_stack_forward: base + l for the probabilities of layer l
    assert [AD.kernel_site(k) for k in (("vit", 0, "probs"), ("vit", 3, "probs"), ("langonly", 1, "probs"),
                                        ("joint", 11, "probs"))] == [0, 3, 101, 211]


def test_attention_dropout_hook_scale_identity_and_gradient():
    seed = 2 ** 32 + 5
    x = torch.rand(2, 3, 20, 20, generator=torch.Generator().manual_seed(0), requires_grad=True)
    assert AD.dropout_hook(seed, 0.1, 0.2)(("joint", 1, "probs"), x) is x  # p_attn defaults to 0
    assert AD.dropout_hook(seed, 0.1, 0.2, 0.0)(("vit", 0, "probs"), x) is x
    hook = AD.dropout_hook(seed, 0.0, 0.0, 0.25)
    y = hook(("langonly", 1, "probs"), x)
    factor = torch.from_numpy(AD.attention_keep(seed, 101, 2, 3, 20, 0.25)).float() * float(DM.dropout_scale(0.25))
    assert torch.equal(y, x * factor)
    y.sum().backward()
    assert torch.equal(x.grad, factor)
    h = torch.randn(40, 128)
    assert hook(("joint", 0, "ffn"), h) is h  # hidden sites keep their own probability (0 here)


def _tiny_oracle_case(cfg):
    g = torch.Generator().manual_seed(0)
    image = torch.rand(4, 64, 96, 3, generator=g)
    ids = torch.randint(100, 1000, (2, 2, 16), generator=g, dtype=torch.int32)
    ids[:, :, 0] = O.START
    ids[:, :, 12:] = 0
    params = O.init_params(cfg, 1, perturb=0.05)
    shuf = torch.tensor([0, 1, 17, 16], dtype=torch.int32)
    draws = O.make_mask_draws(2, 32, 6, 1000, seed=2)
    return image, ids, params, dict(mask_input=True, shuffled_idx_img=shuf, mask_draws=draws)


def test_transformer_wrapper_without_attention_dropout_is_the_oracle(tiny_cfg, monkeypatch):
    """The wrapper with p_attn = 0 (the hook hands the probabilities back untouched) and with no hook at all: every output of a
    training-mode oracle step bit for bit the oracle's own."""
    image, ids, params, kw = _tiny_oracle_case(tiny_cfg)

    def outputs(hook):
        m = O.MerlotOracle(tiny_cfg, params, image, ids, dropout=hook, **kw)
        return [m.attention_summs, m.encoder_info["self_attn_probs"], m.encoder_hidden_states["viz"], m.encoder_hidden_states["lang"],
                m.lang_transformer_info["hidden_state"], m.vision_transformer_info["hidden_state"]]
    ref = [outputs(DM.dropout_hook(3, 0.1, 0.2)), outputs(None)]
    monkeypatch.setattr(O, "transformer", AD.transformer)
    got = [outputs(AD.dropout_hook(3, 0.1, 0.2, 0.0)), outputs(None)]
    for r, g in zip(ref, got):
        for a, b in zip(r, g):
            assert torch.equal(a, b)


def test_attention_dropout_hook_call_sites_and_self_attn_probs(tiny_cfg, monkeypatch):
    """With the wrapper installed the hook is called once per layer of each stack on the softmax probabilities
    [B, heads, S, S] (key (stack, layer, "probs")), before the hidden-dropout calls of that layer; self_attn_probs -- and with
    them the attention sums that drive masking -- are the head means of what it returns."""
    cfg = dict(tiny_cfg, attention_probs_dropout_prob=0.1)
    image, ids, params, kw = _tiny_oracle_case(cfg)
    train = AD.dropout_hook(2 ** 32 + 1, 0.1, 0.2, 0.1)
    calls, outs = [], {}

    def spy(key, x):
        calls.append((key, tuple(x.shape)))
        y = train(key, x)
        if key[-1] == "probs":
            outs[key] = y.detach()
        return y
    monkeypatch.setattr(O, "transformer", AD.transformer)
    m = O.MerlotOracle(cfg, params, image, ids, dropout=spy, **kw)
    monkeypatch.undo()
    heads = cfg["num_attention_heads"]
    probs_calls = [c for c in calls if c[0][-1] == "probs"]
    n_vit, n_lo, n_j = (cfg["num_vision_transformer_hidden_layers"], cfg["num_lang_transformer_hidden_layers"],
                        cfg["num_hidden_layers"])
    S_vit, S_lo, S_j = (64 // 16) * (96 // 16) + 2, 32, m.P + m.L
    want = ([(("vit", l, "probs"), (4, heads, S_vit, S_vit)) for l in range(n_vit)]
            + [(("langonly", l, "probs"), (2, heads, S_lo, S_lo)) for l in range(n_lo)]
            + [(("joint", l, "probs"), (m.B, heads, S_j, S_j)) for l in range(n_j)])
    assert probs_calls == want
    for stack in ("vit", "langonly", "joint"):  # each layer: probabilities first, then the two hidden-dropout sites
        keys = [c[0] for c in calls if c[0][0] == stack]
        assert keys[:3] == [(stack, 0, "probs"), (stack, 0, "attn"), (stack, 0, "ffn")]
    lo = m.lang_transformer_info["self_attn_probs"]
    j = m.encoder_info["self_attn_probs"]
    for l in range(n_lo):
        assert torch.equal(lo[:, l], outs[("langonly", l, "probs")].mean(1))
    for l in range(n_j):
        assert torch.equal(j[:, l], outs[("joint", l, "probs")].mean(1))
    assert torch.equal(m.attention_summs, lo.sum((1, 2)))  # model/modeling.py:428
    assert float((j.sum(-1) - 1).abs().max()) > 1e-2  # dropped rows no longer sum to one
    assert O.transformer is AD._oracle_transformer and O.attention_core is AD._oracle_attention_core  # nothing left patched
