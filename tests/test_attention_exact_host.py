"""The attention checks of tests/attention_exact_oracle.py on the CPU: the constructions' claims hold in float64 and in a float32
replay of the kernels' log2-domain arithmetic, a float32 emulation of the kernels' rounding points meets every per-element
bound, and doctored outputs (a dropped or admitted key, a row from the neighbouring head, a missing query chunk or dQ slice, an
LSE entry off by log(1 + 1/S), a padding query in the column sums) each fail the check aimed at them, where the
relative-Frobenius bars of test_gpu_kernels.py (1e-2 ctx, 1.5e-2 dq/dk/dv, 2e-3 column sums) accept several of them."""
import math

import numpy as np
import pytest
import torch

from tests import attention_exact_oracle as X

CTX_BAR, DQKV_BAR, COLSUM_BAR = 1e-2, 1.5e-2, 2e-3


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def loc(idx):
    return str(idx)


ROUTED = [(1, 1, 1, "none"), (2, 63, 2, "none"), (3, 129, 2, "ragged"), (2, 200, 3, "pair"), (2, 65, 1, "len1"),
          (2, 130, 2, "empty"), (1, 257, 1, "ragged")]


@pytest.mark.parametrize("B,S,heads,kind", ROUTED)
def test_routed_construction_claims(B, S, heads, kind):
    v = X.validity(kind, B, S)
    pair = X.pair_for(S) if kind == "pair" else (0, 0)
    c = X.routed(B, S, heads, v, pair, seed=S)
    qkv, tg = c["qkv"], c["targets"]
    nb = c["nb"]
    assert X.max_partial_units(qkv, B, S, heads) < 2 ** 16 / A_GRANULE
    x = qkv.double().reshape(B, S, 3, heads, 64)
    vm = X.valid_or_ones(v, B, S)
    m = X.score_mask(v, B, S, pair)
    sc2 = np.float32(X.SC2)
    for b in range(B):
        # keys of the next sequence, as the kernels' last tiles read them: every one of them is poisoned
        nxt = x[b + 1] if b + 1 < B else None
        for h in range(heads):
            q, k = x[b, :, 0, h], x[b, :, 1, h]
            s = q @ k.t() * X.SCALE  # exact: integers times 64
            t32 = ((q @ k.t()).float() * torch.tensor(sc2)).double()  # the kernels' log2-domain scores, float32
            for i in range(S):
                if not vm[b, i]:
                    assert tg[b, h, i, 0] == -1
                    continue
                a, a2 = int(tg[b, h, i, 0]), int(tg[b, h, i, 1])
                assert a >= 0 and m[b, i, a]
                top = [a] if a2 < 0 else [a, a2]
                if a2 >= 0:
                    assert bin(a ^ a2).count("1") == 1 and m[b, i, a2]
                assert all(float(s[i, j]) == 0.0 and float(t32[i, j]) == 0.0 for j in top)
                others = m[b, i].clone()
                others[top] = False
                if others.any():
                    gap = 2 * X.A * X.SCALE * (1 if a2 < 0 else 2)
                    assert float(s[i, others].max()) <= -gap
                    assert float(t32[i, others].max()) < -150.0  # ex2 underflows (flushed below 2^-126)
                forbidden = ~m[b, i]
                if forbidden.any():  # a leaked key beats the target
                    assert float(s[i, forbidden].min()) >= 2 * X.A * X.SCALE
                if nxt is not None:
                    assert float((q[i] @ nxt[:, 1, h].t()).min() * X.SCALE) >= 2 * X.A * X.SCALE
    # every expected output is exact in float32, its bf16 rounding the kernels' result
    ref = X.reference(qkv, c["d_ctx"], B, S, heads, v, pair, weights=lambda b, h: X.routed_weights(tg, v, b, h, S))
    vr = vm.reshape(-1)
    assert torch.equal(ref["ctx"][vr], ref["ctx_emul"][vr].double())  # (V_a + V_b) / 2: bf16-exact
    for name in ("D", "dqkv", "bias"):
        assert torch.equal(ref[name].float().double(), ref[name]), name
    lse = ref["lse"].float()
    vb = vm[:, None, :].expand(B, heads, S)
    two = tg[..., 1] >= 0
    assert torch.equal(lse[vb & ~two], torch.zeros(int((vb & ~two).sum())))
    assert bool((lse[vb & two] == X.LN2_F32).all())
    dq = ref["dqkv"].reshape(B, S, 3, heads, 64)[:, :, 0]
    one_hot = (vm[:, :, None] & ~two.permute(0, 2, 1))
    assert float(dq[one_hot].abs().sum()) == 0.0  # one-hot rows: dS = 0 exactly
    if bool((vb & two).any()):
        assert float(dq.abs().max()) > 0  # two-hot rows: non-zero dQ
    for key, val in ref["cs"].items():  # valid queries only: per head, a sum of probabilities 1 and 1/2
        if key[0]:
            assert torch.allclose(val * heads * 2, (val * heads * 2).round(), rtol=0, atol=1e-9)


A_GRANULE = 1  # max_partial_units counts in units of A (the q granule) x 1 (the k granule)


def test_counting_construction_recovers_the_admitted_sets():
    B, S, heads = 2, 300, 1
    v = X.validity("pair", B, S)
    pair = X.pair_for(S)
    v[1, 40:] = False
    v[1, 5] = True
    c = X.counting(B, S, heads)
    adm = X.admitted(v, B, S, pair)
    ref = X.reference(c["qkv"], c["d_ctx"], B, S, heads, v, pair, weights=lambda b, h: adm[b].double())
    V = c["qkv"].double().reshape(B, S, 3, heads, 64)[0, :, 2, 0]
    for b in range(B):
        for i in (0, 1, 31, 32, 119, 120, 153, 154, 299):
            n = int(adm[b, i].sum())
            want = adm[b, i].double() @ V
            assert int(want.max()) <= 124
            got = X.decode_counts(ref["ctx_emul"][b * S + i, :64].float(), n)
            assert torch.equal(got, want.long()), (b, i)


def test_emulation_meets_every_bound():
    """The float32 emulation of the kernels' rounding points, on random, masked, pair-masked and peaked data."""
    worst = {}
    for B, S, heads, kind, peaked in [(2, 129, 2, "ragged", False), (1, 200, 2, "pair", False), (2, 70, 1, "empty", True),
                                      (1, 300, 1, "none", True)]:
        v = X.validity(kind, B, S)
        pair = X.pair_for(S) if kind == "pair" else (0, 0)
        qkv, d_ctx = X.random_case(B, S, heads, seed=S, peaked=peaked)
        ref = X.reference(qkv, d_ctx, B, S, heads, v, pair, bounds=True)
        em = X.emulate_fp32(qkv, d_ctx, B, S, heads, v, pair)
        for name, out_bf16 in (("ctx", True), ("lse", False), ("D", False), ("dqkv", True)):
            r = X.bound_check(em[name], ref[name], ref["bar_" + name], name, loc, out_bf16=out_bf16)
            worst[name] = max(worst.get(name, 0.0), r)
        r = X.bound_check(em["cs"], ref["cs"][(False, 0)] + ref["cs"][(False, 1)],
                          ref["bar_cs"][(False, 0)] + ref["bar_cs"][(False, 1)], "colsum", loc, out_bf16=False)
        worst["colsum"] = max(worst.get("colsum", 0.0), r)
    # the bf16 terms dominate: the emulation uses a good part of the bound, never all of it
    assert all(0.05 < w <= 1.0 for k, w in worst.items() if k not in ("lse", "D", "colsum")), worst


# ---------------------------------------------------------------------------------------------------------------------
# doctored outputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rand_case():
    """Random data, B = 2, S = 700 (more than 4 key tiles), 2 heads, ragged lengths: the reference and its bounds."""
    B, S, heads = 2, 700, 2
    v = X.validity("ragged", B, S)
    qkv, d_ctx = X.random_case(B, S, heads, seed=7)
    ref = X.reference(qkv, d_ctx, B, S, heads, v, bounds=True)
    return B, S, heads, v, qkv, d_ctx, ref


def test_dropped_last_key_is_caught(rand_case):
    """Key S - 1 dropped for 8 queries: exact mismatch on the counting construction, past the bound on random data, and within
    the ctx Frobenius bar."""
    B, S, heads, v, qkv, d_ctx, ref = rand_case
    v0 = torch.ones(1, S, dtype=torch.bool)
    adm = X.admitted(v0, 1, S)
    rows = [3, 64, 65, 127, 128, 300, 511, 699]
    bad = adm.clone()
    bad[0, rows, S - 1] = False
    c = X.counting(1, S, heads)
    want = X.reference(c["qkv"], c["d_ctx"], 1, S, heads, None, weights=lambda b, h: adm[b].double())["ctx_emul"]
    got = X.reference(c["qkv"], c["d_ctx"], 1, S, heads, None, weights=lambda b, h: bad[b].double())["ctx_emul"]
    with pytest.raises(AssertionError, match=r"elements differ; first at \(3, "):
        X.exact_check(got, want, "ctx", loc)
    # random data: the softmax without that key for the same rows
    b = 0
    x = qkv.double().reshape(B, S, 3, heads, 64)
    doctored = ref["ctx"].clone()
    for h in range(heads):
        q, k, vv = x[b, :, 0, h], x[b, :, 1, h], x[b, :, 2, h]
        s = q[rows] @ k[:S - 1].t() * X.SCALE
        doctored[rows, h * 64:(h + 1) * 64] = torch.softmax(s, 1) @ vv[:S - 1]
    assert rel(doctored, ref["ctx"]) < CTX_BAR
    with pytest.raises(AssertionError, match="x the bound"):
        X.bound_check(doctored, ref["ctx"], ref["bar_ctx"], "ctx", loc)


def test_admitted_padding_key_is_caught():
    B, S, heads = 2, 129, 2
    v = X.validity("ragged", B, S)
    c = X.routed(B, S, heads, v, seed=1)
    tg = c["targets"]
    ref = X.reference(c["qkv"], c["d_ctx"], B, S, heads, v, weights=lambda b, h: X.routed_weights(tg, v, b, h, S))
    pad = int((~v[1]).nonzero()[0])

    def leaky(b, h):
        W = X.routed_weights(tg, v, b, h, S)
        if b == 1:  # a poisoned key that leaks takes all the probability of a valid row
            W[10] = 0.0
            W[10, pad] = 1.0
        return W
    got = X.reference(c["qkv"], c["d_ctx"], B, S, heads, v, weights=leaky)
    with pytest.raises(AssertionError, match=r"first at \(" + str(S + 10) + ", "):
        X.exact_check(got["ctx_emul"], ref["ctx_emul"], "ctx", loc)


def test_row_from_the_neighbouring_head_is_caught(rand_case):
    B, S, heads, v, qkv, d_ctx, ref = rand_case
    doctored = ref["ctx"].clone()
    r = S + 70
    doctored[r, 64:128] = ref["ctx"][r, 0:64]
    with pytest.raises(AssertionError, match=r"x the bound"):
        X.bound_check(doctored, ref["ctx"], ref["bar_ctx"], "ctx", lambda idx: X.where_qkv("query", B, S, heads, *idx))


def test_missing_query_chunk_in_dv_is_caught(rand_case):
    """Key tile 1 of (b 0, h 1) without query chunk 3 in its dV."""
    B, S, heads, v, qkv, d_ctx, ref = rand_case
    x = qkv.double().reshape(B, S, 3, heads, 64)
    q, k = x[0, :, 0, 1], x[0, :, 1, 1]
    vm = v[0]
    t = torch.where(vm[:, None] & vm[None], q @ k.t() * X.SCALE, torch.full((S, S), -math.inf, dtype=torch.float64))
    t = torch.where(vm[:, None], t, torch.zeros_like(t))
    P = torch.softmax(t, 1)
    dO = d_ctx.double().reshape(B, S, heads, 64)[0, :, 1]
    keys, chunk = slice(128, 256), slice(192, 256)
    doctored = ref["dqkv"].clone()
    doctored[keys, 2 * 128 + 64:3 * 128] -= P[chunk, keys].t() @ dO[chunk]
    with pytest.raises(AssertionError, match=r"K3/K4 key tile 1"):
        X.bound_check(doctored, ref["dqkv"], ref["bar_dqkv"], "dqkv", lambda idx: X.where_qkv("key", B, S, heads, *idx))


@pytest.mark.parametrize("twice", [False, True])
def test_dq_slice_twice_or_missing_is_caught(twice):
    """dQ in slices mode (S <= 512): key tile 1's slice added twice, or left out, on the routed construction's two-hot rows."""
    B, S, heads = 1, 300, 2
    c = X.routed(B, S, heads, None, seed=3)
    tg = c["targets"]
    ref = X.reference(c["qkv"], c["d_ctx"], B, S, heads, None, weights=lambda b, h: X.routed_weights(tg, None, b, h, S))
    x = c["qkv"].double().reshape(B, S, 3, heads, 64)
    doctored = ref["dqkv"].clone()
    for h in range(heads):
        W = X.routed_weights(tg, None, 0, h, S)
        P = W / W.sum(1, keepdim=True)
        k, vv = x[0, :, 1, h], x[0, :, 2, h]
        dO = c["d_ctx"].double().reshape(B, S, heads, 64)[0, :, h]
        D = (dO * ref["ctx"][:, h * 64:(h + 1) * 64]).sum(1)
        dS = P * (dO @ vv.t() - D[:, None])
        part = X.SCALE * dS[:, 128:256] @ k[128:256]
        doctored[:, h * 64:(h + 1) * 64] += part if twice else -part
    assert X.dq_parts(S) == 3
    with pytest.raises(AssertionError, match="elements differ"):
        X.exact_check(doctored.float().bfloat16(), ref["dqkv"].float().bfloat16(), "dqkv", loc)


def test_lse_off_by_one_key_is_caught(rand_case):
    B, S, heads, v, qkv, d_ctx, ref = rand_case
    doctored = ref["lse"].clone()
    doctored[1, 0, 200] += math.log1p(1.0 / S)
    X.bound_check(ref["lse"].float(), ref["lse"], ref["bar_lse"], "lse", loc, out_bf16=False)
    with pytest.raises(AssertionError, match=r"\(1, 0, 200\)"):
        X.bound_check(doctored, ref["lse"], ref["bar_lse"], "lse", loc, out_bf16=False)


def test_padding_query_in_valid_q_colsum_is_caught(rand_case):
    """One padding query row (1/S on every key) counted in the valid_q column sums: within the column-sum Frobenius bar."""
    B, S, heads, v, qkv, d_ctx, ref = rand_case
    key = (True, 0)
    want = ref["cs"][key] + ref["cs"][(True, 1)]
    bar = ref["bar_cs"][key] + ref["bar_cs"][(True, 1)]
    pad_b = 1
    assert not bool(v[pad_b].all())
    doctored = want.clone()
    doctored[pad_b] += 1.0 / S
    assert rel(doctored, want) < COLSUM_BAR
    with pytest.raises(AssertionError, match="x the bound"):
        X.bound_check(doctored, want, bar, "colsum", loc, out_bf16=False)


def test_exact_and_ulp_checks_name_the_element():
    want = torch.arange(12, dtype=torch.float32).reshape(3, 4)
    got = want.clone()
    got[2, 1] = float(np.nextafter(np.float32(9.0), np.float32(10.0)))
    with pytest.raises(AssertionError, match=r"1 of 12 elements differ; first at \(2, 1\)"):
        X.exact_check(got, want, "t", loc)
    X.ulp_check(got, want.double(), 1, "t", loc)
    got[0, 3] = 3.0 + 3 * 2.0 ** -22
    with pytest.raises(AssertionError, match=r"\(0, 3\)"):
        X.ulp_check(got, want.double(), 2, "t", loc)
