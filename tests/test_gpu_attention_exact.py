"""The fused attention kernels element by element (pytest -m gpu): K2 forward and its LSE, K3 backward with the dsum and dQ
finish passes and the q/k/v bias gradient, K4 column sums (plain, split into two buffers, valid queries only) and the
probability export, on the constructions and bounds of tests/attention_exact_oracle.py.

- Routed softmax: every output bitwise (torch.equal), except fp32 sums whose order the kernels leave open (stated per check).
- Counting: the admitted set of every query row, through ctx bitwise; K3 on d_ctx = 0 gives exactly zero.
- Random data: every element within its bound; the worst error-to-bound ratio per output is printed (run with -s).

The sweep straddles the 64-key K2 tile, the 128-key K3/K4 tile, the 64-query chunk, the 32-position mask word, the slices /
atomic dQ boundary (S = 512 / 513) and the longest accepted sequence (3968); B up to 3, so the last tiles of one sequence
read the next one's rows; every mask kind; packed and wider pitches, with each operand in a NaN-filled buffer and every
element outside the outputs' views checked to be NaN afterwards; and the dQ workspace as consecutive layers hand it over
(atomic mode returns it exactly zero, slices mode ignores the NaN left in it)."""

import pytest
import torch

from tests import attention_exact_oracle as X

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
LENGTHS = [1, 63, 64, 65, 127, 128, 129, 191, 255, 256, 257, 511, 512, 513, 640, 1100, 3968]
KINDS = ["none", "ragged", "len1", "empty", "pair"]
# P of a padding query row (or of any counting row) is ex2(-lse log2 e) with the LSE within 4 fp32 ulps of ln n (log2f is
# within 1 ulp, and the products by ln 2 and log2 e round twice): relative error <= 4 * 2^-23 * ln(4096) + 2^-22 < 2^-17
EPS_P = 2.0 ** -17
LSE_ULPS = 4
WORST = {}


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst error / bound on random data: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def dims(S, kind):
    """(B, heads): S = 3968 runs at B = 1 and 2 heads, long sequences at B = 2, the rest cycle through B in {1, 2, 3} and
    heads in {1, 2, 12}."""
    if S >= 3968:
        return 1, 2
    if S > 640:
        return 2, 2
    i = LENGTHS.index(S) + KINDS.index(kind)
    B = (1, 2, 3)[i % 3]
    heads = (1, 2, 12)[(i // 3) % 3] if S <= 257 else 2
    if kind in ("len1", "empty") and B == 1:
        B = 2
    return B, heads


def wide_for(S, kind):
    return (LENGTHS.index(S) + KINDS.index(kind)) % 2 == 1


def nan_view(rows, cols, dtype, wide, extra_cols=24):
    """A [rows, cols] view; wide: into a NaN-filled buffer with 3 more rows and a wider row pitch.  Returns (buf, view)."""
    if not wide:
        t = torch.full((rows, cols), NAN, dtype=dtype, device=DEV)
        return t, t
    buf = torch.full((rows + 3, cols + extra_cols), NAN, dtype=dtype, device=DEV)
    return buf, buf[:rows, :cols]


def outside_is_nan(buf, rows, cols, what):
    if buf.shape == (rows, cols):
        return
    assert bool(torch.isnan(buf[:, cols:].float()).all()) and bool(torch.isnan(buf[rows:].float()).all()), \
        f"{what}: wrote outside its [{rows}, {cols}] view"


def run(ops, qkv, d_ctx, B, S, heads, v, pair, wide, split, bias_start=True):
    """Every kernel once, from (wide) NaN-padded views; returns the outputs on the CPU."""
    H = heads * 64
    vd = None if v is None else v.to(torch.uint8).reshape(-1).contiguous().to(DEV)
    qbuf, qv = nan_view(B * S, 3 * H, torch.bfloat16, wide, extra_cols=72)
    qv.copy_(qkv)
    cbuf, cv = nan_view(B * S, H, torch.bfloat16, wide, extra_cols=40)
    dbuf = torch.full_like(cbuf, NAN)
    dv = dbuf[:B * S, :H]
    dv.copy_(d_ctx)
    lse = torch.full((B, heads, S), NAN, device=DEV)
    ops.attention_fwd(qv, B, S, heads, vd, ctx=cv, lse=lse, pair=pair)
    outside_is_nan(cbuf, B * S, H, "ctx")
    xbuf, xv = nan_view(B * S, 3 * H, torch.bfloat16, wide, extra_cols=24)
    dsum = torch.full((B, heads, S), NAN, device=DEV)
    start = torch.arange(3 * H, dtype=torch.float32, device=DEV) % 7 - 3
    if not bias_start:
        start.zero_()
    bias = start.clone()
    ws = ops.attention_bwd_workspace(B, S, heads, DEV)
    parts = X.dq_parts(S)
    if parts:
        ws.fill_(NAN)  # slices mode overwrites every slice
    ops.attention_bwd(qv, cv, dv, lse, B, S, heads, vd, dqkv=xv, dq_accum=ws, dsum=dsum, pair=pair, d_bias_qkv=bias)
    outside_is_nan(xbuf, B * S, 3 * H, "dqkv")
    if not parts:
        assert torch.equal(ws, torch.zeros_like(ws)), "atomic mode must hand the dQ workspace back zeroed"
    cs = torch.zeros(B, S, device=DEV)
    ops.attention_colsum(qv, lse, cs, B, S, heads, vd, pair=pair)
    c1, c2 = torch.zeros(B, S, device=DEV), torch.zeros(B, S, device=DEV)
    ops.attention_colsum(qv, lse, c1, B, S, heads, vd, pair=pair, colsum2=c2, split=split, valid_q=vd is not None)
    ex = ops.attention_probs(qv, lse, B, S, heads, vd, pair=pair)
    out = dict(ctx=cv, lse=lse, D=dsum, dqkv=xv, bias=bias, cs=cs, c1=c1, c2=c2, export=ex)
    return {k: t.cpu() for k, t in out.items()}, start.cpu()


def locators(B, S, heads):
    H = heads * 64

    def rows(idx):
        return X.where_qkv("query", B, S, heads, *idx)

    def qkv_cols(idx):
        return X.where_qkv("query" if idx[1] < H else "key", B, S, heads, *idx) + f" block {'qkv'[idx[1] // H]}"

    def bhs(idx):
        return X.where_bhs(B, S, heads, idx)

    def keys(idx):
        b, k = idx[-2:]
        return f"(b={b}, key={k}) [K3/K4 key tile {k // X.AT_N}, word {k // 32}]" + (f" query {idx[1]}" if len(idx) == 3 else "")

    def export(idx):
        b, q, k = idx
        return f"(b={b}, q={q}, k={k}) [query chunk {q // X.BQ}, key tile {k // X.AT_N}, word {k // 32}]"
    return dict(ctx=rows, dqkv=qkv_cols, lse=bhs, D=bhs, cs=keys, export=export, bias=lambda idx: f"column {idx[0]}")


def case(S, kind):
    B, heads = dims(S, kind)
    v = X.validity(kind, B, S)
    pair = X.pair_for(S) if kind == "pair" else (0, 0)
    return B, heads, v, pair, S // 2 + 1


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("S", LENGTHS)
def test_routed_exact(ops, S, kind):
    B, heads, v, pair, split = case(S, kind)
    c = X.routed(B, S, heads, v, pair, seed=S * 7 + KINDS.index(kind))
    tg = c["targets"]
    ref = X.reference(c["qkv"], c["d_ctx"], B, S, heads, v, pair, split=split, device=DEV,
                      weights=lambda b, h: X.routed_weights(tg, v, b, h, S))
    got, start = run(ops, c["qkv"], c["d_ctx"], B, S, heads, v, pair, wide_for(S, kind), split)
    L = locators(B, S, heads)
    tag = f"S={S} {kind} B={B} heads={heads}"
    vm = X.valid_or_ones(v, B, S)
    X.exact_check(got["ctx"], ref["ctx_emul"], f"ctx {tag}", L["ctx"])
    vb = vm[:, None, :].expand(B, heads, S)
    X.exact_check(got["lse"][vb], ref["lse"][vb].float(), f"lse (valid rows: 0 or ln 2) {tag}", lambda i: f"valid entry {i}")
    if bool((~vb).any()):
        X.ulp_check(got["lse"][~vb], ref["lse"][~vb], LSE_ULPS, f"lse (padding rows: ln S) {tag}", lambda i: f"padding entry {i}")
    X.exact_check(got["D"], ref["D"].float(), f"D {tag}", L["D"])
    want_dqkv = ref["dqkv"].float().bfloat16()
    X.exact_check(got["dqkv"], want_dqkv, f"dqkv {tag}", L["dqkv"])
    X.exact_check(got["bias"], (start.double() + want_dqkv.double().sum(0)).float(), f"bias gradient {tag}", L["bias"])
    # column sums over valid queries: per head an exact fp32 sum of 1s and 1/2s, divided by heads, added over heads in an open
    # order: exact for heads <= 2, within `heads` fp32 ulps otherwise (each of the <= heads roundings is <= 1/2 ulp)
    for name, key in (("c1", (v is not None, 0)), ("c2", (v is not None, 1))):
        want = ref["cs"][key]
        if v is not None or not bool((~vm).any()):
            X.ulp_check(got[name], want, 0 if heads <= 2 else heads, f"colsum {name} {tag}", L["cs"])
    # all queries: padding query rows add ~1/S each, with P's relative error EPS_P, to K4's fp32 running sum over <= S
    # queries (relative error gam = 2 (S + 64) 2^-24, as in the random-data model)
    want = ref["cs"][(False, 0)] + ref["cs"][(False, 1)]
    n_pad = (~vm).sum(1, keepdim=True).double()
    bar = (heads * 2.0 ** -23 + 2 * (S + 64) * X.U) * want + n_pad / S * EPS_P
    X.bound_check(got["cs"], want, bar, f"colsum {tag}", L["cs"], out_bf16=False)
    # export: valid rows exactly fl(sum_h P_h * fl(1 / heads)); padding rows ~1/S
    acc = (ref["export"] * heads * 2).round() / 2
    want_ex = acc.float() * torch.tensor(1.0 / heads, dtype=torch.float32)
    rows = vm[:, :, None].expand(B, S, S)
    X.exact_check(got["export"][rows], want_ex[rows], f"export (valid rows) {tag}", lambda i: f"valid element {i}")
    if bool((~rows).any()):
        X.bound_check(got["export"][~rows], ref["export"][~rows], ref["export"][~rows] * (EPS_P + 2.0 ** -21 + heads * 2.0 ** -23),
                      f"export (padding rows) {tag}", lambda i: f"padding element {i}", out_bf16=False)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("S", LENGTHS)
def test_counting_exact(ops, S, kind):
    B, heads, v, pair, split = case(S, kind)
    c = X.counting(B, S, heads)
    adm = X.admitted(v, B, S, pair)
    ref = X.reference(c["qkv"], c["d_ctx"], B, S, heads, v, pair, split=split, device=DEV, weights=lambda b, h: adm[b].double())
    got, start = run(ops, c["qkv"], c["d_ctx"], B, S, heads, v, pair, not wide_for(S, kind), split)
    L = locators(B, S, heads)
    tag = f"S={S} {kind} B={B} heads={heads}"
    n = adm.sum(2)  # [B, S]

    def ctx_loc(idx):
        r, col = idx
        b, i = divmod(r, S)
        h = (col % (heads * 64)) // 64
        want = (adm[b, i].double() @ c["qkv"].double()[b * S:(b + 1) * S, 2 * heads * 64 + h * 64:2 * heads * 64 + h * 64 + 64])
        cnt = X.decode_counts(got["ctx"][r, h * 64:h * 64 + 64].float(), int(n[b, i]))
        diff = (cnt - want.long()).nonzero().flatten().tolist()
        what = [f"position {d} of a word" if d < 32 else f"word {d - 32} (mod 32)" for d in diff[:4]]
        return f"{L['ctx'](idx)}: {int(n[b, i])} admitted keys; the counts differ at {', '.join(what)}"
    X.exact_check(got["ctx"], ref["ctx_emul"], f"ctx {tag}", ctx_loc)
    X.ulp_check(got["lse"], ref["lse"], LSE_ULPS, f"lse = ln(admitted count) {tag}", L["lse"])
    X.exact_check(got["D"], torch.zeros(B, heads, S), f"D {tag}", L["D"])
    X.exact_check(got["dqkv"], torch.zeros(B * S, 3 * heads * 64, dtype=torch.bfloat16), f"dqkv (d_ctx = 0) {tag}", L["dqkv"])
    X.exact_check(got["bias"], start, f"bias gradient {tag}", L["bias"])
    gam = 2 * (S + 64) * X.U
    for name, want in (("cs", ref["cs"][(False, 0)] + ref["cs"][(False, 1)]), ("c1", ref["cs"][(v is not None, 0)]),
                       ("c2", ref["cs"][(v is not None, 1)])):
        X.bound_check(got[name], want, want * (EPS_P + gam + heads * 2.0 ** -23), f"colsum {name} {tag}", L["cs"], out_bf16=False)
    X.bound_check(got["export"], ref["export"], ref["export"] * (EPS_P + 2.0 ** -21 + heads * 2.0 ** -23), f"export {tag}",
                  L["export"], out_bf16=False)


RANDOM = [(63, "none", False), (129, "ragged", False), (257, "pair", False), (512, "ragged", True), (513, "empty", False),
          (640, "pair", True), (1100, "ragged", False), (191, "len1", True), (65, "none", True), (3968, "none", True),
          (3968, "ragged", False)]


@pytest.mark.parametrize("S,kind,peaked", RANDOM)
def test_random_within_bounds(ops, S, kind, peaked):
    B, heads, v, pair, split = case(S, kind)
    qkv, d_ctx = X.random_case(B, S, heads, seed=S + 11 * KINDS.index(kind), peaked=peaked)
    ref = X.reference(qkv, d_ctx, B, S, heads, v, pair, split=split, bounds=True, device=DEV)
    got, _ = run(ops, qkv, d_ctx, B, S, heads, v, pair, wide_for(S, kind), split, bias_start=False)
    L = locators(B, S, heads)
    tag = f"S={S} {kind} peaked={peaked} B={B} heads={heads}"
    H = heads * 64
    ratios = dict(ctx=X.bound_check(got["ctx"], ref["ctx"], ref["bar_ctx"], f"ctx {tag}", L["ctx"]),
                  lse=X.bound_check(got["lse"], ref["lse"], ref["bar_lse"], f"lse {tag}", L["lse"], out_bf16=False),
                  D=X.bound_check(got["D"], ref["D"], ref["bar_D"], f"D {tag}", L["D"], out_bf16=False),
                  bias=X.bound_check(got["bias"], ref["bias"], ref["bar_bias"], f"bias gradient {tag}", L["bias"], out_bf16=False),
                  export=X.bound_check(got["export"], ref["export"], ref["bar_export"], f"export {tag}", L["export"], out_bf16=False))
    for i, name in enumerate(("dq", "dk", "dv")):
        blk = slice(i * H, (i + 1) * H)
        ratios[name] = X.bound_check(got["dqkv"][:, blk], ref["dqkv"][:, blk], ref["bar_dqkv"][:, blk], f"{name} {tag}",
                                     lambda idx, i=i: L["dqkv"]((idx[0], idx[1] + i * H)))
    cs = ref["cs"]
    bcs = ref["bar_cs"]
    vq = v is not None
    ratios["colsum"] = max(
        X.bound_check(got["cs"], cs[(False, 0)] + cs[(False, 1)], bcs[(False, 0)] + bcs[(False, 1)], f"colsum {tag}", L["cs"], out_bf16=False),
        X.bound_check(got["c1"], cs[(vq, 0)], bcs[(vq, 0)], f"colsum (queries < {split}) {tag}", L["cs"], out_bf16=False),
        X.bound_check(got["c2"], cs[(vq, 1)], bcs[(vq, 1)], f"colsum2 (queries >= {split}) {tag}", L["cs"], out_bf16=False))
    for k, r in ratios.items():
        WORST[k] = max(WORST.get(k, 0.0), r)
