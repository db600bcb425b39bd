"""The checks of tests/rowwise_exact_oracle.py hold on a float32 restatement of the row-wise LayerNorm kernels and can fail.

Restatement.  emu_ln_fwd / emu_ln_bwd / emu_columns replay ln_fwd_kernel, ln_bwd_kernel (+ reduce_partials_kernel),
ln_bwd_fused_kernel and colsum_kernel in NumPy float32, operation by operation and in the kernels' order: each lane's chain
over its chunks, the 5-level butterfly, the IEEE division by H (fl(1/H) times the sum in the fused kernel), rsqrtf as the
correctly rounded 1/sqrt, the column sums per warp, per block and per block partial.  Once with every product-sum contracted
into an FMA (a float32 FMA is the product and sum formed in float64 and rounded once to float32; the rare double rounding is
far inside any bound) and once without.  On the GPU tests' operand generators, at every width and row class, the restatement
stays within the bounds: the worst error is 0.34 of the bound for rstd and y, 0.12 for the column sums (0.065 for colsum), and
0.98 for mean and dx where one correctly rounded operation is all that is left (the division of an exactly summed row by H;
the residual add onto a row whose LayerNorm term is tiny beside dres) -- a single rounding can come as close to u |result| as
it likes, so no bound can keep a margin there.

Doctored outputs: unbiased variance, eps 1e-6, a stale ring slot, a missing last chunk at H = 264, a dropped block partial and
dbeta off by one are each caught; where the relative-Frobenius bars of test_gpu_kernels.py (4e-3, 6e-3, 2e-3) accept the
doctored output, the test asserts that too.  Rejection: unaligned or short leading dimensions and unaligned base pointers
fail the host-side validation of all four entry points with fake addresses, before any CUDA call, on a machine without a GPU.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from merlot_b200 import _lib
from tests import rowwise_exact_oracle as R

f32, f64 = np.float32, np.float64
FWD_BAR, BWD_BAR, COL_BAR = 4e-3, 6e-3, 2e-3
FWD_WIDTHS = [8, 64, 248, 256, 264, 512, 520, 768, 776, 1016, 1024]
BWD_WIDTHS = [8, 64, 256, 264, 320, 512, 520, 768, 776, 1024]
EMU_SMS = 2  # a small grid, so that every warp of the restated backwards owns several rows


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def fma(a, b, c):
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32)


# ---------------------------------------------------------------------------------------------------------------------
# float32 restatement
# ---------------------------------------------------------------------------------------------------------------------
def lane_cols(H):
    """[32, 8 NCH] column indices lane l reads in order (chunks l, l + 32, ...), -1 where the lane has no chunk."""
    K = 8 * R.nch(H)
    idx = np.full((32, K), -1)
    for l in range(32):
        cols = [c * 8 + i for j in range(R.nch(H)) for c in [l + 32 * j] if c < H // 8 for i in range(8)]
        idx[l, :len(cols)] = cols
    return idx


def gather(v, idx):
    return np.where(idx >= 0, v[:, idx.clip(0)], f32(0)).astype(f32)


def lane_chain(a, b=None, use_fma=False, pairs=False):
    """Per-lane running sums over the last axis of a [rows, 32, K] (of a * b when b is given); pairs: the fused kernel adds
    the two values of each bf16x2 word first."""
    acc = np.zeros(a.shape[:2], f32)
    step = 2 if pairs else 1
    for k in range(0, a.shape[2], step):
        if b is None:
            t = (a[..., k] + a[..., k + 1]).astype(f32) if pairs else a[..., k]
            acc = (acc + t).astype(f32)
        elif pairs:
            t = fma(a[..., k], b[..., k], (a[..., k + 1] * b[..., k + 1]).astype(f32)) if use_fma else \
                ((a[..., k] * b[..., k]).astype(f32) + (a[..., k + 1] * b[..., k + 1]).astype(f32)).astype(f32)
            acc = (acc + t).astype(f32)
        else:
            acc = fma(a[..., k], b[..., k], acc) if use_fma else (acc + (a[..., k] * b[..., k]).astype(f32)).astype(f32)
    return acc


def butterfly(v):
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, lanes ^ o]).astype(f32)
    return v[:, 0]


def emu_ln_fwd(x, gamma, beta, eps=R.EPS, use_fma=False, unbiased=False, drop_last_chunk=False):
    """ln_fwd_kernel in float32: (y fp32, mean, rstd).  unbiased / drop_last_chunk: doctored kernels (divisor H - 1; the
    last 16-byte chunk of the row left out of the statistics)."""
    x, gamma, beta = (np.asarray(t, f32) for t in (x, gamma, beta))
    H = x.shape[1]
    idx = lane_cols(H)
    if drop_last_chunk:
        idx = np.where(idx >= H - 8, -1, idx)
    X = gather(x, idx)
    mean = (butterfly(lane_chain(X)) / f32(H)).astype(f32)
    D = np.where(idx >= 0, (X - mean[:, None, None]).astype(f32), f32(0))
    var = (butterfly(lane_chain(D, D, use_fma)) / f32(H - 1 if unbiased else H)).astype(f32)
    t = (var + f32(eps)).astype(f32)
    rstd = (1.0 / np.sqrt(t.astype(f64))).astype(f32)
    s = (rstd[:, None] * gamma[None]).astype(f32)
    ms = (mean[:, None] * s).astype(f32)
    y = fma(x, s, -ms) if use_fma else ((x * s).astype(f32) - ms).astype(f32)
    return (y + beta).astype(f32), mean, rstd


def emu_ln_bwd(dy, x, mean, rstd, gamma, dres=None, keep=None, scale=1.0, use_fma=False, fused=False):
    """ln_bwd_kernel (fused=False) or ln_bwd_fused_kernel (fused=True) per row in float32: (dx fp32, dv, xh), dv and xh the
    factors of the column terms."""
    dy, x, gamma = (np.asarray(t, f32) for t in (dy, x, gamma))
    mu, rs = np.asarray(mean, f32)[:, None], np.asarray(rstd, f32)[:, None]
    H = x.shape[1]
    dv = dy if keep is None else np.where(keep, (dy * f32(scale)).astype(f32), f32(0))
    xh = ((x - mu).astype(f32) * rs).astype(f32)
    gd = (gamma * dv).astype(f32)
    idx = lane_cols(H)
    G, XH = gather(gd, idx), gather(xh, idx)
    s1, s2 = butterfly(lane_chain(G, pairs=fused)), butterfly(lane_chain(G, XH, use_fma, pairs=fused))
    if fused:
        inv = f32(1) / f32(H)
        s1, s2 = (s1 * inv).astype(f32)[:, None], (s2 * inv).astype(f32)[:, None]
    else:
        s1, s2 = (s1 / f32(H)).astype(f32)[:, None], (s2 / f32(H)).astype(f32)[:, None]
    if use_fma:
        t = fma(gamma, dv, -s1) if fused else (gd - s1).astype(f32)
        inner = fma(-xh, s2, t)
        o = fma(rs, inner, np.asarray(dres, f32)) if dres is not None else (rs * inner).astype(f32)
    else:
        inner = ((gd - s1).astype(f32) - (xh * s2).astype(f32)).astype(f32)
        o = (rs * inner).astype(f32)
        if dres is not None:
            o = (o + np.asarray(dres, f32)).astype(f32)
    return o, dv, xh


def _warp_chains(a, b, W, use_fma):
    """[W, H] per-warp chains over rows w, w + W, ... of a (a * b)."""
    acc = np.zeros((W, a.shape[1]), f32)
    for r in range(a.shape[0]):
        w = r % W
        acc[w] = fma(a[r], b[r], acc[w]) if (b is not None and use_fma) else \
            (acc[w] + (a[r] if b is None else (a[r] * b[r]).astype(f32))).astype(f32)
    return acc


def emu_columns(a, b, prefill, sms, kind, use_fma=False, skip_block=None, launches=1):
    """The column sums of a (a * b) onto prefill as the kernel `kind` forms them: 'fused' (12-warp blocks, one red.add per
    block), 'unfused' (8-warp blocks, then reduce_partials_kernel's RSPLIT chains), 'colsum' (colsum_kernel's slabs).
    skip_block: a block whose contribution is dropped (a doctored kernel)."""
    rows = a.shape[0]
    out = np.asarray(prefill, f32).copy()
    for _ in range(launches):
        if kind == "colsum":
            Y = R.colsum_slabs(rows)
            acc = np.zeros((Y, 8, a.shape[1]), f32)
            for r in range(rows):
                y, w = (r // 8) % Y, r % 8
                acc[y, w] = (acc[y, w] + a[r]).astype(f32)
            blocks = []
            for y in range(Y):
                s = np.zeros(a.shape[1], f32)
                for w in range(8):
                    s = (s + acc[y, w]).astype(f32)
                blocks.append(s)
            parts = blocks
        else:
            nw = R.LNF_WARPS if kind == "fused" else R.LN_BWD_WARPS
            B = R.fused_grid(rows, sms) if kind == "fused" else R.unfused_grid(rows, sms)
            acc = _warp_chains(a, b, B * nw, use_fma)
            blocks = []
            for blk in range(B):
                s = acc[blk * nw].copy()
                for w in range(1, nw):
                    s = (s + acc[blk * nw + w]).astype(f32)
                blocks.append(np.zeros_like(s) if blk == skip_block else s)
            if kind == "fused":
                parts = blocks
            else:
                parts = []
                for y in range(R.RSPLIT):
                    s = np.zeros(a.shape[1], f32)
                    for blk in range(y, B, R.RSPLIT):
                        s = (s + blocks[blk]).astype(f32)
                    parts.append(s)
        for s in parts:
            out = (out + s).astype(f32)
    return out


def _params(H, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(H, generator=g), torch.randn(H, generator=g)


# ---------------------------------------------------------------------------------------------------------------------
# the restatement meets the bounds
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_fma", [False, True])
@pytest.mark.parametrize("x_dtype", [torch.bfloat16, torch.float32])
def test_restated_forward_meets_the_bounds(x_dtype, use_fma):
    worst = 0.0
    for H in FWD_WIDTHS:
        x = R.ln_rows(2 * len(R.ROW_CLASSES), H, H, x_dtype).float()
        gam, bet = _params(H, H + 1)
        y, mean, rstd = emu_ln_fwd(x.numpy(), gam.numpy(), bet.numpy(), use_fma=use_fma)
        y, mean, rstd = (torch.from_numpy(t) for t in (y, mean, rstd))
        assert R.check_exact_stats(mean, rstd, x) >= 4
        E_mean, E_rstd, E_y = R.ln_fwd_bounds(x, gam, bet)
        ref_y, ref_mean, ref_rstd = R.ln_fwd_ref(x, gam, bet)
        R.check_f32(mean, ref_mean, E_mean, f"H={H} mean")  # up to 0.97: on exact sums only the division's rounding is left
        worst = max(worst, R.check_f32(rstd, ref_rstd, E_rstd, f"H={H} rstd"), R.check_f32(y, ref_y, E_y, f"H={H} y"))
        R.check_ln_fwd(y.bfloat16(), mean, rstd, x, gam, bet, what=f"H={H} bf16")
        keep = torch.rand(x.shape, generator=torch.Generator().manual_seed(H)) > 0.1
        scale = float(np.float32(1) / (np.float32(1) - np.float32(0.1)))
        yd = np.where(keep.numpy(), (y.numpy() * f32(scale)).astype(f32), f32(0))
        R.check_ln_fwd(torch.from_numpy(yd), mean, rstd, x, gam, bet, keep=keep, scale=scale, what=f"H={H} dropout")
    assert worst < 0.4, worst  # 0.34


@pytest.mark.parametrize("use_fma", [False, True])
@pytest.mark.parametrize("fused", [False, True])
def test_restated_backward_meets_the_bounds(fused, use_fma):
    worst, worst_col = 0.0, 0.0
    for H in BWD_WIDTHS:
        rows = 61
        x = R.ln_rows(rows, H, H + 3, torch.bfloat16).float()
        mean, rstd = (torch.from_numpy(t) for t in emu_ln_fwd(x.numpy(), np.ones(H), np.zeros(H))[1:])
        g = torch.Generator().manual_seed(H)
        dy = torch.randn(rows, H, generator=g).bfloat16().float()
        dres = torch.randn(rows, H, generator=g).bfloat16().float()
        gam = torch.randn(H, generator=g)
        keep, scale = (None, 1.0) if fused else (torch.rand(rows, H, generator=g) > 0.1, float(np.float32(1) / np.float32(0.9)))
        dx, dv, xh = emu_ln_bwd(dy.numpy(), x.numpy(), mean.numpy(), rstd.numpy(), gam.numpy(), dres.numpy(), keep=keep,
                                scale=scale, use_fma=use_fma, fused=fused)
        ref, t_g, t_b = R.ln_bwd_ref(dy, x, mean, rstd, gam, dres, keep, scale)
        E_dx, e_g, e_b = R.ln_bwd_bounds(dy, x, mean, rstd, gam, dres, keep, scale)
        worst = max(worst, R.check_f32(torch.from_numpy(dx), ref, E_dx, f"H={H} dx"))
        R.check_bf16(torch.from_numpy(dx).bfloat16(), ref, E_dx, f"H={H} dx bf16")
        kind = "fused" if fused else "unfused"
        depth = (R.col_depth_fused if fused else R.col_depth_unfused)(rows, EMU_SMS, launches=2)
        P = torch.randint(-4, 5, (H,), generator=g).float()
        for a, b, terms, err in ((dv, xh, t_g, e_g), (dv, None, t_b, e_b)):
            got = emu_columns(a, b, P.numpy(), EMU_SMS, kind, use_fma, launches=2)
            want, E = R.col_ref_bound(terms, err, P, depth, launches=2)
            worst_col = max(worst_col, R.check_f32(torch.from_numpy(got), want, E, f"H={H} columns"))
    assert worst <= 1.0 and worst_col < 0.25, (worst, worst_col)  # 0.98 (see the module docstring) and 0.12


def test_restated_colsum_meets_the_bound_and_integer_sums_are_exact():
    g = torch.Generator().manual_seed(0)
    for rows, N in [(1, 8), (65, 264), (700, 248)]:
        dy = torch.randn(rows, N, generator=g).bfloat16().float()
        P = torch.randn(N, generator=g)
        got = emu_columns(dy.numpy(), None, P.numpy(), None, "colsum")
        want, E = R.col_ref_bound(dy.double(), torch.zeros(rows, N, dtype=torch.float64), P, R.col_depth_colsum(rows))
        assert R.check_f32(torch.from_numpy(got), want, E, "colsum") < 0.25  # 0.065
        di = R.int_rows(rows, N, rows, dtype=torch.float32) * 2  # p = 0.5: kept values times exactly 2
        Pi = torch.randint(-1000, 1000, (N,), generator=g).float()
        assert R.exact_int_sum_holds(di, Pi)
        got = emu_columns(di.numpy(), None, Pi.numpy(), None, "colsum", launches=2)
        R.exact_check(torch.from_numpy(got), (Pi.double() + 2 * di.double().sum(0)).float(), "integer colsum")


def test_row_classes_and_geometry():
    x = R.ln_rows(16, 264, 0, torch.bfloat16)
    assert R.exact_stats_rows(x).sum() == 6  # zero_sum, constant and zero rows, twice each
    zs = x[[i for i in range(16) if R.ROW_CLASSES[i % 8] == "zero_sum"]].double()
    assert (zs.sum(-1) == 0).all() and (zs.abs().max() <= 8) and ((zs * zs).sum(-1) < 2 ** 24).all()
    assert [R.nch(H) for H in (8, 256, 264, 520, 776, 1024)] == [1, 1, 2, 3, 4, 4]
    assert (lane_cols(264) >= 0).sum(1).tolist() == [16] + [8] * 31  # only lane 0 owns a second chunk
    assert R.col_depth_fused(12 * 132, 132) == 1 + 12 + 132 + 1 and R.col_depth_fused(12 * 132 + 1, 132) == 2 + 12 + 132 + 1
    assert R.colsum_slabs(8192) == 128 and R.colsum_slabs(8193) == 128 and R.colsum_slabs(65) == 2


# ---------------------------------------------------------------------------------------------------------------------
# doctored outputs
# ---------------------------------------------------------------------------------------------------------------------
def _fwd_problem(H=768, rows=64, dtype=torch.bfloat16):
    x = R.ln_rows(rows, H, 5, dtype).float()
    gam, bet = _params(H, 9)
    return x, gam, bet


def test_unbiased_variance_is_caught_where_the_bf16_bar_is_not():
    x, gam, bet = _fwd_problem()
    y, mean, rstd = (torch.from_numpy(t) for t in emu_ln_fwd(x.numpy(), gam.numpy(), bet.numpy(), unbiased=True))
    ref_y = R.ln_fwd_ref(x, gam, bet)[0]
    assert rel(y.bfloat16(), ref_y) < FWD_BAR  # the old bar accepts the bf16 output
    exact = R.exact_stats_rows(x)
    first_zero_sum = next(i for i in range(64) if R.ROW_CLASSES[(i + 5) % 8] == "zero_sum")
    assert exact[first_zero_sum]
    with pytest.raises(AssertionError, match=rf"rstd of exact rows \(2 ulp\): 8 of 64 elements differ; first at \({first_zero_sum},\)"):
        R.check_ln_fwd(y.bfloat16(), mean, rstd, x, gam, bet)
    with pytest.raises(AssertionError, match="y: .* elements differ"):  # and the fp32 output on its own
        R.check_ln_fwd(y, None, None, x, gam, bet)
    with pytest.raises(AssertionError, match="rstd: .* elements differ"):
        R.check_f32(rstd, R.ln_fwd_ref(x, gam, bet)[2], R.ln_fwd_bounds(x, gam, bet)[1], "rstd")


def test_wrong_eps_on_rows_with_variance_near_eps_is_caught():
    _, gam, bet = _fwd_problem(H=256)
    x = R.ln_rows(32, 256, 1, torch.bfloat16, classes=("near_eps",)).float()
    y, mean, rstd = (torch.from_numpy(t) for t in emu_ln_fwd(x.numpy(), gam.numpy(), bet.numpy(), eps=1e-6))
    with pytest.raises(AssertionError, match="rstd: 32 of 32 elements differ"):
        R.check_ln_fwd(y, mean, rstd, x, gam, bet)
    R.check_ln_fwd(*(torch.from_numpy(t) for t in emu_ln_fwd(x.numpy(), gam.numpy(), bet.numpy())), x, gam, bet)


def test_missing_last_chunk_at_h_264_is_caught():
    """nchunk = 33: lane 0 alone owns chunk 32.  A kernel that leaves it out of the statistics (NCH taken as H / 256)."""
    x, gam, bet = _fwd_problem(H=264, rows=16)
    y, mean, rstd = (torch.from_numpy(t) for t in emu_ln_fwd(x.numpy(), gam.numpy(), bet.numpy(), drop_last_chunk=True))
    with pytest.raises(AssertionError, match="elements differ"):
        R.check_ln_fwd(y.bfloat16(), mean, rstd, x, gam, bet)


@pytest.fixture(scope="module")
def many_rows():
    """120000 rows of H = 64 and the bf16 dx the fused backward should give."""
    rows, H = 120000, 64
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(rows, H, generator=g) * 2 + 0.5).bfloat16().float()
    mean = x.mean(-1)
    rstd = torch.rsqrt(x.var(-1, unbiased=False) + 1e-5)
    dy = torch.randn(rows, H, generator=g).bfloat16().float()
    gam = torch.randn(H, generator=g)
    ref, _, _ = R.ln_bwd_ref(dy, x, mean, rstd, gam)
    E, _, _ = R.ln_bwd_bounds(dy, x, mean, rstd, gam)
    return dict(x=x, mean=mean, rstd=rstd, dy=dy, gam=gam, ref=ref, E=E)


def test_stale_ring_slot_row_is_caught_where_the_bar_is_not(many_rows):
    """One row of dx replaced by the row another warp reduced (a ring slot read one phase late): sqrt(2 / rows) in relative
    Frobenius norm, which the 6e-3 bar accepts from about 60000 rows on."""
    ref, E = many_rows["ref"], many_rows["E"]
    good = ref.bfloat16()
    R.check_bf16(good, ref, E, "dx")
    got = good.clone()
    got[31337] = good[31337 + 12 * 132]
    assert rel(got, ref) < BWD_BAR
    with pytest.raises(AssertionError, match=r"dx: \d+ of 7680000 elements differ; first at \(31337, "):
        R.check_bf16(got, ref, E, "dx")


def test_dropped_block_partial_is_caught():
    rows, H = 300, 264
    g = torch.Generator().manual_seed(2)
    x = R.ln_rows(rows, H, 7, torch.bfloat16).float()
    mean, rstd = (torch.from_numpy(t) for t in emu_ln_fwd(x.numpy(), np.ones(H), np.zeros(H))[1:])
    dy = torch.randn(rows, H, generator=g).bfloat16().float()
    gam = torch.randn(H, generator=g)
    _, dv, xh = emu_ln_bwd(dy.numpy(), x.numpy(), mean.numpy(), rstd.numpy(), gam.numpy(), fused=True)
    _, t_g, _ = R.ln_bwd_ref(dy, x, mean, rstd, gam)
    _, e_g, _ = R.ln_bwd_bounds(dy, x, mean, rstd, gam)
    P = torch.zeros(H)
    want, E = R.col_ref_bound(t_g, e_g, P, R.col_depth_fused(rows, 8))
    R.check_f32(torch.from_numpy(emu_columns(dv, xh, P.numpy(), 8, "fused")), want, E, "dgamma")
    got = torch.from_numpy(emu_columns(dv, xh, P.numpy(), 8, "fused", skip_block=5))
    with pytest.raises(AssertionError, match="dgamma: .* elements differ"):
        R.check_f32(got, want, E, "dgamma")


def test_dbeta_off_by_one_is_caught_where_the_bar_is_not():
    rows, H = 60000, 768
    dy = R.int_rows(rows, H, 3)
    P = torch.randint(-100, 100, (H,), generator=torch.Generator().manual_seed(0)).float()
    assert R.exact_int_sum_holds(dy, P)
    want = (P.double() + dy.double().sum(0)).float()
    got = want.clone()
    got[100] += 1
    assert rel(got - P, want - P) < COL_BAR
    with pytest.raises(AssertionError, match=r"dbeta: 1 of 768 elements differ; first at \(100,\)"):
        R.exact_check(got, want, "dbeta")


def test_bf16_check_admits_the_neighbour_only_next_to_a_midpoint():
    ref = torch.tensor([1.0 + 2 ** -8, 1.0 + 2 ** -8 + 2 ** -12, 3.0], dtype=torch.float64)  # a midpoint, off it, a bf16 value
    E = torch.tensor([2 ** -20, 2 ** -20, 2 ** -20], dtype=torch.float64)
    assert R.check_bf16(torch.tensor([1.0, 1.0078125, 3.0]).bfloat16(), ref, E, "t") == 0  # ties to even: 1.0
    assert R.check_bf16(torch.tensor([1.0078125, 1.0078125, 3.0]).bfloat16(), ref, E, "t") == 1  # the neighbour, admitted
    with pytest.raises(AssertionError, match=r"1 of 3 elements differ; first at \(1,\)"):
        R.check_bf16(torch.tensor([1.0, 1.0, 3.0]).bfloat16(), ref, E, "t")


# ---------------------------------------------------------------------------------------------------------------------
# host-side validation, with fake device addresses (no GPU needed: every case fails before any CUDA call)
# ---------------------------------------------------------------------------------------------------------------------
A = 0x7F0000000000  # a 16-byte aligned fake address; A + 8 is not


def _rejects(call, match):
    lib = _lib.lib()
    n = lib.merlot_launch_count()
    with pytest.raises(_lib.MerlotError, match=match) as e:
        call()
    assert e.value.code in (_lib.MERLOT_EINVAL, _lib.MERLOT_ESHAPE), e.value.code  # a validation failure, not a CUDA error
    assert lib.merlot_launch_count() == n


def _fwd_desc(**kw):
    d = _lib.merlot_ln_t()
    d.x, d.ld_x, d.y, d.ld_y, d.gamma, d.beta = A, 264, A + 0x100000, 264, A + 0x200000, A + 0x201000
    d.H, d.eps, d.rows = 264, 1e-5, 0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _bwd_desc(**kw):
    d = _lib.merlot_ln_bwd_t()
    d.dy, d.ld_dy, d.x, d.ld_x, d.dres, d.ld_dres, d.dx, d.ld_dx = A, 264, A + 0x100000, 264, A + 0x200000, 264, A + 0x300000, 264
    d.mean, d.rstd, d.gamma, d.dgamma, d.dbeta, d.workspace = (A + 0x400000 + 0x1000 * i for i in range(6))
    d.H, d.rows = 264, 0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_valid_fake_descriptors_pass_the_checks_without_a_gpu():
    """rows = 0 with every argument valid returns before any CUDA call: the rejections below are each due to one field."""
    lib = _lib.lib()
    assert lib.merlot_layernorm_fwd(C.byref(_fwd_desc()), None) == 0
    assert lib.merlot_layernorm_bwd(C.byref(_bwd_desc()), None) == 0
    assert lib.merlot_layernorm_bwd(C.byref(_bwd_desc(dres=None, ld_dres=0)), None) == 0  # ld_dres unused without dres
    assert lib.merlot_layernorm_bwd_fused(*_fused_args(), None) == 0
    assert lib.merlot_bias_grad(A, 0, 264, 0, 264, A + 0x1000, 0.0, 0, 0, None) == 0


@pytest.mark.parametrize("field,value", [("ld_x", 260), ("ld_y", 268), ("ld_x", 256), ("ld_y", 8),
                                         ("x", A + 8), ("y", A + 0x100000 + 4), ("gamma", A + 0x200004), ("beta", A + 0x201008)])
def test_layernorm_fwd_rejects_unaligned_or_short_rows(field, value):
    lib = _lib.lib()
    _rejects(lambda: lib.merlot_layernorm_fwd(C.byref(_fwd_desc(**{field: value})), None),
             "leading dims" if field.startswith("ld") else "16-byte aligned")


@pytest.mark.parametrize("field,value", [("ld_dy", 268), ("ld_x", 270), ("ld_dres", 260), ("ld_dx", 2), ("ld_dy", 256),
                                         ("ld_x", 8), ("ld_dres", 0), ("ld_dx", 256), ("dy", A + 8), ("x", A + 0x100002),
                                         ("dres", A + 0x200008), ("dx", A + 0x300004), ("gamma", A + 0x402008)])
def test_layernorm_bwd_rejects_unaligned_or_short_rows(field, value):
    lib = _lib.lib()
    _rejects(lambda: lib.merlot_layernorm_bwd(C.byref(_bwd_desc(**{field: value})), None),
             "leading dims" if field.startswith("ld") else "16-byte aligned")


def test_layernorm_bwd_rejects_a_dtype_combination_before_any_cuda_call():
    lib = _lib.lib()
    _rejects(lambda: lib.merlot_layernorm_bwd(C.byref(_bwd_desc(x_f32=1, dx_f32=0, rows=5)), None), "dtype combination")


FUSED_ARGS = ["dy", "x", "mean", "rstd", "gamma", "dres", "dx", "dmask", "dgamma", "dbeta", "dbias"]


def _fused_args(rows=0, **bad):
    ptrs = [bad.get(n, A + 0x100000 * i) for i, n in enumerate(FUSED_ARGS)]
    return (*ptrs, None, rows, 264, 0.1, 0, 0)


@pytest.mark.parametrize("name,off", [("dy", 8), ("x", 2), ("dres", 8), ("dx", 4), ("dmask", 8), ("gamma", 4),
                                      ("dgamma", 8), ("dbeta", 4), ("dbias", 12)])
def test_layernorm_bwd_fused_rejects_unaligned_pointers(name, off):
    lib = _lib.lib()
    _rejects(lambda: lib.merlot_layernorm_bwd_fused(*_fused_args(rows=7, **{name: A + 0x100000 * FUSED_ARGS.index(name) + off}),
                                                    None), "16-byte aligned")


@pytest.mark.parametrize("ld,N,dy", [(260, 256, A), (248, 256, A), (0, 8, A), (264, 264, A + 8), (264, 264, A + 2)])
def test_bias_grad_rejects_unaligned_or_short_rows(ld, N, dy):
    lib = _lib.lib()
    _rejects(lambda: lib.merlot_bias_grad(dy, 0, ld, 100, N, A + 0x10000, 0.0, 0, 0, None), "multiples of 8|16-byte aligned")
