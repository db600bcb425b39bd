"""The row-wise LayerNorm kernels element by element against float64 (tests/rowwise_exact_oracle.py; pytest -m gpu).

merlot_layernorm_fwd: every width class (H % 256 in {0, 8, 248}, one to four chunks per lane), the four x / y dtype pairs,
row counts around one block of 8 rows, every row class; mean and rstd per row, exact statistics on the integer rows, y per
element; strided rows, remapped rows and dropout, with NaN sentinels in the columns past H and in the rows the remap skips.
merlot_layernorm_bwd: its four dtype triples, strided views, remap and dropout, row counts that cross the 2 x SMs grid cap
into the grid-stride loop, non-zero prefilled accumulators.  merlot_layernorm_bwd_fused: every NCH with and without partial
lanes, row counts on the ring's edges (one row per warp, exactly one lap of 3 stages, one past), dres / dbias / dropout, two
launches onto prefilled accumulators, once under merlot_set_sm_reserve.  merlot_bias_grad: slab-count edges, strided fp32 and
bf16 rows.  Integer dy makes dbeta and the bias gradient bit-exact.  Last, references that are wrong on purpose must miss.
"""
import itertools

import numpy as np
import pytest
import torch

from oracle import dropout_mask as DM
from tests import rowwise_exact_oracle as R
from tests.test_gpu_sm_reserve import sm_reserve

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
BF, F = torch.bfloat16, torch.float32
DROPS = [(0.1, 2 ** 40 + 3, 223), (0.5, 7, 3), (0.1, 0, 1)]  # (p, seed, site)


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def keep_of(p, seed, site, rows, N):
    return torch.from_numpy(DM.counter_dropout_keep(seed, site, rows, N, p)).to(DEV)


def scale_of(p):
    return float(DM.dropout_scale(p))


def in_nan(t, extra_cols=0, extra_rows=0, at=None):
    """(buffer, view): t copied into a NaN-filled device buffer with extra columns (a row pitch past H) and rows; `at` places
    the rows of t at those buffer rows (a remap)."""
    rows, H = t.shape
    n = rows + extra_rows if at is None else int(at.max()) + 1 + extra_rows
    buf = torch.full((n, H + extra_cols), NAN, dtype=t.dtype, device=DEV)
    if at is None:
        buf[:rows, :H] = t.to(DEV)
    else:
        buf[at.to(DEV), :H] = t.to(DEV)
    return buf, buf[:, :H]


def nan_outside(buf, H, rows_used, what):
    outside = torch.ones(buf.shape[0], dtype=torch.bool, device=DEV)
    outside[rows_used] = False
    assert bool(buf[:, H:].float().isnan().all()), f"{what}: wrote past column H"
    assert bool(buf[outside].float().isnan().all()), f"{what}: wrote a row it does not own"


def remap_rows(rows, remap):
    per, stride, off = remap
    r = torch.arange(rows)
    return (r // per) * stride + off + r % per if per > 0 else r


def rand_gradient(rows, H, seed, dtype, integer):
    """Integers in [-8, 8] (dbeta and the bias gradients become exact sums) or 2 N(0, 1), rounded to dtype, on the GPU."""
    g = torch.Generator(device=DEV).manual_seed(int(seed))
    if integer:
        return torch.randint(-8, 9, (rows, H), generator=g, device=DEV).to(dtype)
    return (torch.randn(rows, H, generator=g, device=DEV) * 2).to(dtype)


def params(H, seed):
    g = torch.Generator().manual_seed(int(seed))
    return torch.randn(H, generator=g).to(DEV), torch.randn(H, generator=g).to(DEV)


def stats_of(x):
    """fp32 mean and rstd of x's rows (what a forward hands the backward)."""
    x64 = x.to(DEV).double()
    m = x64.mean(-1)
    return m.float(), (1.0 / torch.sqrt(((x64 - m[:, None]) ** 2).mean(-1) + R.eps32())).float()


# ---------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------
FWD_WIDTHS = [8, 64, 248, 256, 264, 512, 520, 768, 776, 1016, 1024]
FWD_DTYPES = [(BF, BF), (F, BF), (F, F), (BF, F)]
FWD_ROWS = [1, 7, 8, 9, 4097]
# (extra columns of x and y, row remap, dropout): contiguous; strided; strided + remap + dropout; dropout
FWD_LAYOUTS = [(0, (0, 0, 0), None), (8, (0, 0, 0), None), (16, (3, 5, 1), DROPS[0]), (0, (0, 0, 0), DROPS[1])]
FWD_CASES = [(*c, FWD_LAYOUTS[i % len(FWD_LAYOUTS)]) for i, c in enumerate(itertools.product(FWD_WIDTHS, FWD_DTYPES, FWD_ROWS))]


def run_fwd(ops, x, gam, bet, xdt, ydt, extra, remap, drop, eps=R.EPS):
    rows, H = x.shape
    orow = remap_rows(rows, remap)
    xbuf, xv = in_nan(x.to(xdt), extra, 2)
    ybuf = torch.full((int(orow.max()) + 1 + (4 if remap[0] else 2), H + extra), NAN, dtype=ydt, device=DEV)
    mean, rstd = torch.full((rows,), NAN, device=DEV), torch.full((rows,), NAN, device=DEV)
    ops.layernorm_fwd(xv[:rows], ybuf[:, :H], gam, bet, mean, rstd, rows=rows, remap=remap, dropout=drop or (0.0, 0, 0), eps=eps)
    return ybuf, orow, mean, rstd


@pytest.mark.parametrize("H,dts,rows,layout", FWD_CASES)
def test_layernorm_fwd_exact(ops, H, dts, rows, layout):
    xdt, ydt = dts
    extra, remap, drop = layout
    seed = H * 7 + rows
    x = R.ln_rows(rows, H, seed, xdt)
    gam, bet = params(H, seed)
    ybuf, orow, mean, rstd = run_fwd(ops, x, gam, bet, xdt, ydt, extra, remap, drop)
    keep, scale = (None, 1.0) if drop is None else (keep_of(drop[0], drop[1], drop[2], rows, H), scale_of(drop[0]))
    what = f"H={H} {xdt}->{ydt} rows={rows} layout={layout}"
    R.check_ln_fwd(ybuf[orow.to(DEV), :H], mean, rstd, x.float(), gam, bet, keep=keep, scale=scale, what=what)
    nan_outside(ybuf, H, orow.to(DEV), what)


# ---------------------------------------------------------------------------------------------------------------------
# unfused backward
# ---------------------------------------------------------------------------------------------------------------------
BWD_TRIPLES = [(BF, BF, BF), (F, BF, F), (F, F, F), (BF, F, BF)]  # (x, dy, dx) -- dres takes dx's dtype


def bwd_rows():
    S = sms()
    return [1, 9, 16 * S, 16 * S + 1, 20000]


BWD_WIDTHS_UNFUSED = [264, 768, 8, 1024, 520]
# (extra columns of every operand, remap, dropout, dres)
BWD_LAYOUTS = [(8, (0, 0, 0), None, True), (0, (37, 50, 5), DROPS[1], True), (16, (0, 0, 0), DROPS[0], False),
               (8, (11, 12, 1), DROPS[2], True)]
BWD_CASES = [(t, i, BWD_WIDTHS_UNFUSED[i % 5], BWD_LAYOUTS[i % 4]) for i, t in
             enumerate(tp for tp in BWD_TRIPLES for _ in range(5))]


def unfused_case(ops, xdt, dydt, dxdt, rows, H, extra, remap, drop, with_dres, integer, seed):
    x = R.ln_rows(rows, H, seed, xdt)
    mean, rstd = stats_of(x)
    gam, _ = params(H, seed)
    orow = remap_rows(rows, remap)
    dy = rand_gradient(rows, H, seed + 1, dydt, integer)
    dres = rand_gradient(rows, H, seed + 2, dxdt, False) if with_dres else None
    _, xv = in_nan(x.to(xdt), extra)
    _, dyv = in_nan(dy, extra, at=orow)
    dxbuf, dxv = in_nan(torch.full((rows, H), NAN, dtype=dxdt), extra, 1)
    dresv = in_nan(dres, extra)[1][:rows] if with_dres else None
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = torch.randint(-50, 51, (2, H), generator=g, device=DEV).float()
    dg, db = P[0].clone(), P[1].clone()
    ops.layernorm_bwd(dyv, xv[:rows], mean, rstd, gam, dxv[:rows], dg, db, dres=dresv, rows=rows, remap=remap,
                      dropout=drop or (0.0, 0, 0))
    return dict(x=x, mean=mean, rstd=rstd, gam=gam, dy=dy, dres=dres, dxbuf=dxbuf, dg=dg, db=db, P=P)


@pytest.mark.parametrize("dts,i,H,layout", BWD_CASES)
def test_layernorm_bwd_exact(ops, dts, i, H, layout):
    xdt, dydt, dxdt = dts
    rows = bwd_rows()[i % 5]
    extra, remap, drop, with_dres = layout
    integer = i % 2 == 0
    seed = 1000 + i
    c = unfused_case(ops, xdt, dydt, dxdt, rows, H, extra, remap, drop, with_dres, integer, seed)
    keep, scale = (None, 1.0) if drop is None else (keep_of(drop[0], drop[1], drop[2], rows, H), scale_of(drop[0]))
    what = f"{dts} rows={rows} H={H} layout={layout}"
    xd = c["x"].to(DEV)
    ref, t_g, t_b = R.ln_bwd_ref(c["dy"], xd, c["mean"], c["rstd"], c["gam"], c["dres"], keep, scale)
    E, e_g, e_b = R.ln_bwd_bounds(c["dy"], xd, c["mean"], c["rstd"], c["gam"], c["dres"], keep, scale)
    R.check_out(c["dxbuf"][:rows, :H], ref, E, f"{what}: dx")
    nan_outside(c["dxbuf"], H, torch.arange(rows, device=DEV), f"{what}: dx")
    depth = R.col_depth_unfused(rows, sms())
    want, Eg = R.col_ref_bound(t_g, e_g, c["P"][0], depth)
    R.check_f32(c["dg"], want, Eg, f"{what}: dgamma")
    if integer and (drop is None or drop[0] == 0.5):
        assert R.exact_int_sum_holds(t_b, c["P"][1])
        R.exact_check(c["db"], (c["P"][1].double() + t_b.sum(0)).float(), f"{what}: dbeta (exact)")
    else:
        want, Eb = R.col_ref_bound(t_b, e_b, c["P"][1], depth)
        R.check_f32(c["db"], want, Eb, f"{what}: dbeta")


# ---------------------------------------------------------------------------------------------------------------------
# fused backward
# ---------------------------------------------------------------------------------------------------------------------
FUSED_WIDTHS = [8, 64, 256, 264, 320, 512, 520, 768, 776, 1024]
FUSED_VARIANTS = [(True, True, 0.1), (False, False, 0.0), (True, True, 0.5), (True, False, 0.0), (False, True, 0.1),
                  (False, True, 0.0), (True, True, 0.0)]  # (dres, dbias, p)


def fused_rows(G):
    return [1, 11, 12, 13, 12 * G - 1, 12 * G, 12 * G + 1, 36 * G, 36 * G + 1, 60000]


FUSED_CASES = [(H, j, FUSED_VARIANTS[i % len(FUSED_VARIANTS)]) for i, (H, j) in enumerate(itertools.product(FUSED_WIDTHS, range(10)))]


def fused_case(ops, rows, H, with_dres, with_bias, p, seed, G):
    x = R.ln_rows(rows, H, seed, BF)
    xd = x.to(DEV)
    mean, rstd = stats_of(x)
    gam, _ = params(H, seed)
    integer = seed % 2 == 0
    dy = rand_gradient(rows, H, seed + 1, BF, integer)
    dres = rand_gradient(rows, H, seed + 2, BF, False) if with_dres else None
    dx = torch.full((rows, H), NAN, dtype=BF, device=DEV)
    dmask = torch.full((rows, H), NAN, dtype=BF, device=DEV) if p > 0 else None
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = torch.randint(-50, 51, (3, H), generator=g, device=DEV).float()
    acc = P.clone()
    site = 5 + seed % 7
    for _ in range(2):  # the accumulators add up; the ring barriers start fresh every launch
        ops.layernorm_bwd_fused(dy, xd, mean, rstd, gam, dx, acc[0], acc[1], dres=dres, dmask=dmask,
                                dbias=acc[2] if with_bias else None, dropout=(p, 2 ** 40 + seed, site))
    what = f"fused rows={rows} H={H} dres={with_dres} dbias={with_bias} p={p}"
    ref, t_g, t_b = R.ln_bwd_ref(dy, xd, mean, rstd, gam, dres)
    E, e_g, e_b = R.ln_bwd_bounds(dy, xd, mean, rstd, gam, dres)
    R.check_bf16(dx, ref, E, f"{what}: dx")
    depth = R.col_depth_fused(rows, G, launches=2)
    want, Eg = R.col_ref_bound(t_g, e_g, P[0], depth, launches=2)
    R.check_f32(acc[0], want, Eg, f"{what}: dgamma")
    if integer:
        assert R.exact_int_sum_holds(torch.cat([t_b, t_b]), P[1])
        R.exact_check(acc[1], (P[1].double() + 2 * t_b.sum(0)).float(), f"{what}: dbeta (exact)")
    else:
        want, Eb = R.col_ref_bound(t_b, e_b, P[1], depth, launches=2)
        R.check_f32(acc[1], want, Eb, f"{what}: dbeta")
    q = dx
    if p > 0:  # dmask = bf16(bf16(dx) keep scale), bit for bit from the kernel's own dx
        keep = keep_of(p, 2 ** 40 + seed, site, rows, H)
        R.exact_check(dmask, (dx.float() * keep * scale_of(p)).bfloat16(), f"{what}: dmask")
        q = dmask
    if with_bias:
        qd = q.double()
        want, Eb = R.col_ref_bound(qd, torch.zeros_like(qd), P[2], depth, launches=2)
        R.check_f32(acc[2], want, Eb, f"{what}: dbias")
    else:
        R.exact_check(acc[2], P[2], f"{what}: dbias untouched")
    return ref, E, dx


@pytest.mark.parametrize("H,j,variant", FUSED_CASES)
def test_layernorm_bwd_fused_exact(ops, H, j, variant):
    G = sms()
    rows = fused_rows(G)[j]
    fused_case(ops, rows, H, *variant, seed=H + 31 * j, G=G)


def test_layernorm_bwd_fused_exact_under_reserve(ops):
    """merlot_set_sm_reserve shrinks the fused grid to SMs - reserve blocks: ring laps and column chains move with it."""
    reserve = 20
    G = sms() - reserve
    with sm_reserve(reserve):
        fused_case(ops, 12 * G + 1, 768, True, True, 0.1, seed=4, G=G)
        fused_case(ops, 36 * G + 1, 264, False, True, 0.0, seed=6, G=G)


# ---------------------------------------------------------------------------------------------------------------------
# bias gradient
# ---------------------------------------------------------------------------------------------------------------------
BIAS_N = [8, 248, 256, 264, 768, 3072]
BIAS_ROWS = [1, 63, 64, 65, 8192, 8193, 100000]
BIAS_LAYOUTS = [(BF, 0, 0.0), (F, 8, 0.5), (BF, 16, 0.1), (F, 0, 0.1), (BF, 8, 0.5), (F, 16, 0.0)]  # (dtype, extra, p)
BIAS_CASES = [(N, rows, BIAS_LAYOUTS[i % len(BIAS_LAYOUTS)]) for i, (N, rows) in enumerate(itertools.product(BIAS_N, BIAS_ROWS))]


@pytest.mark.parametrize("N,rows,layout", BIAS_CASES)
def test_bias_grad_exact(ops, N, rows, layout):
    dt, extra, p = layout
    seed, site = N + rows, 9
    drop = (p, seed, site)
    keep = keep_of(p, seed, site, rows, N).double() if p > 0 else None
    scale = scale_of(p) if p > 0 else 1.0
    depth = R.col_depth_colsum(rows)
    g = torch.Generator(device=DEV).manual_seed(seed)
    what = f"bias_grad N={N} rows={rows} {dt} ld={N + extra} p={p}"
    for integer in (True, False):
        dy = rand_gradient(rows, N, seed + integer, dt, integer)
        _, dyv = in_nan(dy, extra)
        P = torch.randint(-1000, 1001, (N,), generator=g, device=DEV).float() if integer else \
            torch.randn(N, generator=g, device=DEV)
        out = P.clone()
        ops.bias_grad(dyv, out, rows=rows, N=N, dropout=drop)
        dv = dy.double() if keep is None else dy.double() * keep * float(np.float32(scale))
        if integer and p in (0.0, 0.5):
            assert R.exact_int_sum_holds(dv, P)
            R.exact_check(out, (P.double() + dv.sum(0)).float(), f"{what}: integer (exact)")
        else:
            err = R.U * dv.abs() if scale != 1.0 else torch.zeros_like(dv)
            want, E = R.col_ref_bound(dv, err, P, depth)
            R.check_f32(out, want, E, f"{what}: {'integer' if integer else 'random'}")


# ---------------------------------------------------------------------------------------------------------------------
# wrong references must miss
# ---------------------------------------------------------------------------------------------------------------------
def test_wrong_references_miss_the_bars(ops):
    """The GPU's outputs against references that are wrong on purpose: each must fail, so the bounds discriminate on real
    output -- unbiased variance (fp32 y and the statistics), eps x 0.1 (rows with variance near eps), the dropout mask of
    site + 1 (unfused backward), dx rows shifted by one (fused backward)."""
    H, rows = 768, 64
    x = R.ln_rows(rows, H, 3, F)
    gam, bet = params(H, 3)
    ybuf, orow, mean, rstd = run_fwd(ops, x, gam, bet, F, F, 0, (0, 0, 0), None)
    y = ybuf[:rows, :H]
    R.check_ln_fwd(y, mean, rstd, x, gam, bet)
    with pytest.raises(AssertionError, match="elements differ"):
        R.check_ln_fwd(y, None, None, x, gam, bet, unbiased_ref=True)
    with pytest.raises(AssertionError, match="rstd: .* elements differ"):
        R.check_ln_fwd(y, mean, rstd, x, gam, bet, unbiased_ref=True)
    xe = R.ln_rows(rows, H, 4, BF, classes=("near_eps",))
    ybuf, _, mean, rstd = run_fwd(ops, xe, gam, bet, BF, F, 0, (0, 0, 0), None)
    R.check_ln_fwd(ybuf[:rows, :H], mean, rstd, xe.float(), gam, bet)
    with pytest.raises(AssertionError, match="rstd: 64 of 64 elements differ"):
        R.check_ln_fwd(ybuf[:rows, :H], mean, rstd, xe.float(), gam, bet, ref_eps=R.EPS * 0.1)

    p, seed, site = DROPS[0]
    c = unfused_case(ops, BF, BF, BF, 300, 264, 8, (0, 0, 0), (p, seed, site), False, False, 77)
    xd = c["x"].to(DEV)
    for s, ok in ((site, True), (site + 1, False)):
        keep = keep_of(p, seed, s, 300, 264)
        ref, *_ = R.ln_bwd_ref(c["dy"], xd, c["mean"], c["rstd"], c["gam"], None, keep, scale_of(p))
        E, *_ = R.ln_bwd_bounds(c["dy"], xd, c["mean"], c["rstd"], c["gam"], None, keep, scale_of(p))
        if ok:
            R.check_bf16(c["dxbuf"][:300, :264], ref, E, "dx")
        else:
            with pytest.raises(AssertionError, match="elements differ"):
                R.check_bf16(c["dxbuf"][:300, :264], ref, E, "dx, mask of site + 1")

    ref, E, dx = fused_case(ops, 12 * sms() + 1, 256, True, False, 0.0, seed=8, G=sms())
    with pytest.raises(AssertionError, match="elements differ"):
        R.check_bf16(dx, ref.roll(1, 0), E.roll(1, 0), "dx, rows shifted by one")
