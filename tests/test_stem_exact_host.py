"""The checks of tests/stem_exact_oracle.py hold and can fail, on the CPU.  (1) The exact-input construction: fp32 sums of
x and x^2 in shuffled, blocked and reversed orders equal the float64 sums at every group size the GPU tests use.  (2) An fp32
emulation of each K13 kernel's arithmetic, with the launch's own reduction chains, meets every per-element bound.  (3) Each
doctored output below fails the check aimed at it; where noted, the relative-Frobenius bars of test_gpu_stem.py (6e-3
GroupNorm forward, 4e-3 pool / col2im / weight standardisation, OP_BAR = 2e-2 backward) accept it."""
import math

import numpy as np
import pytest
import torch

from tests import stem_exact_oracle as S
from tests import test_gpu_stem_exact as G

F32 = torch.float32
GN_FWD_BAR, POOL_BAR, WS_BAR, OP_BAR = 6e-3, 4e-3, 4e-3, 2e-2


def rel(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm())


def f32(v):
    return torch.tensor(v, dtype=F32)


# ---------------------------------------------------------------------------------------------------------------------
# fp32 emulations of the kernels, with the launch's reduction structure
# ---------------------------------------------------------------------------------------------------------------------
def chains(t, N, HW, C, cg=None, skip_block=None):
    """Sums of t [N, HW, C] (float32) as gn_stats / gn_bwd_reduce form them: each thread chains its rows (r0 + rl + k lanes),
    the lanes meet in shared memory, the blocks in global memory.  cg: per group of cg channels -> [N, C // cg];
    else per channel over all samples -> [C].  skip_block drops that block's partial (a doctored reduction)."""
    geo = S.gn_geometry(HW, C)
    lanes, rpb, nb, rpt = geo["lanes"], geo["rows_per_block"], geo["blocks"], geo["rows_per_thread"]
    b, k, l = torch.meshgrid(torch.arange(nb), torch.arange(rpt), torch.arange(lanes), indexing="ij")
    local = k * lanes + l
    row = b * rpb + local
    valid = (local < rpb) & (row < HW)
    T = t[:, row.clamp(max=HW - 1)] * valid[None, ..., None]           # [N, blocks, rpt, lanes, C]
    acc = torch.zeros(N, nb, lanes, C, dtype=F32)
    for i in range(rpt):
        acc = acc + T[:, :, i]
    if cg is not None:
        acc = acc.reshape(N, nb, lanes, C // cg, cg).permute(0, 1, 3, 2, 4).reshape(N, nb, C // cg, lanes * cg)
        blk = torch.zeros(N, nb, C // cg, dtype=F32)
        for i in range(lanes * cg):
            blk = blk + acc[..., i]
        out = torch.zeros(N, C // cg, dtype=F32)
        for i in range(nb):
            if i != skip_block:
                out = out + blk[:, i]
        return out
    blk = torch.zeros(N, nb, C, dtype=F32)
    for i in range(lanes):
        blk = blk + acc[:, :, i]
    out = torch.zeros(C, dtype=F32)
    for n in range(N):
        for i in range(nb):
            if (n, i) != skip_block:
                out = out + blk[n, i]
    return out


def emu_gn_stats(x, N, HW, C, groups=32, skip=None):
    x = x.float().reshape(N, HW, C)
    cg = C // groups
    return torch.stack((chains(x, N, HW, C, cg, skip), chains(x * x, N, HW, C, cg, skip)), -1).reshape(-1)


def emu_moments(stats, N, HW, C, groups, eps=S.GN_EPS):
    cg = C // groups
    inv = f32(1.0) / (f32(HW) * f32(cg))
    st = stats.float().reshape(N, groups, 2)
    mean = st[..., 0] * inv
    var = st[..., 1] * inv - mean * mean
    rstd = torch.rsqrt(var + f32(eps))
    ch = lambda v: v.repeat_interleave(cg, 1).reshape(N, 1, C)
    return ch(mean), ch(rstd), inv


def emu_gn_apply(x, stats, gamma, beta, N, HW, C, groups=32, relu=True, shortcut=None, skip_round=False, moments=None):
    mean, rstd, _ = moments or emu_moments(stats, N, HW, C, groups)
    o = (x.float().reshape(N, HW, C) - mean) * rstd * gamma.float() + beta.float()
    if shortcut is not None:
        o = (o if skip_round else o.bfloat16().float()) + shortcut.float().reshape(N, HW, C)
    if relu:
        o = o.clamp(min=0)
    return o.bfloat16().reshape(N * HW, C)


def emu_gn_bwd(dy, x, y, stats, gamma, dgamma0, dbeta0, N, HW, C, groups=32, relu=True, skip_block=None, mask_dsc=True):
    cg = C // groups
    mean, rstd, inv = emu_moments(stats, N, HW, C, groups)
    d = dy.float().reshape(N, HW, C)
    g = torch.where(y.float().reshape(N, HW, C) > 0, d, torch.zeros(())) if relu else d
    xh = (x.float().reshape(N, HW, C) - mean) * rstd
    gg = g * gamma.float()
    red = torch.stack((chains(gg, N, HW, C, cg), chains(gg * xh, N, HW, C, cg)), -1)
    dgamma = dgamma0.float() + chains(g * xh, N, HW, C, skip_block=skip_block)
    dbeta = dbeta0.float() + chains(g, N, HW, C)
    ch = lambda v: v.repeat_interleave(cg, 1).reshape(N, 1, C)
    dx = rstd * (gg - ch(red[..., 0] * inv) - xh * ch(red[..., 1] * inv))
    return dict(dx=dx.bfloat16(), dshortcut=(g if mask_dsc else d).bfloat16(), dgamma=dgamma, dbeta=dbeta, red=red.reshape(-1))


def emu_ws(w, eps=S.WS_EPS):
    """ws_channels in fp32: warp chains over rows warp + 32 k, the 32 warp sums in order, one division per moment."""
    rows, cout = w.shape
    w = w.float()

    def block_sum(t):
        pad = torch.zeros(-(-rows // 32) * 32, cout, dtype=F32)
        pad[:rows] = t
        part = torch.zeros(32, cout, dtype=F32)
        for k in range(pad.shape[0] // 32):
            part = part + pad[32 * k:32 * k + 32]
        tot = torch.zeros(cout, dtype=F32)
        for i in range(32):
            tot = tot + part[i]
        return tot / f32(rows)

    mean = block_sum(w)
    var = block_sum((w - mean) ** 2)
    rstd = torch.rsqrt(var + f32(eps))
    return mean, rstd, block_sum


def emu_ws_fwd(w, eps=S.WS_EPS):
    mean, rstd, _ = emu_ws(w, eps)
    return ((w.float() - mean) * rstd).bfloat16()


def emu_ws_bwd(dws, w, dw0):
    mean, rstd, block_sum = emu_ws(w)
    wh = (w.float() - mean) * rstd
    m1, m2 = block_sum(dws.float()), block_sum(dws.float() * wh)
    return dw0.float() + rstd * (dws.float() - m1 - wh * m2)


def emu_pool(x, N, h, w, C, ragged_by_4=False):
    ho, wo = (h + 1) // 2, (w + 1) // 2
    xp = torch.zeros(N, 2 * ho, 2 * wo, C, dtype=F32)
    xp[:, :h, :w] = x.float().reshape(N, h, w, C)
    s = xp[:, 0::2, 0::2] + xp[:, 0::2, 1::2] + xp[:, 1::2, 0::2] + xp[:, 1::2, 1::2]
    cnt = torch.full((ho, wo), 4.0) if ragged_by_4 else S.pool_counts(h, w).float()
    return (s * (1.0 / cnt)[None, :, :, None]).bfloat16().reshape(-1, C)


def emu_pool_bwd(dy, N, h, w, C, ragged_by_4=False):
    ho, wo = (h + 1) // 2, (w + 1) // 2
    cnt = torch.full((ho, wo), 4.0) if ragged_by_4 else S.pool_counts(h, w).float()
    d = dy.float().reshape(N, ho, wo, C) * (1.0 / cnt)[None, :, :, None]
    return d.repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :h, :w].bfloat16().reshape(-1, C)


def emu_col2im(dcol, N, h, w, C, stride, drop_last_row_ky2=False):
    ho, wo = S.conv_out(h, w, stride)
    d4 = dcol.float().reshape(N, ho, wo, 9, C)
    out = torch.zeros(N, h + 2, w + 2, C, dtype=F32)
    for t in range(9):
        ky, kx = t // 3, t % 3
        v = d4[:, :, :, t].clone()
        if drop_last_row_ky2 and ky == 2:
            v[:, (h - 1 + 1 - 2) // stride] = 0  # the output row whose ky = 2 tap lands on input row h - 1
        out[:, ky:ky + (ho - 1) * stride + 1:stride, kx:kx + (wo - 1) * stride + 1:stride] += v
    return out[:, 1:h + 1, 1:w + 1].bfloat16().reshape(-1, C)


# ---------------------------------------------------------------------------------------------------------------------
# (1) the exact-input construction
# ---------------------------------------------------------------------------------------------------------------------
def _orders(k, rng):
    """fp32 sequential sums of k (float32 array) in four orders: as given, reversed, shuffled, blocked (2048-row blocks
    summed first, then the block sums)."""
    seq = lambda a: np.cumsum(a, dtype=np.float32)[-1]
    blocks = np.array([seq(k[i:i + 2048]) for i in range(0, len(k), 2048)], np.float32)
    return [seq(k), seq(k[::-1]), seq(rng.permutation(k)), seq(blocks)]


@pytest.mark.parametrize("n", sorted({hw * cg for hw, cg in G.GROUP_SIZES}))
def test_fp32_sums_are_exact_in_any_order(n):
    """For every (HW x channels per group) the GPU tests use, with the extreme values +-max_k(n) present."""
    kmax = S.max_k(n)
    rng = np.random.default_rng(n)
    k = rng.integers(-kmax, kmax + 1, n).astype(np.float32)
    k[:2] = (kmax, -kmax)
    delta = 2.0 ** -5
    x = (k * delta).astype(np.float32)
    for v, want in ((x, float(np.sum(x.astype(np.float64)))), (x * x, float(np.sum(x.astype(np.float64) ** 2)))):
        assert all(float(s) == want for s in _orders(v, rng)), n
    all_max = np.full(n, kmax * delta, np.float32)  # the worst case reaches n kmax^2 < 2^24 delta^2
    assert float(np.cumsum(all_max * all_max, dtype=np.float32)[-1]) == n * (kmax * delta) ** 2
    assert not S.exact_sums_hold(n, int(math.isqrt(2 ** 24 // n)) + 1)


# ---------------------------------------------------------------------------------------------------------------------
# (2) fp32 emulations meet the bounds; (3) doctored outputs fail them
# ---------------------------------------------------------------------------------------------------------------------
def _gn_problem(N, HW, C, seed, groups=32, center=0):
    n = HW * C // groups
    kmax = S.max_k(n * 4) if center else S.max_k(n)
    x = S.dyadic((N * HW, C), kmax, 2.0 ** -4, seed, center=center)
    g = torch.Generator().manual_seed(seed + 1)
    gamma = (torch.randn(C, generator=g) * 0.3 + 1.0).float()
    beta = (torch.randn(C, generator=g) * 0.2).float()
    return x, gamma, beta


@pytest.mark.parametrize("N,HW,C,groups", [(2, 2049, 64, 32), (1, 3 * 672 + 1, 96, 32), (2, 300, 256, 8), (1, 33, 2048, 32)])
def test_emulated_group_norm_forward_meets_the_bounds(N, HW, C, groups):
    x, gamma, beta = _gn_problem(N, HW, C, HW + C, groups)
    S.assert_exact_grid(x, HW * C // groups, 2.0 ** -4)
    stats = emu_gn_stats(x, N, HW, C, groups)
    S.check_gn_stats(stats, x, N, HW, C, groups)
    o, _ = S.gn_fwd_ref(x, stats, gamma, beta, N, HW, C, groups)
    sc = S.rounding_sensitive_shortcut(o, 5)
    for relu, short in ((True, None), (False, None), (True, sc)):
        y = emu_gn_apply(x, stats, gamma, beta, N, HW, C, groups, relu, short)
        S.check_gn_fwd(y, x, stats, gamma, beta, N, HW, C, groups, relu=relu, shortcut=short)


def test_emulated_group_norm_statistics_edges():
    """A constant group (variance 0 < eps: out = beta) and a group whose mean is 4 std (one-pass cancellation)."""
    N, HW, C = 1, 1500, 64
    x, gamma, beta = _gn_problem(N, HW, C, 3)
    x = x.reshape(HW, 32, 2).clone()
    x[:, 3] = 0.75
    x[:, 4] = S.dyadic((HW, 2), 2, 2.0 ** -4, 9, center=8)
    x = x.reshape(N * HW, C)
    S.assert_exact_grid(x, HW * 2, 2.0 ** -4)
    stats = emu_gn_stats(x, N, HW, C)
    S.check_gn_stats(stats, x, N, HW, C)
    y = emu_gn_apply(x, stats, gamma, beta, N, HW, C, relu=False)
    S.check_gn_fwd(y, x, stats, gamma, beta, N, HW, C, relu=False)
    assert torch.equal(y.reshape(HW, 32, 2)[:, 3].float(), beta.reshape(32, 2)[3].expand(HW, 2).bfloat16().float())


def test_emulated_group_norm_backward_meets_the_bounds():
    for N, HW, C, relu, short in ((2, 2049, 64, True, True), (1, 700, 96, False, False)):
        x, gamma, beta = _gn_problem(N, HW, C, 7)
        gamma = 2.0 ** torch.randint(-1, 2, (C,), generator=torch.Generator().manual_seed(1)).float()
        dy = S.dyadic((N * HW, C), 4, 2.0 ** -6, 8)
        stats = emu_gn_stats(x, N, HW, C)
        y = emu_gn_apply(x, stats, gamma, beta, N, HW, C, relu=relu)
        dg0, db0 = torch.full((C,), 0.25), torch.full((C,), -0.5)
        out = emu_gn_bwd(dy, x, y, stats, gamma, dg0, db0, N, HW, C, relu=relu)
        if not short:
            out["dshortcut"] = None
        S.check_gn_bwd(out, dy, x, y, stats, gamma, N, HW, C, relu=relu, exact=True, dgamma0=dg0, dbeta0=db0)


def test_emulated_pool_col2im_ws_meet_the_bounds():
    for N, h, w, C in ((2, 9, 7, 32), (1, 12, 22, 64)):
        x = S.dyadic((N * h * w, C), 16, 2.0 ** -4, h)
        S.exact_check(emu_pool(x, N, h, w, C), S.bf16_rn(S.avgpool_ref(x, N, h, w, C)[0]), "pool")
        dy = S.dyadic((N * ((h + 1) // 2) * ((w + 1) // 2), C), 16, 2.0 ** -4, w)
        S.exact_check(emu_pool_bwd(dy, N, h, w, C), S.avgpool_bwd_ref(dy, N, h, w, C), "pool bwd")
    for N, h, w, C, stride in ((2, 9, 7, 32, 1), (1, 10, 14, 32, 2), (1, 9, 11, 64, 2)):
        ho, wo = S.conv_out(h, w, stride)
        dcol = S.dyadic((N * ho * wo, 9 * C), 16, 2.0 ** -4, h + stride)
        S.exact_check(emu_col2im(dcol, N, h, w, C, stride), S.bf16_rn(S.col2im_ref(dcol, N, h, w, C, stride)[0]), "col2im")
    g = torch.Generator().manual_seed(4)
    for rows, cout in ((27, 32), (576, 64), (2304, 256)):
        w2 = torch.randn(rows, cout, generator=g) * 0.2 + 0.05
        ref, E = S.ws_ref(w2)
        S.interval_check(emu_ws_fwd(w2), ref, E, "ws")
        dws, dw0 = torch.randn(rows, cout, generator=g), torch.full((rows, cout), 0.5)
        ref, E = S.ws_bwd_ref(dws, w2, dw0)
        S.bound_check(emu_ws_bwd(dws, w2, dw0), ref, E, "ws bwd")


def test_shortcut_without_the_intermediate_rounding_is_caught():
    N, HW, C = 2, 600, 64
    x, gamma, beta = _gn_problem(N, HW, C, 11)
    stats = emu_gn_stats(x, N, HW, C)
    o, _ = S.gn_fwd_ref(x, stats, gamma, beta, N, HW, C)
    sc = S.rounding_sensitive_shortcut(o, 2)
    bad = emu_gn_apply(x, stats, gamma, beta, N, HW, C, shortcut=sc, skip_round=True)
    with pytest.raises(AssertionError, match="outside the bound"):
        S.check_gn_fwd(bad, x, stats, gamma, beta, N, HW, C, shortcut=sc)
    want = (S.bf16_rn(o).float() + sc.float().reshape(N, HW, C)).clamp(min=0)
    assert rel(bad, want) < GN_FWD_BAR


def test_slab_missing_from_one_groups_statistics_is_caught():
    N, HW, C = 2, 3 * 2048 + 1, 32
    x, gamma, beta = _gn_problem(N, HW, C, 12)
    good = emu_gn_stats(x, N, HW, C)
    slab = emu_gn_stats(x, N, HW, C, skip=1).reshape(N, 32, 2)
    stats = good.clone().reshape(N, 32, 2)
    stats[1, 5] = slab[1, 5]  # sample 1, group 5 lost the rows of its second block
    stats = stats.reshape(-1)
    with pytest.raises(AssertionError, match=r"gn stats: 2 of 128 elements differ; first at \(1, 5, 0\)"):
        S.check_gn_stats(stats, x, N, HW, C)


def test_neighbour_groups_moments_at_a_group_boundary_are_caught():
    """C = 96: 3 channels per group, so a 16-byte chunk of 8 channels straddles three groups."""
    N, HW, C = 1, 700, 96
    x, gamma, beta = _gn_problem(N, HW, C, 13)
    stats = emu_gn_stats(x, N, HW, C)
    mean, rstd, inv = emu_moments(stats, N, HW, C, 32)
    mean, rstd = mean.clone(), rstd.clone()
    mean[..., 9], rstd[..., 9] = mean[..., 8], rstd[..., 8]  # channel 9 opens group 3; it uses group 2's moments
    bad = emu_gn_apply(x, stats, gamma, beta, N, HW, C, moments=(mean, rstd, inv))
    with pytest.raises(AssertionError, match=r"outside the bound; first at \(0, \d+, 9\)"):
        S.check_gn_fwd(bad, x, stats, gamma, beta, N, HW, C)
    assert rel(bad, torch.relu(S.gn_fwd_ref(x, stats, gamma, beta, N, HW, C)[0])) < GN_FWD_BAR


@pytest.fixture(scope="module")
def bwd_problem():
    N, HW, C = 2, 4 * 1024 + 1, 64
    x, gamma, beta = _gn_problem(N, HW, C, 14)
    gamma = 2.0 ** torch.randint(-1, 2, (C,), generator=torch.Generator().manual_seed(2)).float()
    dy = S.dyadic((N * HW, C), 4, 2.0 ** -6, 15)
    stats = emu_gn_stats(x, N, HW, C)
    y = emu_gn_apply(x, stats, gamma, beta, N, HW, C)
    dg0, db0 = torch.full((C,), 0.25), torch.full((C,), -0.5)
    return N, HW, C, x, gamma, dy, stats, y, dg0, db0


def test_dshortcut_without_the_relu_mask_is_caught(bwd_problem):
    N, HW, C, x, gamma, dy, stats, y, dg0, db0 = bwd_problem
    out = emu_gn_bwd(dy, x, y, stats, gamma, dg0, db0, N, HW, C, mask_dsc=False)
    with pytest.raises(AssertionError, match="dshortcut"):
        S.check_gn_bwd(out, dy, x, y, stats, gamma, N, HW, C, exact=True, dgamma0=dg0, dbeta0=db0)


def test_block_partial_missing_from_dgamma_is_caught(bwd_problem):
    N, HW, C, x, gamma, dy, stats, y, dg0, db0 = bwd_problem
    out = emu_gn_bwd(dy, x, y, stats, gamma, dg0, db0, N, HW, C, skip_block=(1, 2))
    with pytest.raises(AssertionError, match="dgamma"):
        S.check_gn_bwd(out, dy, x, y, stats, gamma, N, HW, C, exact=True, dgamma0=dg0, dbeta0=db0)


def test_ragged_pool_cells_divided_by_4_are_caught():
    N, h, w, C = 2, 9, 7, 32
    x = S.dyadic((N * h * w, C), 16, 2.0 ** -4, 1)
    with pytest.raises(AssertionError, match="pool: .* differ"):
        S.exact_check(emu_pool(x, N, h, w, C, ragged_by_4=True), S.bf16_rn(S.avgpool_ref(x, N, h, w, C)[0]), "pool")
    dy = S.dyadic((N * 5 * 4, C), 16, 2.0 ** -4, 2)
    with pytest.raises(AssertionError, match="pool bwd: .* differ"):
        S.exact_check(emu_pool_bwd(dy, N, h, w, C, ragged_by_4=True), S.avgpool_bwd_ref(dy, N, h, w, C), "pool bwd")


def test_col2im_missing_the_last_rows_ky2_tap_is_caught():
    N, h, w, C, stride = 2, 96, 176, 32, 2
    ho, wo = S.conv_out(h, w, stride)
    dcol = S.dyadic((N * ho * wo, 9 * C), 16, 2.0 ** -4, 3)
    ref = S.col2im_ref(dcol, N, h, w, C, stride)[0]
    bad = emu_col2im(dcol, N, h, w, C, stride, drop_last_row_ky2=True)
    with pytest.raises(AssertionError, match=r"col2im: .* differ; first at \(16720, "):  # row 95 of map 0
        S.exact_check(bad, S.bf16_rn(ref), "col2im")
    assert rel(bad, ref) < 0.15  # the last input row of each map has no other tap: 1 of 96 rows zeroed


def test_sub_half_on_the_padding_ring_is_caught():
    N, h, w, C, stride = 1, 9, 7, 3, 2
    x = torch.rand(N * h * w, C, generator=torch.Generator().manual_seed(4)).bfloat16()
    ho, wo = S.conv_out(h, w, stride)
    good = S.im2col_ref(x, N, h, w, C, stride, 32, sub_half=True)
    bad = good.float()
    xp = torch.full((N, h + 2, w + 2, C), -0.5)
    xp[:, 1:h + 1, 1:w + 1] = (x.float().reshape(N, h, w, C) - 0.5).bfloat16().float()
    taps = [xp[:, ky:ky + (ho - 1) * stride + 1:stride, kx:kx + (wo - 1) * stride + 1:stride] for ky in range(3) for kx in range(3)]
    bad[:, :27] = torch.stack(taps, 3).reshape(-1, 27)
    with pytest.raises(AssertionError, match=r"im2col: .* differ; first at \(0, 0\)"):
        S.exact_check(bad.bfloat16(), good, "im2col")


def test_wgrad_split_added_twice_is_caught():
    M, kp, cout, splits = 4096, 32, 32, 7
    a = S.dyadic((M, kp), 1, 1.0, 1).float()
    dy = S.dyadic((M, cout), 1, 1.0, 2).float()
    init = torch.randint(-8, 9, (kp, cout), generator=torch.Generator().manual_seed(3)).float()
    want = S.wgrad_exact(a, dy, init)
    parts = [a[i:i + M // splits + 1].t() @ dy[i:i + M // splits + 1] for i in range(0, M, M // splits + 1)]
    got = init.clone()
    for p in parts + parts[2:3]:
        got += p
    with pytest.raises(AssertionError, match="wgrad: .* differ"):
        S.exact_check(got, want, "wgrad")


def test_weight_standardisation_with_the_wrong_eps_or_moments_is_caught():
    rows, cout = 576, 64
    w2 = torch.randn(rows, cout, generator=torch.Generator().manual_seed(5)) * 0.2 + 0.05
    ref, E = S.ws_ref(w2)
    bad_eps = emu_ws_fwd(w2, eps=1e-4)
    with pytest.raises(AssertionError, match="ws: .* outside the bound"):
        S.interval_check(bad_eps, ref, E, "ws")
    assert rel(bad_eps, ref) < WS_BAR
    per_tap = torch.cat([emu_ws_fwd(w2[i * 64:(i + 1) * 64]) for i in range(9)])  # moments over cin only
    with pytest.raises(AssertionError, match="ws: .* outside the bound"):
        S.interval_check(per_tap, ref, E, "ws")
