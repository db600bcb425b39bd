"""The hybrid stem's K13 kernels (merlot_b200/csrc/stem.cu) element by element against float64 (tests/stem_exact_oracle.py),
at the shipped map sizes and at the edges of their launch grids (pytest -m gpu).

Dyadic inputs make every reduction exact, so GroupNorm statistics, dbeta, the S1 half of `red`, im2col, col2im, avg-pool
(forward and backward) and the conv wgrads through K1 are compared bit for bit; GroupNorm outputs, dgamma, S2, dx and the
weight standardisation meet per-element bounds derived from the kernels' own arithmetic and reduction chains.

GroupNorm shapes (N x HW x C, groups 32 unless noted): channels per group, rows_per_block = (256 / (C/8)) * 32 (capped at
HW), blocks per sample.
    shipped, 192x352 input:  16896 x 32 (1, 2048, 9)   16896 x 64 (2, 1024, 17)   4224 x 256 (8, 256, 17)
                             1056 x 512 (16, 128, 9)   264 x 1024 (32, 64, 5)
    shipped, 384x704 input:  67584 x 32 (1, 2048, 33)  67584 x 64 (2, 1024, 66)   16896 x 256 (8, 256, 66)
                             4224 x 512 (16, 128, 33)  1056 x 1024 (32, 64, 17)
    shipped, 384x384 input:  36864 x 32 (1, 2048, 18)  36864 x 64 (2, 1024, 36)   9216 x 256 (8, 256, 36)
                             2304 x 512 (16, 128, 18)  576 x 1024 (32, 64, 9)
    grid edges (C = 256):    1024 (8, 256, 4)   1025 (8, 256, 5)   1 (8, 1, 1)   N = 200 x 257 (8, 256, 2): gridDim.y 200
    group layouts:           4224 x 128 (4, 512, 9)   2017 x 96 (3, 672, 4: 21 lanes, 4 idle threads, chunks straddle
                             groups)   65 x 2048 (64, 32, 3: the API's largest C)   4224 x 256 groups 8 (32, 256, 17)
                             4224 x 64 groups 64 (1, 1024, 5)
Conv wgrads (K = N * ho * wo): stem1 at the 192x352 map of the 384x704 input, N = 16: K = 1 081 344 > 2^20, kp 288, cout
32; stem0 (27 rows padded to 32) on a 96x176 output; a 3x3 128 -> 128 and a 1x1 1024 -> 256 with K = 16896; each with the
automatic split, 1 and 7, and all but stem1 with the largest split count (one 64-wide k-block per split).
In situ: lite_resnet50 [3, 4, 9] forward and backward at 192x352, N = 2 (maps 96x176, 48x88, 24x44, 12x22)."""
import functools

import pytest
import torch

from merlot_b200.stem import stem_ops
from tests import gemm_exact_oracle as X
from tests import stem_exact_oracle as S

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
DELTA = 2.0 ** -4

SHIPPED = [(2, 16896, 32), (2, 16896, 64), (2, 4224, 256), (2, 1056, 512), (2, 264, 1024),
           (2, 67584, 32), (2, 67584, 64), (2, 16896, 256), (2, 4224, 512), (2, 1056, 1024),
           (2, 36864, 32), (2, 36864, 64), (2, 9216, 256), (2, 2304, 512), (2, 576, 1024)]
EDGES = [(3, 1024, 256), (3, 1025, 256), (5, 1, 256), (200, 257, 256)]
LAYOUTS = [(2, 4224, 128), (2, 2017, 96), (2, 65, 2048)]
GN_SHAPES = [(N, HW, C, 32) for N, HW, C in SHIPPED + EDGES + LAYOUTS] + [(2, 4224, 256, 8), (2, 4224, 64, 64)]
GROUP_SIZES = [(HW, C // g) for _, HW, C, g in GN_SHAPES]  # (rows, channels) of one group: the host test checks exactness


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def _params(C, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(C, generator=g) * 0.3 + 1.0).to(DEV), (torch.randn(C, generator=g) * 0.2).to(DEV)


def _gn_input(N, HW, C, groups, seed):
    x = S.dyadic((N * HW, C), S.max_k(HW * C // groups), DELTA, seed, device=DEV)
    S.assert_exact_grid(x, HW * C // groups, DELTA)
    return x


def _gn_fwd(ops, x, gamma, beta, N, HW, C, groups, relu, shortcut=None):
    y, stats = nan(N * HW, C, dtype=torch.bfloat16), nan(N * groups * 2)
    ops.group_norm_fwd(x, gamma, beta, y, stats, N, HW, C, groups, S.GN_EPS, relu, shortcut)
    return y, stats


@pytest.mark.parametrize("N,HW,C,groups", GN_SHAPES)
def test_group_norm_forward_exact(ops, N, HW, C, groups):
    """Statistics bit for bit; outputs within the midpoint rule with ReLU, without, and relu(bf16(gn) + shortcut)."""
    x = _gn_input(N, HW, C, groups, HW + C + groups)
    gamma, beta = _params(C, C)
    y, stats = _gn_fwd(ops, x, gamma, beta, N, HW, C, groups, False)
    S.check_gn_stats(stats, x, N, HW, C, groups)
    mids = {"plain": S.check_gn_fwd(y, x, stats, gamma, beta, N, HW, C, groups, relu=False)}
    y, _ = _gn_fwd(ops, x, gamma, beta, N, HW, C, groups, True)
    mids["relu"] = S.check_gn_fwd(y, x, stats, gamma, beta, N, HW, C, groups, relu=True)
    o, _ = S.gn_fwd_ref(x, stats, gamma, beta, N, HW, C, groups)
    sc = S.rounding_sensitive_shortcut(o, HW)
    y, _ = _gn_fwd(ops, x, gamma, beta, N, HW, C, groups, True, sc)
    mids["shortcut"] = S.check_gn_fwd(y, x, stats, gamma, beta, N, HW, C, groups, relu=True, shortcut=sc)
    unrounded = (o + sc.double().reshape(o.shape)).clamp(min=0)
    assert int((S.bf16_rn(unrounded) != y.double().reshape(o.shape)).sum()) > y.numel() // 10  # the rounding matters here
    assert max(mids.values()) <= y.numel() // 100, mids


def test_group_norm_statistics_edges(ops):
    """Constant groups (variance 0 < eps, as a blank or zero-padded frame gives) come out as beta; a group with mean 4 std
    meets the bound of the one-pass formula, its fp32 cancellation included.  (The kernel computes var = E[x^2] - mean^2
    like the reference; for a large constant group that can round below 0, and var + eps stays positive while it is above
    -eps.)"""
    N, HW, C = 2, 16896, 64
    x = _gn_input(N, HW, C, 32, 1).reshape(N, HW, 32, 2).clone()
    x[0, :, 3] = 0.75
    x[1, :, 7] = -1.0
    x[1, :, 8] = 0.0
    x[0, :, 9] = S.dyadic((HW, 2), 2, DELTA, 9, center=8, device=DEV).reshape(HW, 2)  # mean 0.5, std ~0.09
    x = x.reshape(N * HW, C)
    S.assert_exact_grid(x, HW * 2, DELTA)
    gamma, beta = _params(C, 3)
    y, stats = _gn_fwd(ops, x, gamma, beta, N, HW, C, 32, False)
    S.check_gn_stats(stats, x, N, HW, C)
    S.check_gn_fwd(y, x, stats, gamma, beta, N, HW, C, relu=False)
    yb, b = y.reshape(N, HW, 32, 2).double(), S.bf16_rn(beta.double()).reshape(32, 2)
    for n, grp in ((0, 3), (1, 7), (1, 8)):
        assert torch.equal(yb[n, :, grp], b[grp].expand(HW, 2)), (n, grp)


BWD_SHAPES = [(2, 16896, 32, 32, True, False), (2, 67584, 64, 32, True, True), (2, 4224, 256, 32, False, False),
              (2, 1056, 1024, 32, True, True), (3, 1025, 256, 32, True, True), (2, 2017, 96, 32, True, False),
              (2, 65, 2048, 32, True, True), (2, 4224, 256, 8, True, True), (200, 257, 256, 32, False, True)]


@pytest.mark.parametrize("N,HW,C,groups,relu,short", BWD_SHAPES)
def test_group_norm_backward_exact(ops, N, HW, C, groups, relu, short):
    """dbeta, S1 and dshortcut bit for bit (dyadic dy, gamma powers of two), dgamma / S2 / dx within their chain bounds;
    dgamma and dbeta accumulate onto non-zero buffers; red, dx and dshortcut start as NaN."""
    x = _gn_input(N, HW, C, groups, HW + C)
    g = torch.Generator().manual_seed(C)
    gamma = (2.0 ** torch.randint(-1, 2, (C,), generator=g)).float().to(DEV)
    beta = (torch.randn(C, generator=g) * 0.2).to(DEV)
    sc = S.dyadic((N * HW, C), 16, DELTA, 5, device=DEV) if short else None
    y, stats = _gn_fwd(ops, x, gamma, beta, N, HW, C, groups, relu, sc)
    dy = S.dyadic((N * HW, C), 4, 2.0 ** -6, HW, device=DEV)
    assert N * HW * 4 < 2 ** 24 and HW * (C // groups) * 4 * 2 < 2 ** 24  # dbeta and S1 sums are exact
    dx, dsc, red = nan(N * HW, C, dtype=torch.bfloat16), nan(N * HW, C, dtype=torch.bfloat16) if short else None, nan(N * groups * 2)
    dg0, db0 = torch.full((C,), 0.25, device=DEV), torch.full((C,), -0.5, device=DEV)
    dg, db = dg0.clone(), db0.clone()
    ops.group_norm_bwd(dy, x, y if relu else None, stats, gamma, dx, dsc, dg, db, red, N, HW, C, groups, S.GN_EPS, relu)
    out = dict(dx=dx, dshortcut=dsc, dgamma=dg, dbeta=db, red=red)
    mids = S.check_gn_bwd(out, dy, x, y, stats, gamma, N, HW, C, groups, relu=relu, exact=True, dgamma0=dg0, dbeta0=db0)
    assert mids <= dx.numel() // 100, mids


IM2COL = [  # N, h, w, C, stride, ld, sub_half  (vector path iff C % 8 == 0 and ld == 9C and not sub_half)
    (2, 192, 352, 3, 2, 32, True), (1, 9, 7, 3, 2, 32, True), (2, 96, 176, 32, 1, 288, False), (2, 12, 22, 256, 1, 2304, False),
    (2, 9, 7, 32, 1, 288, False), (2, 9, 7, 32, 2, 288, False), (1, 10, 14, 64, 2, 576, False), (2, 9, 7, 32, 1, 296, False),
    (1, 11, 6, 16, 2, 160, False), (1, 8, 8, 8, 1, 72, True)]


@pytest.mark.parametrize("N,h,w,C,stride,ld,sub_half", IM2COL)
def test_im2col_exact(ops, N, h, w, C, stride, ld, sub_half):
    x = S.dyadic((N * h * w, C), 16, DELTA, h * w + C, device=DEV)
    if sub_half:  # the image lies in [0, 1]
        x = (x.float().abs() * 0.5).bfloat16()
    ho, wo = S.conv_out(h, w, stride)
    buf = nan(N * ho * wo + 2, ld, dtype=torch.bfloat16)  # the row pitch is the padded width ld: columns [9C, ld) get 0
    out = buf[:N * ho * wo]
    ops.im2col3x3(x, N, h, w, C, stride, out, sub_half=sub_half)
    S.exact_check(out, S.im2col_ref(x, N, h, w, C, stride, ld, sub_half), "im2col")
    assert bool(buf[N * ho * wo:].isnan().all()), "im2col wrote past its last row"


@pytest.mark.parametrize("N,h,w,C,stride,extra", [(2, 96, 176, 32, 1, 0), (2, 9, 7, 32, 1, 0), (2, 10, 14, 32, 2, 0),
                                                   (1, 9, 11, 64, 2, 8), (2, 12, 22, 256, 1, 0), (1, 7, 5, 128, 2, 0)])
def test_col2im_exact(ops, N, h, w, C, stride, extra):
    ho, wo = S.conv_out(h, w, stride)
    dcol = S.dyadic((N * ho * wo, 9 * C + extra), 16, DELTA, h + w, device=DEV)
    dx = nan(N * h * w, C, dtype=torch.bfloat16)
    ops.col2im3x3(dcol, N, h, w, C, stride, dx)
    S.exact_check(dx, S.bf16_rn(S.col2im_ref(dcol, N, h, w, C, stride)[0]), "col2im")


@pytest.mark.parametrize("N,h,w,C", [(2, 9, 7, 32), (1, 13, 22, 64), (2, 96, 176, 64), (2, 48, 88, 256), (3, 1, 1, 8),
                                     (2, 24, 44, 512)])
def test_avgpool_exact(ops, N, h, w, C):
    ho, wo = (h + 1) // 2, (w + 1) // 2
    x = S.dyadic((N * h * w, C), 16, DELTA, h * w, device=DEV)
    y = nan(N * ho * wo, C, dtype=torch.bfloat16)
    ops.avgpool2_same(x, N, h, w, C, y)
    S.exact_check(y, S.bf16_rn(S.avgpool_ref(x, N, h, w, C)[0]), "pool")
    dy = S.dyadic((N * ho * wo, C), 16, DELTA, h + w, device=DEV)
    dx = nan(N * h * w, C, dtype=torch.bfloat16)
    ops.avgpool2_same_bwd(dy, N, h, w, C, dx)
    S.exact_check(dx, S.avgpool_bwd_ref(dy, N, h, w, C), "pool bwd")


def test_add_bf16_exact(ops):
    a = S.dyadic((1 << 16,), 200, 2.0 ** -3, 1, device=DEV)
    b = (S.dyadic((1 << 16,), 100, 2.0 ** -9, 2, device=DEV).float() * 3.0).bfloat16()
    out = nan(1 << 16, dtype=torch.bfloat16)
    ops.add_bf16(a, b, out)
    S.exact_check(out, S.bf16_rn(a.double() + b.double()), "add_bf16")


WGRAD = [  # label, N, h, w, cin, cout, k, stride, sub_half
    ("stem1 @192x352 N16", 16, 192, 352, 32, 32, 3, 1, False),
    ("stem0 @192x352", 2, 192, 352, 3, 32, 3, 2, True),
    ("3x3 128->128", 4, 48, 88, 128, 128, 3, 1, False),
    ("1x1 1024->256", 16, 24, 44, 1024, 256, 1, 1, False)]


@functools.lru_cache(maxsize=1)
def _wgrad_problem(label):
    from merlot_b200 import ops
    _, N, h, w, cin, cout, k, stride, sub_half = next(c for c in WGRAD if c[0] == label)
    x = S.dyadic((N * h * w, cin), 1, 1.0, cin + h, device=DEV)
    if sub_half:
        x = (x.float() + 0.5).bfloat16()  # the image conv sees x - 0.5: ternary again
    kp = (k * k * cin + 7) // 8 * 8
    ho, wo = S.conv_out(h, w, stride) if k == 3 else (h, w)
    M = N * ho * wo
    if k == 1:
        a = x
    else:
        a = torch.empty(M, kp, dtype=torch.bfloat16, device=DEV)
        ops.im2col3x3(x, N, h, w, cin, stride, a, sub_half=sub_half)
    dy = S.dyadic((M, cout), 1, 1.0, cout, device=DEV)
    init = torch.randint(-8, 9, (kp, cout), generator=torch.Generator().manual_seed(kp)).float().to(DEV)
    want = init.double()
    for i in range(0, M, 1 << 17):  # float64 a^T dy in slabs of rows
        want += a[i:i + (1 << 17)].double().t() @ dy[i:i + (1 << 17)].double()
    return a, dy, init, want.float(), kp, cout, M


@pytest.mark.parametrize("label", [c[0] for c in WGRAD])
def test_conv_wgrad_exact(ops, label):
    """The wgrad call of HybridStem.backward on ternary operands into an integer-valued gradient: fp32 == int64 for any
    split; the automatic split, 1, 7 and the largest (one k-block per split)."""
    a, dy, init, want, kp, cout, M = _wgrad_problem(label)
    assert M < 2 ** 24 - 8 and float(want.abs().max()) < 2 ** 24
    for splits in (0, 1, 7, -(-M // 64)):
        if splits > 4096 and M > 2 ** 20:
            continue  # 16896 split partials per element: covered at the shorter K
        dws = init.clone()
        ops.gemm(a, dy, a_mn_major=True, b_mn_major=True, out=dws, atomic=True, M=kp, N=cout, K=M, splits=splits)
        S.exact_check(dws, want, f"wgrad {label} splits={splits}")
    assert M <= 2 ** 20 or label.startswith("stem1")


def _ws_shapes():
    return sorted({(op.k * op.k * op.cin, op.cout) for op in stem_ops("s", (3, 4, 9)) if op.kind == "conv"})


def test_weight_standardisation_every_stem_kernel(ops):
    """WsPlan (one launch for every conv kernel of lite_resnet50 [3, 4, 9]): the standardised bf16 operand within the
    midpoint rule and its pad rows 0; the backward accumulated onto dw = 0.5 within its chain bound."""
    shapes = _ws_shapes()
    assert (27, 32) in shapes and (2304, 256) in shapes and max(c for _, c in shapes) == 1024
    g = torch.Generator().manual_seed(21)
    kernels = {f"k{i}": (torch.randn(r, c, generator=g) * 0.2 + 0.05).to(DEV) for i, (r, c) in enumerate(shapes)}
    grads = {n: torch.full(t.shape, 0.5, device=DEV) for n, t in kernels.items()}
    plan = ops.WsPlan(kernels, grads, DEV)
    plan.wstd_arena.fill_(NAN)
    plan.standardise()
    for n, w in kernels.items():
        rows = w.shape[0]
        ref, E = S.ws_ref(w)
        mids = S.interval_check(plan.wstd[n][:rows], ref, E, f"ws {tuple(w.shape)}")
        assert mids <= w.numel() // 100 + 1
        assert bool((plan.wstd[n][rows:] == 0).all())
    for n in kernels:
        plan.dws[n].copy_(torch.randn(plan.dws[n].shape, generator=g))
    plan.backward()
    for n, w in kernels.items():
        ref, E = S.ws_bwd_ref(plan.dws[n][:w.shape[0]], w, torch.full_like(w, 0.5))
        S.bound_check(grads[n], ref, E, f"ws bwd {tuple(w.shape)}")


def test_hybrid_stem_in_situ_192x352(tiny_cfg):
    """lite_resnet50 [3, 4, 9] at 192x352, N = 2, forward and backward on the device: every tape op against float64 on the
    GPU's own saved input and incoming gradient -- GroupNorm statistics, output and backward (dgamma / dbeta from the
    gradient arena), pooling both ways, col2im through the dgrad, each wgrad and the weight-standardisation backward."""
    from merlot_b200 import ops
    from merlot_b200.modeling import _Buffers
    from merlot_b200.stem import HybridStem
    from tests.test_gpu_model import build
    layers = [3, 4, 9]
    cfg = dict(tiny_cfg, resnet_layers=layers, hidden_dropout_prob=0.0)
    _, store, _ = build(cfg)
    N, h0, w0 = 2, 192, 352
    img = torch.rand(N, h0, w0, 3, generator=torch.Generator().manual_seed(0)).bfloat16().to(DEV)
    stem = HybridStem(store, _Buffers(store), layers, save=True)
    out, hs, ws = stem.forward(img, N, h0, w0)
    assert (hs, ws) == (12, 22)
    d_out = (torch.randn(out.shape, generator=torch.Generator().manual_seed(1)) * 0.1).bfloat16().to(DEV)
    store.g.zero_()
    trace = []
    stem.backward(d_out.clone(), trace=trace)
    torch.cuda.synchronize()
    plan = stem.plan()
    seen = {"gn": 0, "pool": 0, "conv": 0, "col2im": 0}
    for t in trace:
        r, kind, dy = t["r"], t["kind"], t["dy"]
        if kind == "gn":
            hw, c = r["hw"], r["c"]
            gamma, beta = store.P(f"{r['scope']}/gamma"), store.P(f"{r['scope']}/beta")
            S.check_gn_stats_bound(r["stats"][:N * 64], r["x"], N, hw, c, what=f"{r['scope']} stats")
            S.check_gn_fwd(r["y"], r["x"], r["stats"][:N * 64], gamma, beta, N, hw, c, relu=r["relu"], shortcut=r["shortcut"],
                           what=f"{r['scope']} fwd")
            out = dict(dx=t["dx"], dshortcut=t["dsc"], dgamma=store.G(f"{r['scope']}/gamma"), dbeta=store.G(f"{r['scope']}/beta"))
            S.check_gn_bwd(out, dy, r["x"], r["y"], r["stats"][:N * 64], gamma, N, hw, c, relu=r["relu"], what=f"{r['scope']} bwd")
        elif kind == "pool":
            hh, ww, c = r["h"], r["w"], r["c"]
            ref, mag = S.avgpool_ref(r["x"], N, hh, ww, c)
            S.interval_check(r["y"], ref, 3.03 * S.U * mag, "pool")
            S.exact_check(t["dx"], S.avgpool_bwd_ref(dy, N, hh, ww, c), "pool bwd")
        else:
            k, cin, cout, kp = r["k"], r["cin"], r["cout"], r["kp"]
            M = N * r["ho"] * r["wo"]
            a = r["x"] if k == 1 else S.im2col_ref(r["x"], N, r["h"], r["w"], cin, r["stride"], kp, r["sub_half"])
            dws = plan.dws[r["kname"]]
            ref = a.double().t() @ dy.double()
            X.elementwise_bound_check(dws, ref, a.double().abs().t() @ dy.double().abs(), M, out_bf16=False)
            rows = k * k * cin
            wref, E = S.ws_bwd_ref(dws[:rows], store.P(r["kname"]), torch.zeros(rows, cout, dtype=torch.float64, device=DEV))
            S.bound_check(store.G(r["kname"]), wref, E, f"{r['kname']} ws bwd")
            if k == 3 and not r["sub_half"]:
                dcol = ops.gemm(dy, plan.wstd[r["kname"]])  # the dgrad HybridStem.backward fed to col2im
                ref, mag = S.col2im_ref(dcol, N, r["h"], r["w"], cin, r["stride"])
                S.interval_check(t["dx"], ref, 8.08 * S.U * mag, "col2im")
                seen["col2im"] += 1
        seen[kind] += 1
    count = lambda kind: len([o for o in stem.ops if o.kind == kind])
    assert seen == {"gn": count("gn"), "pool": count("pool"), "conv": count("conv"), "col2im": 2 + sum(layers)}, seen
    store.g.zero_()
