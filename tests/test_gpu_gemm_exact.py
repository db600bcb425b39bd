"""K1 (merlot_gemm_bf16) element by element.  Integer operands in [-2, 2] make every partial sum an exact fp32 integer
(tests/gemm_exact_oracle.py), so the main loop, every epilogue kind, split-K reduce-adds and the persistent grids are compared
bitwise with a float64 product and a float32 replay of the epilogue: a wrong element, 8-column group, 16-row slice, k-block,
split or store position fails however large the output.  Random data meets a per-element bound, and the GeLU epilogues and
kernels are checked over every bf16 input (pytest -m gpu)."""
import functools

import numpy as np
import pytest
import torch

from oracle import dropout_mask as DM
from tests import gemm_exact_oracle as X
from tests.test_gpu_sm_reserve import _reserves, sm_reserve

pytestmark = pytest.mark.gpu
DEV = "cuda"
MAJORS = [(False, False), (False, True), (True, True), (True, False)]  # (a_mn, b_mn)
NAN = float("nan")


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def _pad8(n):
    return (n + 7) // 8 * 8


def nan_view(rows, cols, dtype=torch.bfloat16, extra_rows=3, extra_cols=8):
    """A [rows, cols] view into a NaN-filled buffer with more rows and a wider (16-byte multiple) row pitch."""
    buf = torch.full((rows + extra_rows, _pad8(cols) + extra_cols), NAN, dtype=dtype, device=DEV)
    return buf, buf[:rows, :cols]


def operand(t, mn_major):
    """The logical [rows, K] operand t laid out as K1 reads it ([rows, K], or [K, rows] when MN-major), as a view into a
    NaN-filled buffer: extra columns past the row length and extra rows past its end (the K tail of an MN-major operand)."""
    src = t.t() if mn_major else t
    _, v = nan_view(*src.shape)
    v.copy_(src)
    return v


def check_outside_nan(buf, M, N, what):
    assert bool(torch.isnan(buf[:, N:]).all()) and bool(torch.isnan(buf[M:, :]).all()), f"{what}: wrote outside [M, N)"


@pytest.fixture(scope="module", autouse=True)
def _release_problems():
    yield
    _int_problem.cache_clear()


@functools.lru_cache(maxsize=None)
def _int_problem(M, N, K):
    """Integer operands (logical A [M, K], B [N, K], on the GPU) and their exact product (float32, exact)."""
    a = X.int_operands((M, K), M * 131 + K).to(DEV)
    b = X.int_operands((N, K), N * 137 + K + 1).to(DEV)
    return a, b, X.exact_product(a, b).float()


def _main_loop(ops, M, N, K, bn, a_mn, b_mn):
    a, b, want = _int_problem(M, N, K)
    buf, out = nan_view(M, N, torch.float32)
    ops.gemm(operand(a, a_mn), operand(b, b_mn), a_mn_major=a_mn, b_mn_major=b_mn, out=out, block_n=bn)
    X.exact_check(out, want, f"{M}x{N}x{K} bn={bn} a_mn={a_mn} b_mn={b_mn}")
    check_outside_nan(buf, M, N, "fp32 output")


def _main_loop_shapes(bn):
    return [(1, 8, 1), (1, 8, 3), (1, 8, 8),                         # degenerate
            (129, bn + 8, 65), (192, 2 * bn - 8, 127), (255, 3 * bn + 8, 40),  # M % 128 in {1, 64, 127}, N % BN in {8, BN - 8}, K % 64 in {1, 63}, K < 64
            (130, 50376, 768)]                                       # the vocabulary width


MULTI_WAVE = [(8512, 3072, 768), (3168, 768, 3072)]


@pytest.mark.parametrize("a_mn,b_mn", MAJORS, ids=lambda v: "mn" if v else "k")
@pytest.mark.parametrize("bn", [128, 192, 256])
def test_main_loop_exact(ops, bn, a_mn, b_mn):
    """fp32 output of A @ B^T bitwise, for every operand layout, from NaN-padded operand views into a NaN-filled output
    buffer: the tensor maps stop at the logical extents (NaN read past them would reach the result), the stores at [M, N)."""
    for M, N, K in _main_loop_shapes(bn):
        _main_loop(ops, M, N, K, bn, a_mn, b_mn)


@pytest.mark.parametrize("a_mn,b_mn", MAJORS, ids=lambda v: "mn" if v else "k")
@pytest.mark.parametrize("bn", [128, 192, 256])
@pytest.mark.parametrize("M,N,K", MULTI_WAVE)
def test_main_loop_exact_multi_wave(ops, M, N, K, bn, a_mn, b_mn):
    """Persistent grids of several tiles per CTA (8512 x 3072: 67 x 12..24 tiles)."""
    _main_loop(ops, M, N, K, bn, a_mn, b_mn)


# ---------------------------------------------------------------------------------------------------------------------
# every epilogue kind on integer data
# ---------------------------------------------------------------------------------------------------------------------
EPI_SHAPES = [(300, 264, 200), (515, 1000, 136)]  # N % 16 == 8: the fast epilogue's last 16-column step is half outside
SEED, SITE = 2 ** 35 + 9, 77


@pytest.mark.parametrize("bn", [128, 192, 256])
@pytest.mark.parametrize("M,N,K", EPI_SHAPES)
def test_epilogues_exact(ops, M, N, K, bn):
    """Plain, bias, residual, bias + residual, alpha (generic), dropout at p = 0.5 (scale 2: exact) with and without the
    residual, mul_aux (fast and forced generic) and GELU2's pre-activation: bitwise against the float32 replay of
    epi_math8, each written into a NaN-filled wider and taller buffer that must keep its NaN outside [M, N)."""
    a, wt, acc = _int_problem(M, N, K)                   # wt: [N, K] (K-major, the dgrad orientation)
    w = operand(wt, True)                                 # [K, N] (MN-major, the forward orientation)
    g = torch.Generator().manual_seed(M + N + bn)
    bias = torch.randint(-8, 9, (N,), generator=g).float().to(DEV)
    resid = X.int_operands((M, N), M + N + 3, -16, 16).to(DEV)
    aux = X.int_operands((M, N), M + N + 4).to(DEV)
    keep5 = torch.from_numpy(DM.counter_dropout_keep(SEED, SITE, M, N, 0.5)).to(DEV)
    fwd = dict(b_mn_major=True, block_n=bn)
    cases = {
        "plain": (dict(), dict()),
        "bias": (dict(bias=bias), dict(bias=bias)),
        "resid": (dict(resid=resid), dict(resid=resid)),
        "bias_resid": (dict(bias=bias, resid=resid), dict(bias=bias, resid=resid)),
        "alpha0.5": (dict(bias=bias, resid=resid, alpha=0.5), dict(bias=bias, resid=resid, alpha=0.5)),
        "alpha2": (dict(bias=bias, alpha=2.0), dict(bias=bias, alpha=2.0)),
        "dropout": (dict(bias=bias, dropout_p=0.5, dropout_seed=SEED, dropout_site=SITE),
                    dict(bias=bias, keep=keep5, scale=DM.dropout_scale(0.5))),
        "dropout_resid": (dict(bias=bias, resid=resid, dropout_p=0.5, dropout_seed=SEED, dropout_site=SITE),
                          dict(bias=bias, resid=resid, keep=keep5, scale=DM.dropout_scale(0.5))),
        "mul_aux": (dict(mul_aux=aux), dict(aux=aux)),
        "mul_aux_generic": (dict(mul_aux=aux, generic_epilogue=True), dict(aux=aux)),
    }
    for name, (kw, ref_kw) in cases.items():
        want = X.epilogue_ref(acc, **ref_kw)
        for b, extra in ((w, fwd), (wt, dict(block_n=bn))):
            buf, out = nan_view(M, N, extra_rows=5, extra_cols=24)
            ops.gemm(a, b, out=out, **extra, **kw)
            X.exact_check(out, want, f"{name} b_mn={b is w}")
            check_outside_nan(buf, M, N, name)
    for generic in (False, True):
        for grad_out in (False, True):
            pre_buf, pre = nan_view(M, N, extra_rows=5, extra_cols=24)
            act_buf, act = nan_view(M, N, extra_rows=5, extra_cols=24)
            ops.gemm(a, w, bias=bias, gelu=True, out_pre=pre, out=act, gelu_grad_out=grad_out, generic_epilogue=generic,
                     **fwd)
            x = (acc + bias).cpu().numpy()  # the fp32 pre-activation (exact)
            what = f"gelu2 generic={generic} grad_out={grad_out}"
            check_outside_nan(pre_buf, M, N, what)
            check_outside_nan(act_buf, M, N, what)
            X.gelu_bound_check(x.ravel(), act.cpu().ravel(), "gelu")
            if grad_out:
                X.gelu_bound_check(x.ravel(), pre.cpu().ravel(), "dgelu")
            else:
                X.exact_check(pre, X.epilogue_ref(acc, bias=bias), what)


@pytest.mark.parametrize("bn", [128, 256])
def test_dropout_p01_resid_within_one_ulp(ops, bn):
    """Dropout at p = 0.1 with a residual: v * (1 / 0.9) + resid is not exact, and the compiler may contract it into one FMA
    where the replay rounds twice, so the bar is 1 bf16 ulp (and the dropped elements exactly the residual)."""
    M, N, K = 515, 1000, 136
    a, wt, acc = _int_problem(M, N, K)
    resid = X.int_operands((M, N), 5, -16, 16).to(DEV)
    keep = torch.from_numpy(DM.counter_dropout_keep(SEED, SITE, M, N, 0.1)).to(DEV)
    got = ops.gemm(a, wt, resid=resid, dropout_p=0.1, dropout_seed=SEED, dropout_site=SITE, block_n=bn)
    want = X.epilogue_ref(acc, keep=keep, scale=DM.dropout_scale(0.1), resid=resid)
    d = X.bf16_ulps(got, want)
    assert d.max() <= 1, f"max {int(d.max())} ulp"
    X.exact_check(got[~keep], resid[~keep], "dropped elements")


# ---------------------------------------------------------------------------------------------------------------------
# split-K reduce-add (the wgrad orientation: both operands MN-major, fp32 output += A @ B^T)
# ---------------------------------------------------------------------------------------------------------------------
SPLIT_SHAPES = [(768, 768, 8511), (3072, 768, 3199), (200, 264, 575), (64, 8, 1023)]  # K = 64 num_kb - 1: a short last k-block
SPLIT_VARIANTS = {"red_f32": dict(block_n=256), "generic128": dict(block_n=128), "generic192": dict(block_n=192),
                  "generic256": dict(block_n=256, generic_epilogue=True)}


def _split_k(ops, M, N, K, splits, variant):
    x, dy, prod = _int_problem(M, N, K)  # logical [M, K] and [N, K]
    init = X.int_operands((M, N), M + N, -64, 64).float().to(DEV)
    dw = init.clone()
    ops.gemm(x.t().contiguous(), dy.t().contiguous(), a_mn_major=True, b_mn_major=True, out=dw, atomic=True,
             splits=splits, **SPLIT_VARIANTS[variant])
    X.exact_check(dw, init + prod, f"{M}x{N}x{K} splits={splits} {variant}")


@pytest.mark.parametrize("variant", list(SPLIT_VARIANTS))
@pytest.mark.parametrize("M,N,K", SPLIT_SHAPES)
def test_split_k_reduce_add_exact(ops, M, N, K, variant):
    """Into a gradient that already holds integers, for 1, 2, 3, 5 and the automatic number of splits: bitwise."""
    assert X.partial_sum_bound(K) + 64 < 2 ** 16
    for splits in (1, 2, 3, 5, 0):
        _split_k(ops, M, N, K, splits, variant)


# ---------------------------------------------------------------------------------------------------------------------
# persistent grids under merlot_set_sm_reserve
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("reserve", _reserves(), ids=lambda n: f"reserve{n}")
@pytest.mark.parametrize("M,N,K", MULTI_WAVE)
def test_multi_wave_exact_under_reserve(ops, reserve, M, N, K):
    """SMs - reserve CTAs: at SMs - 9 each walks ~90 tiles, so the ring phase and the staging parity wrap many times."""
    with sm_reserve(reserve):
        for bn in (128, 192, 256):
            for a_mn, b_mn in MAJORS:
                _main_loop(ops, M, N, K, bn, a_mn, b_mn)


@pytest.mark.parametrize("reserve", _reserves(), ids=lambda n: f"reserve{n}")
@pytest.mark.parametrize("M,N,K", SPLIT_SHAPES)
def test_split_k_exact_under_reserve(ops, reserve, M, N, K):
    """The automatic split count follows the grid; explicit splits run with fewer CTAs than tiles."""
    with sm_reserve(reserve):
        for variant in ("red_f32", "generic128"):
            for splits in (1, 3, 5, 0):
                _split_k(ops, M, N, K, splits, variant)


# ---------------------------------------------------------------------------------------------------------------------
# random data: per-element bound
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(8512, 2304, 768), (8512, 768, 768), (8512, 3072, 768), (3168, 768, 3072)])
def test_random_data_elementwise_bound(ops, M, N, K):
    """The shapes the ViT and joint-encoder layers launch (automatic tile width), plain and bias + residual, on random bf16
    data (mixed exponents, which integers lack): every element within c K 2^-24 (|A||B|)_ij + the epilogue's roundings."""
    g = torch.Generator().manual_seed(M + N + K)
    a = (torch.randn(M, K, generator=g) * 0.3).bfloat16().to(DEV)
    w = (torch.randn(K, N, generator=g) * 0.1).bfloat16().to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    resid = torch.randn(M, N, generator=g).bfloat16().to(DEV)
    ref = a.double() @ w.double()
    absprod = a.double().abs() @ w.double().abs()
    got = ops.gemm(a, w, b_mn_major=True, out_dtype=torch.float32)
    X.elementwise_bound_check(got, ref, absprod, K, out_bf16=False)
    got = ops.gemm(a, w, b_mn_major=True)
    X.elementwise_bound_check(got, ref, absprod, K)
    got = ops.gemm(a, w, b_mn_major=True, bias=bias, resid=resid)
    extra = absprod + bias.double().abs() + resid.double().abs()
    X.elementwise_bound_check(got, ref + bias.double() + resid.double(), absprod, K, extra=extra)


# ---------------------------------------------------------------------------------------------------------------------
# GeLU over every bf16 value
# ---------------------------------------------------------------------------------------------------------------------
ALL = X.all_bf16().float()                 # 65 536 inputs, in bit order
FINITE = torch.isfinite(ALL)


def _same_as_float64(x, got, kind, what):
    """NaN in, NaN out; +-inf as the float64 formula gives them (gelu(+inf) = +inf; -inf * Phi(-inf) and inf * phi(inf)
    are NaN there as here)."""
    with np.errstate(invalid="ignore", over="ignore"):
        x = x.numpy().astype(np.float64)
        ref = X.gelu_ref(x, kind)
        got = got.numpy().astype(np.float64)
    ok = (got == ref) | (np.isnan(got) & np.isnan(ref))
    assert ok.all(), f"{what}: x = {x[~ok][:4]} -> {got[~ok][:4]}, float64 {ref[~ok][:4]}"


def _gelu_checks(got_row, kind, what, out="bf16", **bound):
    got = got_row.float().cpu()
    X.gelu_bound_check(ALL[FINITE], got[FINITE], kind, out=out, **bound)
    _same_as_float64(ALL[~FINITE], got[~FINITE], kind, what)


@pytest.mark.parametrize("generic", [False, True], ids=["fast", "generic"])
@pytest.mark.parametrize("bn", [128, 192, 256])
def test_gelu2_every_bf16(ops, bn, generic):
    """A = 0 and the bias carrying the 65 536 bf16 values as columns: the pre-activation is exactly the bias."""
    M, N, K = 3, 65536, 8
    a = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
    w = torch.ones(K, N, dtype=torch.bfloat16, device=DEV)
    bias = ALL.to(DEV)
    for grad_out in (False, True):
        pre = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        act = ops.gemm(a, w, b_mn_major=True, bias=bias, gelu=True, out_pre=pre, gelu_grad_out=grad_out, block_n=bn,
                       generic_epilogue=generic)
        tag = f"{'generic' if generic else 'fast'} bn={bn}"
        for r in range(M):
            _gelu_checks(act[r], "gelu", f"gelu2 gelu {tag}")
            if grad_out:
                _gelu_checks(pre[r], "dgelu", f"gelu2 gelu' {tag}")
            else:
                X.exact_check(pre[r], X.epilogue_ref(torch.zeros(N, device=DEV), bias=bias), f"pre {tag}", nan_ok=True)


def test_dgelu_aux_every_bf16(ops):
    """MUL_DGELU (generic epilogue): A @ B^T = 1 exactly (one column of ones in each, K = 8), aux = every bf16 value."""
    M, N, K = 2, 65536, 8
    a = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
    b = torch.zeros(N, K, dtype=torch.bfloat16, device=DEV)
    a[:, 3] = 1
    b[:, 3] = 1
    aux = ALL.bfloat16().to(DEV).expand(M, N).contiguous()
    got = ops.gemm(a, b, dgelu_aux=aux)
    for r in range(M):
        _gelu_checks(got[r], "dgelu", "mul_dgelu")


# libdevice erff: 2 ulp; __expf: 2 + floor(1.173 |w|) ulp (CUDA C Programming Guide, mathematical functions appendix).
# gelu_erf = x * 0.5 * (1 + erff(x / sqrt 2)): erff's 2 ulp (<= 1.2e-7 below 1 in magnitude), the rounded argument
# (<= 3e-8 through erf') and the rounding of 1 + erf (<= 6e-8) give <= 2.1e-7 in 1 + erf, so <= 1.1e-7 |x| after the 0.5 x,
# plus the last rounding: |err| <= ulp(ref) + 1.2e-7 max(|x|, 1).
# gelu_erf_grad = Phi + x * 0.39894228 * __expf(-0.5 x x): Phi as above (<= 1.05e-7); pdf's relative error
# 2^-24 (5 + 3.35 w), w = x^2 / 2, times |x| phi(x) is <= 1.2e-7 for every x; so |err| <= ulp(ref) + 2.5e-7.
LIBDEVICE_BOUNDS = {"gelu": 1.2e-7, "dgelu": 2.5e-7}


def test_gelu_f32_kernels_every_bf16(ops):
    """merlot_gelu_f32 / merlot_gelu_bwd_f32 (libdevice erff, __expf) over every bf16 value, dy = 1."""
    x = ALL.to(DEV)
    y = torch.empty_like(x)
    ops.gelu_f32(x, y)
    _gelu_checks(y, "gelu", "gelu_f32", out="f32", abs_coef=LIBDEVICE_BOUNDS["gelu"])
    dx = torch.empty_like(x)
    ops.gelu_bwd_f32(torch.ones_like(x), x, dx)
    _gelu_checks(dx, "dgelu", "gelu_bwd_f32", out="f32", abs_coef=LIBDEVICE_BOUNDS["dgelu"])
