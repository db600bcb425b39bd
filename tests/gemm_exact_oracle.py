"""Element-by-element references for K1 (merlot_gemm_bf16) and its GeLU epilogues.  Test infrastructure only; no GPU needed.

Exact operands.  int_operands() draws bf16 tensors holding integers in [lo, hi] (default [-2, 2]).  With |a|, |b| <= 2 every
product is an integer of magnitude <= 4, and every partial sum of a K-term dot product with K <= K_MAX = 8512 is an integer of
magnitude <= 4 * 8512 = 34 048 < 2^16 (partial_sum_bound).  Such integers are exact in fp32 with 8 bits to spare, so the fp32
result does not depend on the order of the additions, on how the tensor cores align their addends inside one wgmma, on the
k-block split or on the order of split-K reduce-adds: the correct output is known bit for bit at any shape, and a test can
compare with torch.equal instead of a norm.

exact_product() is that result in float64 (exact for these operands on the CPU and on the GPU).  epilogue_ref() replays
epi_math8 (merlot_b200/csrc/gemm_common.cuh) on it in float32, one IEEE operation per torch elementwise op and in epi_math8's
order (alpha, bias, aux, dropout, residual), then rounds to bf16 to nearest even, as the kernel's stores do.

Non-integer data.  elementwise_bound_check() bounds each element on its own: |C - C64| <= c K 2^-24 (|A||B|)_ij (+ the fp32
roundings of the epilogue's additions, + 1/2 bf16 ulp for a bf16 output), and names the worst element.

GeLU.  The K1 epilogues evaluate Phi(x) by Abramowitz-Stegun 7.1.26 with rcp.approx / ex2.approx (ptx.cuh normal_cdf_fast);
normal_cdf_fast_np() restates it in float32 NumPy with an exact reciprocal and exp2 and without flushing denormals.  Over every
finite bf16 input that restatement gives max |Phi_fast - Phi| = 2.3e-7 (near x = -0.09), max |gelu'_fast - gelu'| = 2.4e-7,
max |gelu_fast - gelu| / |x| = 2.2e-7; rounded to bf16, gelu is within 0.52 bf16 ulp for |x| < 4 but up to 8.6 bf16 ulps
away in the far negative tail (x <= -12), where 7.1.26's *relative* error is large and its absolute error is not.
gelu_bound_check() therefore bounds the absolute error:
    |got - ref| <= ulp(ref) + GELU_ABS * max(|x|, 1),      GELU_ABS = 3e-7
(ulp of the output type; the ulp term covers the output's rounding, including a rounding across a power of two).  GELU_ABS is
the emulation's 2.4e-7 rounded up; a GPU result above it is a finding, not a reason to raise it.
"""
from __future__ import annotations

import numpy as np
import torch
from scipy import special

K_MAX = 8512          # the largest K of the exact GEMM tests (joint-encoder rows: the wgrads' reduction length)
GELU_ABS = 3e-7       # absolute GeLU error per unit of max(|x|, 1); see the module docstring
U32 = 2.0 ** -24      # unit roundoff of fp32


# ---------------------------------------------------------------------------------------------------------------------
# exact integer operands
# ---------------------------------------------------------------------------------------------------------------------
def partial_sum_bound(K: int, lo: int = -2, hi: int = 2) -> int:
    """Largest |partial sum| of a K-term dot product of integers in [lo, hi]."""
    m = max(abs(lo), abs(hi))
    return K * m * m


def int_operands(shape, seed: int, lo: int = -2, hi: int = 2) -> torch.Tensor:
    """bf16 CPU tensor of integers drawn uniformly from [lo, hi] (exact in bf16 for |values| <= 256)."""
    assert -256 <= lo <= hi <= 256
    g = torch.Generator().manual_seed(int(seed))
    return torch.randint(lo, hi + 1, tuple(shape), generator=g).to(torch.bfloat16)


def logical(t: torch.Tensor, mn_major: bool) -> torch.Tensor:
    """The [rows, K] operand an MN-major [K, rows] tensor stands for (a view)."""
    return t.t() if mn_major else t


def exact_product(a: torch.Tensor, b: torch.Tensor, a_mn: bool = False, b_mn: bool = False) -> torch.Tensor:
    """float64 A @ B^T for K1's operand layouts (a: [M, K] or [K, M]; b: [N, K] or [K, N]), on a's device."""
    return logical(a, a_mn).double() @ logical(b, b_mn).double().t()


def epilogue_ref(acc: torch.Tensor, *, alpha: float = 1.0, bias=None, aux=None, keep=None, scale=None, resid=None,
                 out_dtype=torch.bfloat16) -> torch.Tensor:
    """epi_math8's non-GeLU steps on acc (float64 or float32) in float32, in its order, then the output rounding.
    keep: bool mask of kept elements (dropout), scale: the float32 inverted-dropout scale."""
    v = acc.float()
    if alpha != 1.0:
        v = v * float(np.float32(alpha))
    if bias is not None:
        v = v + bias.float()
    if aux is not None:
        v = v * aux.float()
    if keep is not None:
        v = torch.where(keep, v * float(np.float32(scale)), torch.zeros((), dtype=v.dtype, device=v.device))
    if resid is not None:
        v = v + resid.float()
    return v.to(out_dtype)


# ---------------------------------------------------------------------------------------------------------------------
# ulps and element-wise bounds
# ---------------------------------------------------------------------------------------------------------------------
def _np32(x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        x = x.detach().float().cpu().numpy()
    return np.ascontiguousarray(x, np.float32)


def bf16_ulps(a, b) -> np.ndarray:
    """Distance in bf16 units of last place between bf16 values given as float32 arrays or tensors (sign-magnitude order:
    +0 and -0 are 0 apart, the largest negative subnormal and the smallest positive one 2)."""
    def order(x):
        bits = (_np32(x).view(np.uint32) >> 16).astype(np.int64)
        return np.where(bits & 0x8000, -(bits & 0x7FFF), bits)
    return np.abs(order(a) - order(b))


def ulp(x, mant_bits: int) -> np.ndarray:
    """Spacing of a binary format with `mant_bits` explicit significand bits and fp32's exponent range (bf16: 7, fp32: 23)
    at |x|: 2^(e - mant_bits) for |x| in [2^e, 2^(e+1)), the subnormal spacing 2^(-126 - mant_bits) below 2^-126."""
    x = np.abs(np.asarray(x, np.float64))
    _, e = np.frexp(x)  # x = m 2^e, m in [0.5, 1); e = 0 at x = 0
    return np.ldexp(1.0, np.where(x == 0, -126, np.maximum(e - 1, -126)) - mant_bits)


def ulp_bf16(x) -> np.ndarray:
    return ulp(x, 7)


def ulp_f32(x) -> np.ndarray:
    return ulp(x, 23)


def _ulp_bf16_t(x: torch.Tensor) -> torch.Tensor:
    """ulp_bf16 on a float64 tensor (on its device)."""
    _, e = torch.frexp(x.abs())
    e = torch.where(x == 0, torch.full_like(e, -126), torch.clamp(e - 1, min=-126))
    return torch.ldexp(torch.ones_like(x), e - 7)


def elementwise_bound_check(got: torch.Tensor, ref: torch.Tensor, absprod: torch.Tensor, K: int, *, c: float = 2.0,
                            extra=None, out_bf16: bool = True):
    """Assert |got - ref| <= c K 2^-24 absprod (+ 2 2^-24 extra) (+ 1/2 bf16 ulp of max(|got|, |ref|)) element by element,
    on ref's device.  ref: the float64 result; absprod: |A| @ |B|^T in float64 (the sum of the magnitudes of the products);
    extra: a bound on the magnitudes of the epilogue's fp32 additions (bias, residual; two roundings).  c = 2 lets each of
    the accumulations of the tensor cores truncate rather than round.  Returns the worst element's (index, err / bound)."""
    got = got.to(ref.device, torch.float64)
    assert bool(torch.isfinite(got).all()), f"{int((~torch.isfinite(got)).sum())} non-finite elements"
    bound = (c * K * U32) * absprod
    if extra is not None:
        bound = bound + (2 * U32) * extra.to(torch.float64)
    if out_bf16:
        bound = bound + 0.5 * _ulp_bf16_t(torch.maximum(got.abs(), ref.abs()))
    bound = bound.clamp(min=2.0 ** -149)
    ratio = (got - ref).abs() / bound
    i = int(ratio.argmax())
    idx = tuple(int(j) for j in np.unravel_index(i, tuple(ratio.shape)))
    worst = float(ratio.reshape(-1)[i])
    assert worst <= 1.0, (f"element {idx}: got {float(got[idx])!r}, float64 {float(ref[idx])!r}, {worst:.3g} x the bound "
                          f"{float(bound[idx]):.3g}")
    return idx, worst


def exact_check(got: torch.Tensor, want: torch.Tensor, what: str = "", nan_ok: bool = False):
    """Equality element by element, naming the first wrong element and how many there are.  A NaN is wrong unless nan_ok
    and want holds NaN there too."""
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, got.dtype, want.shape, want.dtype)
    bad = got.ne(want)
    if nan_ok:
        bad &= ~(got.isnan() & want.isnan())
    n = int(bad.sum())
    if n:
        idx = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} of {got.numel()} elements differ; first at {idx}: got {float(got[idx])!r}, "
                             f"want {float(want[idx])!r}")


# ---------------------------------------------------------------------------------------------------------------------
# GeLU
# ---------------------------------------------------------------------------------------------------------------------
def all_bf16() -> torch.Tensor:
    """The 65 536 bf16 bit patterns, in bit order, as a bf16 tensor."""
    return torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)


def gelu_ref(x, kind: str) -> np.ndarray:
    """float64 reference: kind 'phi' -> Phi(x), 'gelu' -> x Phi(x), 'dgelu' -> Phi(x) + x phi(x) (scipy ndtr)."""
    x = np.asarray(x, np.float64)
    phi_cdf = special.ndtr(x)
    if kind == "phi":
        return phi_cdf
    if kind == "gelu":
        return x * phi_cdf
    if kind == "dgelu":
        with np.errstate(over="ignore"):
            return phi_cdf + x * (np.exp(-0.5 * x * x) / np.sqrt(2 * np.pi))
    raise ValueError(kind)


def gelu_errors(x, got, kind: str, out: str = "bf16") -> dict:
    """Error statistics of got (float32/bf16 values) against gelu_ref over finite x: max |err|, max |err| / max(|x|, 1), the
    worst output-ulp distance overall, for |x| < 4 and for x <= -4."""
    x = np.asarray(_np32(x), np.float64)
    g = np.asarray(_np32(got), np.float64)
    ref = gelu_ref(x, kind)
    err = np.abs(g - ref)
    u = ulp_bf16(ref) if out == "bf16" else ulp_f32(ref)
    ulps = err / u
    mid, tail = np.abs(x) < 4, x <= -4
    i = int(np.argmax(err / np.maximum(np.abs(x), 1)))
    return dict(max_abs=float(err.max()), max_abs_per_x=float((err / np.maximum(np.abs(x), 1)).max()), at=float(x[i]),
                max_ulps=float(ulps.max()), max_ulps_mid=float(ulps[mid].max()) if mid.any() else 0.0,
                max_ulps_tail=float(ulps[tail].max()) if tail.any() else 0.0)


def gelu_bound_check(x, got, kind: str, *, out: str = "bf16", abs_coef: float = GELU_ABS, ulps: float = 1.0):
    """Assert |got - ref| <= ulps * ulp_out(ref) + abs_coef * max(|x|, 1) for every (finite) x; kind: 'gelu', 'dgelu' or
    'phi'; out: 'bf16' or 'f32' (the output format whose ulp the first term takes).  Returns the worst (x, err / bound)."""
    x = np.asarray(_np32(x), np.float64)
    g = np.asarray(_np32(got), np.float64)
    assert x.shape == g.shape and np.isfinite(x).all()
    assert np.isfinite(g).all(), f"{kind}: non-finite output at x = {x[~np.isfinite(g)][:4]}"
    ref = gelu_ref(x, kind)
    u = ulp_bf16(ref) if out == "bf16" else ulp_f32(ref)
    bound = ulps * u + abs_coef * np.maximum(np.abs(x), 1.0)
    err = np.abs(g - ref)
    i = int(np.argmax(err / bound))
    ratio = float(err[i] / bound[i])
    assert ratio <= 1.0, (f"{kind}({x[i]!r}): got {g[i]!r}, float64 {ref[i]!r}, error {err[i]:.3g} is {ratio:.3g} x the "
                          f"bound {bound[i]:.3g}")
    return float(x[i]), ratio


def normal_cdf_fast_np(x):
    """ptx.cuh normal_cdf_fast in float32 NumPy with an exact reciprocal and exp2 (the GPU's rcp.approx / ex2.approx are
    approximations of these) and without flushing denormals; an fmaf is its exact product and sum rounded to float32.
    Returns (Phi(x), exp(-x^2 / 2)) as float32 arrays."""
    f = np.float32
    x = _np32(x)

    def fma(a, b, c):
        return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)

    with np.errstate(over="ignore", under="ignore", invalid="ignore", divide="ignore"):
        t = f(1) / fma(f(0.23164190), np.abs(x), f(1))
        e = np.exp2((x * x) * f(-0.72134752))
        poly = fma(t, f(0.5307027145), f(-0.7265760135))
        poly = fma(poly, t, f(0.7107068705))
        poly = fma(poly, t, f(-0.142248368))
        poly = fma(poly, t, f(0.127414796))
        half_erfc = (poly * t) * e
        cdf = np.where(x >= 0, f(1) - half_erfc, half_erfc).astype(np.float32)
    return cdf, e


def gelu_fast_np(x, kind: str):
    """The fast epilogue's gelu ('gelu': x * Phi) or gelu' ('dgelu': fmaf(x * 0.39894228, e, Phi)) in float32 NumPy."""
    x = _np32(x)
    cdf, e = normal_cdf_fast_np(x)
    with np.errstate(over="ignore", invalid="ignore"):
        if kind == "phi":
            return cdf
        if kind == "gelu":
            return (x * cdf).astype(np.float32)
        return (np.asarray(x * np.float32(0.39894228040143267794), np.float64) * e + cdf).astype(np.float32)
