"""Element-by-element references for the row-wise LayerNorm family of merlot_b200/csrc/rowwise.cu: ln_fwd_kernel
(merlot_layernorm_fwd), ln_bwd_kernel + reduce_partials_kernel (merlot_layernorm_bwd), ln_bwd_fused_kernel
(merlot_layernorm_bwd_fused) and colsum_kernel (merlot_bias_grad).  Test infrastructure only; every function is plain torch
in float64 and runs on the CPU or on the GPU.

References.  ln_fwd_ref is utils/model_utils.py:113-130 in float64 (biased variance, eps as the float32 the kernel is given).
The backward references take the fp32 mean and rstd the kernel was given as INPUTS, so their bounds cover only the kernel's
own arithmetic: xhat = (x - mean) * rstd, dx = rstd * (g dy - mean(g dy) - xhat mean(g dy xhat)) (+ dres).

Bounds.  u = 2^-24 per fp32 rounding.  One warp owns a row; lane l sums its chunks c = l + 32 j (8 values each) one value at
a time, then warp_sum's 5-level butterfly adds the 32 lane sums.  A value therefore passes through at most
    sum_depth(H) = 8 * NCH + 5        (NCH = ceil(H / 256) chunks per lane)
fp32 additions, and every such row sum is within sum_depth(H) * u * sum|terms| of the exact one (the standard bound of
recursive summation; the factor 1/(1 - k u) is inside SLACK).  The division by H is IEEE-rounded (the build has no fast-math):
u relative; the fused backward multiplies by fl(1/H) instead: 2u.  rsqrtf is within 2 ulp: RSQRT_REL = 4u relative.  The
build leaves -fmad on, so nvcc may contract x*s - mean*s + b (and the other product-sums) into FMAs: each product is then
either rounded or not, and the bound of y charges u per operation on every operand it may meet, u (|x s| + |mean s| + |b|)
three times, not u |y|.  This matters when mean is large compared with the row's spread.  Terms of second order in u are
covered by SLACK = 1.01 (they are below 1e-9 relative for every shape here).

Reductions over rows (dgamma, dbeta, the bias gradients) add per-lane chains over the rows a warp owns, then the warps of a
block, then the blocks (through atomics in any order): col_depth_* counts the longest such chain, and the bound is
depth * u * (|prefill| + sum|terms|) plus the propagated error of each term.

Exact operands.  zero_sum rows (a permutation of +-k pairs, 1 <= k <= 8) and constant rows of small integers make every sum
of x and of (x - mean)^2 an integer below 2^24, exact in fp32 in any order: mean_out must equal sum/H exactly and the
kernel's variance is exactly fp32(sum (x - mean)^2 / H), so rstd_out is within 2 ulp of 1 / sqrt(fp32(var32 + eps))
(check_exact_stats).  This catches a wrong divisor, unbiased variance, a wrong eps or a dropped lane whatever the output
dtype.  Integer dy with p in {0, 0.5} (keep scale exactly 2) makes bias_grad and dbeta integer sums below 2^24: bit-exact in
any atomic order, on top of an integer prefill.

bf16 outputs must lie in [bf16_rn(ref - E), bf16_rn(ref + E)] (check_bf16): the correctly rounded value, or its neighbour
only where the float64 value lies within the bound E of a rounding midpoint.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests.stem_exact_oracle import bf16_rn, exact_check  # noqa: F401  (exact_check is part of this module's interface)

U = 2.0 ** -24
RSQRT_REL = 4 * U
SLACK = 1.01
TINY = 2.0 ** -140
EPS = 1e-5
LNF_WARPS = 12        # ln_bwd_fused_kernel: warps per block, one block per SM at most
LNF_STAGES = 3        # its ring depth (rows in flight per warp)
LN_BWD_WARPS = 8      # ln_bwd_kernel: 256 threads; grid capped at 2 * SMs
RSPLIT = 16           # reduce_partials_kernel's split of the block partials
COLSUM_SLAB, COLSUM_MAX_SLABS = 64, 128
ROW_CLASSES = ("random", "zero_sum", "constant", "offset", "near_eps", "spike", "large", "zero")


def eps32(eps: float = EPS) -> float:
    return float(np.float32(eps))


# ---------------------------------------------------------------------------------------------------------------------
# launch geometry
# ---------------------------------------------------------------------------------------------------------------------
def nch(H: int) -> int:
    """16-byte chunks per lane: ceil(H / 256).  Lanes l < (H / 8) % 32 own one chunk more than the others when H % 256 != 0."""
    return -(-H // 256)


def sum_depth(H: int) -> int:
    """fp32 additions a value passes through in a warp's row sum: the lane's chain over its 8 * NCH values, then the butterfly."""
    return 8 * nch(H) + 5


def fused_grid(rows: int, sms: int) -> int:
    return min(-(-rows // LNF_WARPS), sms)


def col_depth_fused(rows: int, sms: int, launches: int = 1) -> int:
    """ln_bwd_fused_kernel's column sums: the warp's chain over its rows, the block's sum over its 12 warp slabs, one red.add
    per block and launch onto the prefilled accumulator."""
    G = fused_grid(rows, sms)
    return -(-rows // (G * LNF_WARPS)) + LNF_WARPS + launches * G + 1


def unfused_grid(rows: int, sms: int) -> int:
    return min(-(-rows // LN_BWD_WARPS), 2 * sms)


def col_depth_unfused(rows: int, sms: int, launches: int = 1) -> int:
    """ln_bwd_kernel + reduce_partials_kernel: the warp's chain over its rows, the 8 warps' shared atomics, one thread's chain
    over every RSPLIT-th block partial, then RSPLIT atomics per launch onto the prefilled accumulator."""
    grid = unfused_grid(rows, sms)
    return -(-rows // (grid * LN_BWD_WARPS)) + LN_BWD_WARPS + -(-grid // RSPLIT) + launches * RSPLIT + 1


def colsum_slabs(rows: int) -> int:
    return min(-(-rows // COLSUM_SLAB), COLSUM_MAX_SLABS)


def col_depth_colsum(rows: int, launches: int = 1) -> int:
    """colsum_kernel: one thread's chain over the rows of its slab (stride 8 * slabs), the 8 warps of the block, one atomic per
    slab and launch onto the prefilled output."""
    slabs = colsum_slabs(rows)
    return -(-rows // (8 * slabs)) + 8 + launches * slabs + 1


# ---------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------
def ln_rows(rows: int, H: int, seed: int, dtype=torch.bfloat16, classes=ROW_CLASSES) -> torch.Tensor:
    """[rows, H] CPU tensor of `dtype`; row i is of class classes[(i + seed) % len(classes)]:
    random (2 N(0,1) + 0.5), zero_sum (+-k pairs, 1 <= k <= 8, permuted), constant (an integer in [-8, 8]), offset (mean about
    256, spread about 2), near_eps (variance about eps), spike (one non-zero of magnitude 1 to 64), large (magnitude 1e4),
    zero."""
    assert H % 2 == 0
    g = torch.Generator().manual_seed(int(seed))
    out = torch.empty(rows, H, dtype=torch.float64)
    cls_of = [(i + seed) % len(classes) for i in range(rows)]
    for ci, cls in enumerate(classes):
        sel = torch.tensor([i for i in range(rows) if cls_of[i] == ci], dtype=torch.long)
        n = len(sel)
        if n == 0:
            continue
        if cls == "random":
            v = torch.randn(n, H, generator=g, dtype=torch.float64) * 2 + 0.5
        elif cls == "zero_sum":
            k = torch.randint(1, 9, (n, H // 2), generator=g).double()
            perm = torch.rand(n, H, generator=g).argsort(-1)
            v = torch.cat([k, -k], 1).gather(1, perm)
        elif cls == "constant":
            v = torch.randint(-8, 9, (n, 1), generator=g).double().expand(n, H)
        elif cls == "offset":
            v = 256 + torch.randn(n, H, generator=g, dtype=torch.float64) * 2
        elif cls == "near_eps":
            v = torch.randn(n, H, generator=g, dtype=torch.float64) * math.sqrt(EPS)
        elif cls == "spike":
            v = torch.zeros(n, H, dtype=torch.float64)
            mag = torch.randint(1, 65, (n,), generator=g).double() * (torch.randint(0, 2, (n,), generator=g) * 2 - 1)
            v[torch.arange(n), torch.randint(0, H, (n,), generator=g)] = mag
        elif cls == "large":
            v = torch.randn(n, H, generator=g, dtype=torch.float64) * 1e4
        elif cls == "zero":
            v = torch.zeros(n, H, dtype=torch.float64)
        else:
            raise ValueError(cls)
        out[sel] = v
    return out.to(dtype)


def int_rows(rows: int, H: int, seed: int, lo: int = -8, hi: int = 8, dtype=torch.bfloat16) -> torch.Tensor:
    """Integers uniform in [lo, hi] (exact in bf16)."""
    g = torch.Generator().manual_seed(int(seed))
    return torch.randint(lo, hi + 1, (rows, H), generator=g).to(dtype)


def exact_int_sum_holds(terms: torch.Tensor, prefill: torch.Tensor) -> bool:
    """Column sums of integer terms onto an integer prefill are exact in fp32 in any order: every partial sum is an integer
    of magnitude below 2^24."""
    t, p = terms.double(), prefill.double()
    return bool((t == t.round()).all() and (p == p.round()).all() and
                float((t.abs().sum(0) + p.abs()).max()) < 2 ** 24)


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
def _first_bad(bad: torch.Tensor, what: str, got, ref, E, extra=""):
    n = int(bad.sum())
    if n:
        idx = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements differ; first at {idx}: got {float(got[idx])!r}, "
                             f"float64 {float(ref[idx])!r} +- {float(E[idx]):.3g}{extra}")


def check_f32(got: torch.Tensor, ref: torch.Tensor, E: torch.Tensor, what: str) -> float:
    """|got - ref| <= E element by element.  Returns the worst |got - ref| / E."""
    g = got.to(ref.device).double()
    E = E.double() + TINY
    bad = ~((g - ref).abs() <= E)  # NaN is bad
    _first_bad(bad, what, g, ref, E)
    return float(((g - ref).abs() / E).max()) if g.numel() else 0.0


def check_bf16(got: torch.Tensor, ref: torch.Tensor, E: torch.Tensor, what: str) -> int:
    """got (bf16) in [bf16_rn(ref - E), bf16_rn(ref + E)].  Returns how many elements differ from bf16_rn(ref)."""
    g = got.to(ref.device).double()
    E = E.double() + TINY
    lo, hi = bf16_rn(ref - E), bf16_rn(ref + E)
    bad = ~((g >= lo) & (g <= hi))
    _first_bad(bad, what, g, ref, E)
    return int((g != bf16_rn(ref)).sum())


def check_out(got: torch.Tensor, ref: torch.Tensor, E: torch.Tensor, what: str):
    return check_bf16(got, ref, E, what) if got.dtype == torch.bfloat16 else check_f32(got, ref, E, what)


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm forward
# ---------------------------------------------------------------------------------------------------------------------
def ln_fwd_ref(x, gamma, beta, eps=EPS, unbiased=False):
    """float64 (y, mean, rstd) of utils/model_utils.py:113-130; eps taken as the float32 the kernel is given.  unbiased:
    the doctored variance with divisor H - 1 (for the tests that show the checks reject it)."""
    x = x.double()
    H = x.shape[-1]
    mean = x.mean(-1)
    d = x - mean[:, None]
    var = (d * d).sum(-1) / (H - 1 if unbiased else H)
    rstd = 1.0 / torch.sqrt(var + eps32(eps))
    y = d * rstd[:, None] * gamma.double() + beta.double()
    return y, mean, rstd


def ln_fwd_bounds(x, gamma, beta, eps=EPS, scale: float = 1.0):
    """Per-row bounds E_mean, E_rstd on the kernel's mean_out and rstd_out and the per-element bound E_y on y (before the
    output rounding), following ln_fwd_kernel's fp32 operations:
      S = sum x (lane chains + butterfly): E_S = sum_depth u sum|x|, 0 where x are integers with sum|x| < 2^24 (exact);
      mean = fl(S / H): E_mean = E_S / H (1 + u) + u |mu|;
      d = fl(x - mean), sq = sum d^2: with e = mean - mu, sum (D - e)^2 = sum D^2 + H e^2 (sum D = 0), and each term carries
      3 roundings (subtraction twice, product) before the chain: E_sq = H E_mean^2 + (sum_depth + 3) u (sum D^2 + H E_mean^2);
      var = fl(sq / H), t = fl(var + eps), rstd = rsqrtf(t): with eta = E_t / (V + eps), |rstd - r| <= r (eta / 2 /
      (1 - eta)^1.5 + 4u);
      s = fl(rstd g); y = x s - mean s + b in up to three roundings, possibly contracted:
      E_y = |g| (|D| E_rstd + rstd_hi E_mean) + u (|D| + E_mean) |s| + 3u (|x s| + (|mu| + E_mean) |s| + |b|);
      dropout (scale != 1): E_y scale + u |y scale|.
    Returns (E_mean, E_rstd, E_y)."""
    x64, g, b = x.double(), gamma.double(), beta.double()
    H = x64.shape[-1]
    k = sum_depth(H)
    absx = x64.abs().sum(-1)
    exact_sum = (x64 == x64.round()).all(-1) & (absx < 2 ** 24)
    E_S = torch.where(exact_sum, torch.zeros_like(absx), k * U * absx)
    mu = x64.mean(-1)
    E_mean = E_S / H * (1 + U) + U * mu.abs()
    D = x64 - mu[:, None]
    sumD2 = (D * D).sum(-1)
    V = sumD2 / H
    E_sq = H * E_mean ** 2 + (k + 3) * U * (sumD2 + H * E_mean ** 2)
    E_var = E_sq / H + U * (V + E_sq / H)
    e = eps32(eps)
    E_t = E_var + U * (V + e + E_var)
    eta = (E_t / (V + e)).clamp(max=0.5)
    r = 1.0 / torch.sqrt(V + e)
    E_rstd = SLACK * r * (0.5 * eta / (1 - eta) ** 1.5 + RSQRT_REL)
    r_hi = (r + E_rstd)[:, None]
    s_abs = r_hi * g.abs() * (1 + U)
    Em = E_mean[:, None]
    E_y = SLACK * (g.abs() * (D.abs() * E_rstd[:, None] + r_hi * Em) + U * (D.abs() + Em) * s_abs
                   + 3 * U * (x64.abs() * s_abs + (mu.abs()[:, None] + Em) * s_abs + b.abs()))
    if scale != 1.0:
        y = D * r[:, None] * g + b
        E_y = E_y * scale + SLACK * U * (y.abs() + E_y) * scale
    return E_mean, E_rstd, E_y


def exact_stats_rows(x) -> torch.Tensor:
    """bool [rows]: rows of integers whose mean is an integer and whose sums of |x| and (x - mean)^2 stay below 2^24 -- every
    fp32 sum the kernel forms on them is exact (zero_sum, constant and zero rows)."""
    x64 = x.double()
    H = x64.shape[-1]
    S = x64.sum(-1)
    mean = S / H
    d = x64 - mean[:, None]
    return ((x64 == x64.round()).all(-1) & (mean == mean.round()) & (x64.abs().sum(-1) < 2 ** 24)
            & ((d * d).sum(-1) < 2 ** 24))


def check_exact_stats(mean_out, rstd_out, x, eps=EPS, what="ln stats") -> int:
    """On exact_stats_rows: mean_out == sum / H bit for bit and rstd_out within 2 ulp of 1 / sqrt(fp32(var32 + eps)), var32 =
    fp32(sum (x - mean)^2 / H) (one IEEE division of exact integers).  Returns the number of rows checked."""
    rows = exact_stats_rows(x.cpu())
    if not bool(rows.any()):
        return 0
    x64 = x.cpu().double()
    H = x64.shape[-1]
    mean = x64.sum(-1) / H
    sq = ((x64 - mean[:, None]) ** 2).sum(-1).numpy().astype(np.float32)  # exact integers below 2^24 on the exact rows
    var32 = sq / np.float32(H)
    t32 = (var32 + np.float32(eps)).astype(np.float32)
    want = torch.from_numpy(1.0 / np.sqrt(t32.astype(np.float64)))
    got_mean, got = mean_out.cpu().double(), rstd_out.cpu().double()
    _first_bad(rows & (got_mean != mean), f"{what}: mean of exact rows", got_mean, mean, torch.zeros_like(mean))
    _, e = torch.frexp(want)
    ulp2 = torch.ldexp(torch.ones_like(want), e - 23)
    _first_bad(rows & ~((got - want).abs() <= ulp2), f"{what}: rstd of exact rows (2 ulp)", got, want, ulp2)
    return int(rows.sum())


def check_ln_fwd(y, mean_out, rstd_out, x, gamma, beta, eps=EPS, keep=None, scale: float = 1.0, what="ln fwd",
                 unbiased_ref=False, ref_eps=None):
    """Every output of one merlot_layernorm_fwd against float64: the exact statistics of exact rows, mean_out and rstd_out
    per row, y per element (y: the logical rows, [rows, H]; keep: the dropout mask as bool or {0, 1}, or None).
    unbiased_ref / ref_eps doctor the REFERENCE (the wrong-reference tests); the bounds stay those of the kernel."""
    dev = y.device
    xd, gd, bd = x.to(dev), gamma.to(dev), beta.to(dev)
    ref_y, ref_mean, ref_rstd = ln_fwd_ref(xd, gd, bd, eps if ref_eps is None else ref_eps, unbiased=unbiased_ref)
    E_mean, E_rstd, E_y = ln_fwd_bounds(xd, gd, bd, eps, scale)
    if mean_out is not None:
        if not unbiased_ref and ref_eps is None:
            check_exact_stats(mean_out, rstd_out, x, eps, what)
        check_f32(mean_out, ref_mean, E_mean, f"{what}: mean")
        check_f32(rstd_out, ref_rstd, E_rstd, f"{what}: rstd")
    if keep is not None:
        kd = keep.to(dev).double()
        ref_y = ref_y * kd * float(np.float32(scale))
        E_y = E_y * kd
    return check_out(y, ref_y, E_y, f"{what}: y")


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm backward (both kernels)
# ---------------------------------------------------------------------------------------------------------------------
def ln_bwd_ref(dy, x, mean, rstd, gamma, dres=None, keep=None, scale: float = 1.0):
    """float64 dx [rows, H] and the column terms (dv * xhat, dv) of dgamma / dbeta, with the kernel's fp32 mean and rstd as
    inputs.  dy: the logical rows (already read through any row remap); keep: the forward dropout mask re-applied to dy."""
    dv = dy.double()
    if keep is not None:
        dv = dv * keep.double() * float(np.float32(scale))
    mu, rs, g = mean.double()[:, None], rstd.double()[:, None], gamma.double()
    xh = (x.double() - mu) * rs
    gd = g * dv
    H = x.shape[-1]
    s1 = gd.sum(-1, keepdim=True) / H
    s2 = (gd * xh).sum(-1, keepdim=True) / H
    dx = rs * (gd - s1 - xh * s2)
    if dres is not None:
        dx = dx + dres.double()
    return dx, dv * xh, dv


def ln_bwd_bounds(dy, x, mean, rstd, gamma, dres=None, keep=None, scale: float = 1.0):
    """Per-element bound E_dx (before the output rounding) and the per-term errors of the column terms, following
    ln_bwd_kernel / ln_bwd_fused_kernel:
      dv = fl(dy keep scale): E_dv = u |dv| where scale != 1;  xh = fl(fl(x - mean) rstd): E_xh = 2u |xhat|;
      gd = fl(g dv): E_gd = |g| E_dv + u |GD|;
      s1 = sum gd / H: (sum_depth u sum|GD| + sum E_gd) / H, then 2u for the division (fl(1/H) times the sum in the fused
      kernel);  s2 = sum gd xh / H: the terms carry |GD| E_xh + |xhat| E_gd + u |GD xhat| (the product rounding, none when
      contracted), the chain sum_depth u sum|GD xhat|, then 2u;
      o = rstd (gd - s1 - xh s2) (+ dres): the propagated errors times rstd, 3u |rstd| (|GD| + |S1| + |xhat S2|) for the
      product and the two subtractions, u (|rstd inner| + |dres|) for the residual add.
    Returns (E_dx, E_dg_terms, E_db_terms)."""
    dv = dy.double()
    if keep is not None:
        dv = dv * keep.double() * float(np.float32(scale))
    E_dv = U * dv.abs() if scale != 1.0 else torch.zeros_like(dv)
    mu, rs, g = mean.double()[:, None], rstd.double()[:, None], gamma.double()
    H = x.shape[-1]
    k = sum_depth(H)
    xh = (x.double() - mu) * rs
    E_xh = 2 * U * xh.abs()
    gd = g * dv
    E_gd = g.abs() * E_dv + U * gd.abs()
    E_s1sum = k * U * gd.abs().sum(-1, keepdim=True) + E_gd.sum(-1, keepdim=True)
    s1 = gd.sum(-1, keepdim=True) / H
    E_s1 = E_s1sum / H + 2 * U * (s1.abs() + E_s1sum / H)
    p = gd * xh
    E_s2sum = (gd.abs() * E_xh + xh.abs() * E_gd + U * p.abs()).sum(-1, keepdim=True) + k * U * p.abs().sum(-1, keepdim=True)
    s2 = p.sum(-1, keepdim=True) / H
    E_s2 = E_s2sum / H + 2 * U * (s2.abs() + E_s2sum / H)
    A = gd.abs() + s1.abs() + (xh * s2).abs()
    E_dx = rs.abs() * (E_gd + E_s1 + xh.abs() * E_s2 + s2.abs() * E_xh + 3 * U * A) + U * rs.abs() * A
    if dres is not None:
        E_dx = E_dx + U * dres.double().abs()
    E_dg = dv.abs() * E_xh + xh.abs() * E_dv + U * (dv * xh).abs()
    return SLACK * E_dx, SLACK * E_dg, E_dv


def col_ref_bound(terms, term_err, prefill, depth: int, launches: int = 1):
    """A column sum over rows, `launches` times onto `prefill`: (float64 reference, bound depth u (|prefill| + sum|terms|)
    + sum term_err)."""
    P = prefill.double().to(terms.device)
    ref = P + launches * terms.sum(0)
    E = SLACK * (depth * U * (P.abs() + launches * terms.abs().sum(0)) + launches * term_err.sum(0))
    return ref, E
