"""Element-by-element references for the hybrid stem's K13 kernels (merlot_b200/csrc/stem.cu).  Test infrastructure only;
every function runs on the CPU or, for large shapes, on the GPU in float64 (plain torch).

The formulas restate utils/vision_transformer.py:8-170 and utils/model_utils.py:133-222: GroupNorm with the ONE-PASS moments
(mean = sum/n, var = sum(x^2)/n - mean^2, eps 1e-4), weight standardisation per output channel over (kh, kw, cin) with the
biased two-pass variance and eps 1e-5, avg-pool 2x2 SAME (padding not counted), 3x3 im2col with one ring of zero padding.

Exact inputs.  dyadic() draws x = k * delta with small integers k (exact in bf16).  When a sum of n such values satisfies
    n * max|k| < 2^24   and   n * max k^2 < 2^24                                         (exact_sums_hold)
every fp32 partial sum of x and of x^2 is an integer multiple of delta (delta^2) below 2^24 of them, hence exact, in ANY
order: the per-thread chains, the shared-memory atomics and the global atomics of gn_stats give the float64 sums bit for bit.
The same holds for the <= 9 (col2im) and <= 4 (avg-pool) term sums, whose 1/cnt is a power of two.

Bounds.  Where a result is not exact, the check is per element: |kernel - float64| <= E, where E follows the kernel's own
arithmetic with u = 2^-24 per fp32 rounding, 2 ulp (4u relative) for rsqrtf, and for every sum the LONGEST chain of additions
the launch has (gn_geometry: rows per thread + the lanes meeting in shared memory + the blocks meeting in global memory), not
n * u.  A bf16 output is then accepted iff it lies between bf16_rn(ref - E) and bf16_rn(ref + E) (pushed through the
kernel's remaining exact steps): where ref is not within E of a bf16 rounding midpoint that interval holds ONE value, the
correctly rounded one; elsewhere it admits the neighbour, and the checkers count those elements.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24          # fp32 unit roundoff
RSQRT_REL = 4 * U       # rsqrtf: 2 ulp
GN_EPS, WS_EPS = 1e-4, 1e-5
GN_THREADS = 256
WS_WARPS = 32
TINY = 2.0 ** -140      # absolute floor of every bound (fp32 subnormal products)


# ---------------------------------------------------------------------------------------------------------------------
# launch geometry and exact inputs
# ---------------------------------------------------------------------------------------------------------------------
def gn_geometry(HW: int, C: int) -> dict:
    """The grid merlot_group_norm_fwd / _bwd launch for their reductions: lanes = rows in flight per block, rows_per_block,
    blocks per sample and the rows one thread sums on its own."""
    c8n = C // 8
    lanes = max(1, GN_THREADS // c8n)
    rpb = min(HW, lanes * 32)
    return dict(c8n=c8n, lanes=lanes, rows_per_block=rpb, blocks=-(-HW // rpb), rows_per_thread=-(-rpb // lanes))


def exact_sums_hold(n: int, kmax: int) -> bool:
    """Every partial sum of n values k*delta and of their squares, |k| <= kmax, is exact in fp32."""
    return kmax <= 256 and n * kmax < 2 ** 24 and n * kmax * kmax < 2 ** 24


def max_k(n: int) -> int:
    """The largest |k| for which n-term sums of k*delta and (k*delta)^2 are exact in fp32 (at most 16)."""
    k = min(16, int(math.isqrt((2 ** 24 - 1) // n)))
    assert k >= 1 and exact_sums_hold(n, k), n
    return k


def dyadic(shape, kmax: int, delta: float, seed: int, center: int = 0, device="cpu") -> torch.Tensor:
    """bf16 tensor of (center + k) * delta, k uniform in [-kmax, kmax]; delta a power of two."""
    assert math.frexp(delta)[0] == 0.5 and abs(center) + kmax <= 256
    g = torch.Generator().manual_seed(int(seed))
    k = torch.randint(-kmax, kmax + 1, tuple(shape), generator=g) + center
    return (k.double() * delta).to(torch.bfloat16).to(device)


def assert_exact_grid(x: torch.Tensor, n: int, delta: float):
    """Asserts the exactness condition for n-term sums of the values of x (multiples of delta)."""
    k = x.double() / delta
    assert bool((k == k.round()).all()), "not on the grid"
    kmax = int(k.abs().max())
    assert exact_sums_hold(n, kmax), (n, kmax)


def bf16_rn(x: torch.Tensor) -> torch.Tensor:
    """float64 -> the nearest bf16 value (ties to even) in ONE rounding, as float64.  (torch's double -> bf16 cast rounds
    through float32 first, which can round twice.)"""
    m, e = torch.frexp(x.double())
    return torch.ldexp(torch.round(torch.ldexp(m, torch.full_like(e, 8))), e - 8)


def bf16_ulps(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Distance in bf16 ulps between bf16 values (any float dtype), sign-magnitude order."""
    def order(t):
        bits = (t.float().contiguous().view(torch.int32) >> 16).long()
        return torch.where(bits & 0x8000 != 0, -(bits & 0x7FFF), bits & 0x7FFF)
    return (order(a) - order(b)).abs()


def exact_check(got: torch.Tensor, want: torch.Tensor, what: str):
    """Bitwise equality of the values (want may be float64 holding exact values of got's dtype)."""
    g, w = got.double(), want.double().to(got.device)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = (g != w) & ~(g.isnan() & w.isnan())  # a NaN differs from everything but a NaN
    n = int(bad.sum())
    if n:
        idx = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} of {g.numel()} elements differ; first at {idx}: got {float(g[idx])!r}, "
                             f"want {float(w[idx])!r}")


def interval_check(got: torch.Tensor, ref: torch.Tensor, E: torch.Tensor, what: str, finish=None) -> int:
    """got (bf16) must lie in [finish(bf16_rn(ref - E)), finish(bf16_rn(ref + E))]; finish, monotone, replays the kernel's
    exact steps after the rounding (shortcut add, ReLU, final rounding).  Returns how many elements differ from the
    correctly rounded finish(bf16_rn(ref)), i.e. sit next to a rounding midpoint."""
    finish = finish or (lambda v: v)
    ref, E = ref.double(), E.double() + TINY
    g = got.double().to(ref.device)
    assert bool(torch.isfinite(g).all()), f"{what}: {int((~torch.isfinite(g)).sum())} non-finite elements"
    lo, hi, mid = finish(bf16_rn(ref - E)), finish(bf16_rn(ref + E)), finish(bf16_rn(ref))
    bad = (g < lo) | (g > hi)
    n = int(bad.sum())
    if n:
        idx = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} of {g.numel()} elements outside the bound; first at {idx}: got {float(g[idx])!r}, "
                             f"float64 {float(ref[idx])!r} +- {float(E[idx]):.3g}, allowed [{float(lo[idx])!r}, {float(hi[idx])!r}]")
    return int((g != mid).sum())


def bound_check(got: torch.Tensor, ref: torch.Tensor, E: torch.Tensor, what: str) -> float:
    """|got - ref| <= E element by element (fp32 results).  Returns the worst err / bound."""
    g, ref = got.double().to(ref.device), ref.double()
    assert bool(torch.isfinite(g).all()), f"{what}: non-finite elements"
    ratio = (g - ref).abs() / (E.double() + TINY)
    i = int(ratio.argmax())
    idx = tuple(int(j) for j in np.unravel_index(i, tuple(ratio.shape)))
    worst = float(ratio.reshape(-1)[i])
    assert worst <= 1.0, (f"{what}: element {idx}: got {float(g[idx])!r}, float64 {float(ref[idx])!r}, {worst:.3g} x the "
                          f"bound {float(E[idx]):.3g}")
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm (+ReLU, +shortcut): forward
# ---------------------------------------------------------------------------------------------------------------------
def gn_sums(x: torch.Tensor, N: int, HW: int, C: int, groups: int) -> torch.Tensor:
    """float64 [N, groups, 2]: per (sample, group) sum of x and sum of x^2 -- the layout of the kernels' stats buffer."""
    x = x.double().reshape(N, HW, groups, C // groups)
    return torch.stack((x.sum((1, 3)), (x * x).sum((1, 3))), -1)


def _gn_moments(stats, N, HW, C, groups, eps):
    """Moments from the sums the kernels read (stats, [N * groups * 2]) and the fp32 error of their own evaluation:
    mean = fl(s fl(1/n)), var = fl(q fl(1/n)) - fl(mean^2), t = var + eps, rstd = rsqrtf(t).  Per channel, [N, 1, C]."""
    cg = C // groups
    n = HW * cg
    st = stats.double().reshape(N, groups, 2)
    mu, q = st[..., 0] / n, st[..., 1] / n
    t = q - mu * mu + eps
    assert bool((t > 0).all()), "var + eps <= 0: rsqrt of a negative number"
    em = 2.01 * U * mu.abs()
    dt = 8 * U * q.abs() + 1.01 * U * ((q - mu * mu).abs() + t)
    assert bool((dt < t / 2).all())
    rel_r = dt / (2 * (t - dt)) + RSQRT_REL + U
    ch = lambda v: v.repeat_interleave(cg, dim=1).reshape(N, 1, C)
    return ch(mu), ch(1 / t.sqrt()), ch(em), ch(rel_r)


def _xhat(x, mu, r, em, rel_r):
    """xhat = (x - mean) * rstd in float64 and the bound on fl(fl(x - mean) * rstd) - xhat."""
    d = x - mu
    return d * r, r * (em + 1.01 * U * d.abs()) + d.abs() * r * (rel_r + 1.01 * U)


def gn_fwd_ref(x, stats, gamma, beta, N, HW, C, groups=32, eps=GN_EPS):
    """float64 GroupNorm output from the sums in `stats`, and the bound on the kernel's fp32 evaluation
    fl(fl(fl(x - mean) rstd) gamma) + beta (each step rounded, or fused).  x: [N * HW, C]; returns [N, HW, C] pair."""
    x = x.double().reshape(N, HW, C)
    mu, r, em, rel_r = _gn_moments(stats, N, HW, C, groups, eps)
    xh, exh = _xhat(x, mu, r, em, rel_r)
    gm, bt = gamma.double().to(x.device), beta.double().to(x.device)
    o = xh * gm + bt
    E = 1.001 * (exh * gm.abs() + U * (xh * gm).abs()) + 1.01 * U * (o.abs() + bt.abs())
    return o, E


def gn_finish(shortcut, relu: bool):
    """The kernel's steps after the fp32 GroupNorm value o (monotone in o): without a shortcut relu(o) rounded to bf16;
    with one, relu(fl32(bf16(o) + shortcut)) rounded to bf16 (bottleneck_block :96 adds two bf16 tensors)."""
    def finish(v):
        if shortcut is not None:
            v = (v.float() + shortcut.float().reshape(v.shape).to(v.device)).double()  # one fp32 rounding
            v = bf16_rn(v.clamp(min=0) if relu else v)
            return v
        return v.clamp(min=0) if relu else v
    return finish


def rounding_sensitive_shortcut(o: torch.Tensor, seed: int) -> torch.Tensor:
    """A bf16 shortcut for GroupNorm output o (float64): on every other element -bf16_rn(o), so that bf16(o) + shortcut is
    exactly 0 while o + shortcut keeps o's rounding error (which survives the ReLU where positive); elsewhere small dyadic
    values.  A kernel that skips the bf16 rounding before the add fails on about a quarter of the elements."""
    base = dyadic(o.shape, 16, 2.0 ** -4, seed, device=o.device).double()
    alt = (torch.arange(o.numel(), device=o.device).reshape(o.shape) % 2) == 0
    return torch.where(alt, -bf16_rn(o), base).to(torch.bfloat16).reshape(-1, o.shape[-1])


def check_gn_stats(stats, x, N, HW, C, groups=32, what="gn stats"):
    """stats must hold the float64 sums bit for bit (exact inputs: assert_exact_grid first)."""
    exact_check(stats.reshape(N, groups, 2), gn_sums(x, N, HW, C, groups), what)


def check_gn_stats_bound(stats, x, N, HW, C, groups=32, what="gn stats"):
    """Inexact inputs: per (sample, group) |stats - sum| <= L u sum|terms|, L the longest chain of the launch."""
    geo = gn_geometry(HW, C)
    cg = C // groups
    L = geo["rows_per_thread"] + geo["lanes"] * cg + geo["blocks"] + 2
    ref = gn_sums(x, N, HW, C, groups)
    mag = gn_sums(x.double().abs(), N, HW, C, groups)
    return bound_check(stats.reshape(N, groups, 2), ref, 1.01 * L * U * mag, what)


def check_gn_fwd(y, x, stats, gamma, beta, N, HW, C, groups=32, eps=GN_EPS, relu=True, shortcut=None, what="gn fwd"):
    """y (bf16 [N * HW, C]) against the float64 formula from the sums in stats; returns the count of midpoint elements."""
    o, E = gn_fwd_ref(x, stats, gamma, beta, N, HW, C, groups, eps)
    sc = None if shortcut is None else shortcut.reshape(N, HW, C)
    return interval_check(y.reshape(N, HW, C), o, E, what, gn_finish(sc, relu))


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm backward
# ---------------------------------------------------------------------------------------------------------------------
def gn_bwd_ref(dy, x, y, stats, gamma, N, HW, C, groups=32, eps=GN_EPS, relu=True):
    """float64 gradients of GroupNorm(+ReLU/+shortcut) with the moments of `stats`, g = dy [y > 0] (the kernel's mask), and
    the bound of each fp32 result.  Per channel: dbeta = sum g, dgamma = sum g xhat; per (sample, group): S1 = sum g gamma,
    S2 = sum g gamma xhat (the `red` buffer); dx = rstd (g gamma - S1/n - xhat S2/n); dshortcut = g."""
    dev = x.device
    x = x.double().reshape(N, HW, C)
    g = dy.double().reshape(N, HW, C).to(dev)
    if relu:
        g = torch.where(y.reshape(N, HW, C).to(dev).float() > 0, g, torch.zeros((), dtype=g.dtype, device=dev))
    geo = gn_geometry(HW, C)
    cg, n = C // groups, HW * C // groups
    mu, r, em, rel_r = _gn_moments(stats, N, HW, C, groups, eps)
    xh, exh = _xhat(x, mu, r, em, rel_r)
    gm = gamma.double().to(dev)
    gg = g * gm
    grp = lambda t: t.reshape(N, HW, groups, cg).sum((1, 3))             # [N, groups]
    per = lambda t: t.repeat_interleave(cg, dim=1).reshape(N, 1, C) / n  # per channel, divided by n
    L_c = geo["rows_per_thread"] + geo["lanes"] + N * geo["blocks"] + 2   # dgamma / dbeta: thread, shared, global (+ start)
    L_g = geo["rows_per_thread"] + geo["lanes"] * cg + geo["blocks"] + 2  # red: the group's channels meet in shared memory
    S1, S2 = grp(gg), grp(gg * xh)
    E_S1 = 1.01 * L_g * U * grp(gg.abs()) + U * grp(gg.abs())
    E_S2 = grp(gg.abs() * exh) + 1.01 * (L_g + 2) * U * grp((gg * xh).abs())
    dbeta, dgamma = g.sum((0, 1)), (g * xh).sum((0, 1))
    E_db = 1.01 * L_c * U * g.abs().sum((0, 1))
    E_dg = (g.abs() * exh).sum((0, 1)) + 1.01 * (L_c + 1) * U * (g * xh).abs().sum((0, 1))
    b, c = per(S1), xh * per(S2)
    inner = gg - b - c
    e_in = (per(E_S1) + 2.01 * U * b.abs() + exh * per(S2).abs() + xh.abs() * (per(E_S2) + 2.01 * U * per(S2).abs())
            + 3.02 * U * (gg.abs() + b.abs() + c.abs()))
    dx = r * inner
    E_dx = 1.001 * (r * e_in + dx.abs() * (rel_r + 1.01 * U))
    return dict(g=g, S1=S1, S2=S2, E_S1=E_S1, E_S2=E_S2, dbeta=dbeta, E_db=E_db, dgamma=dgamma, E_dg=E_dg, dx=dx, E_dx=E_dx)


def check_gn_bwd(out: dict, dy, x, y, stats, gamma, N, HW, C, groups=32, eps=GN_EPS, relu=True, exact=False, dgamma0=None,
                 dbeta0=None, what="gn bwd") -> int:
    """out: kernel results dx, dshortcut (or None), dgamma, dbeta (accumulated onto dgamma0 / dbeta0), red (or None).
    exact: dy dyadic and gamma powers of two with exact sums -> dbeta and S1 bitwise.  Returns the dx midpoint count."""
    R = gn_bwd_ref(dy, x, y, stats, gamma, N, HW, C, groups, eps, relu)
    dev = R["g"].device
    z = lambda t: torch.zeros(C, dtype=torch.float64, device=dev) if t is None else t.double().to(dev)
    dg0, db0 = z(dgamma0), z(dbeta0)
    if out.get("dshortcut") is not None:
        exact_check(out["dshortcut"].reshape(N, HW, C), R["g"], f"{what}: dshortcut")
    if exact:
        exact_check(out["dbeta"], db0 + R["dbeta"], f"{what}: dbeta")
        if out.get("red") is not None:
            exact_check(out["red"].reshape(N, groups, 2)[..., 0], R["S1"], f"{what}: S1")
    else:
        bound_check(out["dbeta"], db0 + R["dbeta"], R["E_db"] + U * (db0 + R["dbeta"]).abs(), f"{what}: dbeta")
        if out.get("red") is not None:
            bound_check(out["red"].reshape(N, groups, 2)[..., 0], R["S1"], R["E_S1"], f"{what}: S1")
    if out.get("red") is not None:
        bound_check(out["red"].reshape(N, groups, 2)[..., 1], R["S2"], R["E_S2"], f"{what}: S2")
    bound_check(out["dgamma"], dg0 + R["dgamma"], R["E_dg"] + 1.01 * U * (dg0 + R["dgamma"]).abs(), f"{what}: dgamma")
    return interval_check(out["dx"].reshape(N, HW, C), R["dx"], R["E_dx"], f"{what}: dx")


# ---------------------------------------------------------------------------------------------------------------------
# im2col / col2im / avg-pool
# ---------------------------------------------------------------------------------------------------------------------
def conv_out(h: int, w: int, stride: int):
    return (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1


def im2col_ref(x, N, h, w, C, stride, ld, sub_half=False) -> torch.Tensor:
    """bf16 [N*ho*wo, ld]: columns (ky, kx, c) of the zero-padded map, columns [9C, ld) zero; sub_half subtracts 0.5 from
    the image (one bf16 rounding) and leaves the padding ring 0 (vision_transformer.py:193 normalises before padding)."""
    ho, wo = conv_out(h, w, stride)
    xv = x.float().reshape(N, h, w, C)
    if sub_half:
        xv = (xv - 0.5).bfloat16().float()
    xp = torch.zeros(N, h + 2, w + 2, C, dtype=torch.float32, device=x.device)
    xp[:, 1:h + 1, 1:w + 1] = xv
    taps = [xp[:, ky:ky + (ho - 1) * stride + 1:stride, kx:kx + (wo - 1) * stride + 1:stride] for ky in range(3) for kx in range(3)]
    out = torch.zeros(N * ho * wo, ld, dtype=torch.float32, device=x.device)
    out[:, :9 * C] = torch.stack(taps, 3).reshape(N * ho * wo, 9 * C)
    return out.bfloat16()


def col2im_ref(dcol, N, h, w, C, stride):
    """float64 [N*h*w, C]: the adjoint of im2col (scatter-add of the 9 taps), and the sum of the magnitudes of the terms."""
    ho, wo = conv_out(h, w, stride)
    d4 = dcol[:, :9 * C].double().reshape(N, ho, wo, 9, C)
    out = torch.zeros(N, h + 2, w + 2, C, dtype=torch.float64, device=dcol.device)
    mag = torch.zeros_like(out)
    for t in range(9):
        ky, kx = t // 3, t % 3
        out[:, ky:ky + (ho - 1) * stride + 1:stride, kx:kx + (wo - 1) * stride + 1:stride] += d4[:, :, :, t]
        mag[:, ky:ky + (ho - 1) * stride + 1:stride, kx:kx + (wo - 1) * stride + 1:stride] += d4[:, :, :, t].abs()
    crop = lambda t: t[:, 1:h + 1, 1:w + 1].reshape(N * h * w, C)
    return crop(out), crop(mag)


def pool_counts(h, w, device="cpu"):
    """[ho, wo] number of valid pixels of each 2x2 SAME window (bottom / right cells of odd maps hold fewer)."""
    ho, wo = (h + 1) // 2, (w + 1) // 2
    cy = torch.tensor([min(2, h - 2 * i) for i in range(ho)], dtype=torch.float64, device=device)
    cx = torch.tensor([min(2, w - 2 * i) for i in range(wo)], dtype=torch.float64, device=device)
    return cy[:, None] * cx[None, :]


def avgpool_ref(x, N, h, w, C):
    """float64 [N*ho*wo, C] 2x2 SAME average (padding not counted) and the mean of the magnitudes."""
    ho, wo = (h + 1) // 2, (w + 1) // 2
    xp = torch.zeros(N, 2 * ho, 2 * wo, C, dtype=torch.float64, device=x.device)
    xp[:, :h, :w] = x.double().reshape(N, h, w, C)
    cnt = pool_counts(h, w, x.device)[None, :, :, None]
    s = xp.reshape(N, ho, 2, wo, 2, C).sum((2, 4)) / cnt
    m = xp.abs().reshape(N, ho, 2, wo, 2, C).sum((2, 4)) / cnt
    return s.reshape(-1, C), m.reshape(-1, C)


def avgpool_bwd_ref(dy, N, h, w, C):
    """float64 [N*h*w, C]: each input pixel receives dy of its window / the window's count (exact: powers of two)."""
    ho, wo = (h + 1) // 2, (w + 1) // 2
    d = dy.double().reshape(N, ho, wo, C) / pool_counts(h, w, dy.device)[None, :, :, None]
    d = d.repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :h, :w]
    return d.reshape(N * h * w, C)


def wgrad_exact(a, dy, init) -> torch.Tensor:
    """init + a^T dy in float64 (exact for integer operands and integer init below 2^53): the conv wgrad HybridStem.backward
    accumulates into its fp32 gradient arena, a the [pixels, kp] im2col (or activation) matrix, dy [pixels, cout]."""
    return init.double() + a.double().t() @ dy.double()


# ---------------------------------------------------------------------------------------------------------------------
# weight standardisation
# ---------------------------------------------------------------------------------------------------------------------
def _ws_moments(w):
    """float64 per-channel mean / rstd of w [rows, cout] and the bounds of the kernel's fp32 moments: each warp chains
    ceil(rows / 32) rows, then the 32 warp sums are added in shared memory, then one division."""
    rows = w.shape[0]
    L = -(-rows // WS_WARPS) + WS_WARPS + 1
    mu = w.mean(0, keepdim=True)
    d = w - mu
    var = (d * d).mean(0, keepdim=True)
    em = 1.01 * L * U * w.abs().mean(0, keepdim=True) + U * mu.abs()
    ev = ((2 * d.abs() * em + 3.02 * U * d * d).mean(0, keepdim=True) + 1.01 * L * U * var + 1.01 * U * var
          + em * em)
    t = var + WS_EPS
    rel_r = ev / (2 * (t - ev)) + RSQRT_REL + 1.01 * U
    r = 1 / t.sqrt()
    wh = d * r
    ewh = r * (em + 1.01 * U * d.abs()) + d.abs() * r * (rel_r + 1.01 * U)
    return L, r, rel_r, wh, ewh


def ws_ref(w):
    """float64 standardised kernel (w - mean) / sqrt(var + 1e-5) of w [rows, cout] and the bound of the kernel's fp32 value
    before its bf16 rounding."""
    w = w.double()
    _, _, _, wh, ewh = _ws_moments(w)
    return wh, 1.001 * ewh


def ws_bwd_ref(dws, w, dw0):
    """float64 dw0 + rstd (dws - mean(dws) - what mean(dws what)) and its bound (fp32 chains as in _ws_moments)."""
    w, dws, dw0 = w.double(), dws.double(), dw0.double()
    L, r, rel_r, wh, ewh = _ws_moments(w)
    m1, m2 = dws.mean(0, keepdim=True), (dws * wh).mean(0, keepdim=True)
    e1 = 1.01 * L * U * dws.abs().mean(0, keepdim=True) + U * m1.abs()
    e2 = (dws.abs() * (ewh + 1.01 * U * wh.abs())).mean(0, keepdim=True) + 1.01 * L * U * (dws * wh).abs().mean(0, keepdim=True) + U * m2.abs()
    inner = dws - m1 - wh * m2
    e_in = e1 + ewh * m2.abs() + wh.abs() * e2 + 3.02 * U * (dws.abs() + m1.abs() + (wh * m2).abs())
    g = r * inner
    out = dw0 + g
    E = 1.001 * (r * e_in + g.abs() * (rel_r + 1.01 * U)) + 1.01 * U * out.abs()
    return out, E
