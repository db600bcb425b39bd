"""ORACLE -- TEST INFRASTRUCTURE ONLY.  A vectorised float32 restatement of the per-pixel half of the frame input: the TF 1.15
legacy resize kernels that `tf.image.resize_images(..., align_corners=True)` runs (tensorflow/core/kernels/
resize_bilinear_op.cc, resize_nearest_neighbor_op.cc, resize_bicubic_op.cc, resize_area_op.cc, image_resizer_state.h), the
crop and pad of resize_and_pad (utils/model_utils.py:855-940) and lightweight_image_augment's brightness and contrast
(:758-835), at the sizes the pipelines run.

Written from those sources, like tests/input_oracle.py, and not from csrc/frames.cu.  Each output pixel follows the source's
operation order exactly: one np.float32 rounding per operation, no fused multiply-add, taps visited one at a time in the
source's order.  Only the loop over output pixels is vectorised: every array operation below is elementwise across pixels.
Area's variable-length tap loops become masked loops over the tap index (np.where keeps a pixel's running sum once its own
taps are done), so no pixel's sum is reassociated.  Only the pixels inside the crop window are resized; each one depends on
its own coordinates alone, so this equals resizing the whole image and cropping.

The contrast transform takes its per-channel mean as an argument: TensorFlow leaves the order of that float32 sum open, so a
test supplies the mean it wants to check against (the kernel's own, or the float64 mean of padded_mean)."""
import numpy as np

from oracle.oracle_np import bf16_round  # noqa: F401  (part of this module's interface)

F = np.float32
INV255 = F(1.0 / 255.0)  # convert_image_dtype: image * (1 / 255) in float32
METHODS = ("bilinear", "nearest", "bicubic", "area")  # tf.image.ResizeMethod (TF1) 0..3
TRANSFORMS = ("none", "brightness", "contrast")


# ---- image_resizer_state.h --------------------------------------------------------------------------------------------
def resize_scale(in_size, out_size):
    """CalculateResizeScale with align_corners=True."""
    return F(in_size - 1) / F(out_size - 1) if out_size > 1 else F(in_size) / F(out_size)


def legacy_loc(loc, scale):
    """LegacyScaler: static_cast<float>(x) * scale, for an int array of output coordinates."""
    return np.asarray(loc).astype(F) * F(scale)


def bound(v, n):
    """BOUND / Bound: min(n - 1, max(0, v))."""
    return np.minimum(n - 1, np.maximum(0, v))


def _gather(img, rows, cols):
    """img[rows[i], cols[j]] for every output pixel (i, j): [len(rows), len(cols), 3]."""
    return img[np.asarray(rows)[:, None], np.asarray(cols)[None, :]]


# ---- resize_bilinear_op.cc --------------------------------------------------------------------------------------------
def lerp(a, b, t):
    """compute_lerp's a + (b - a) * t, rounded after the subtraction, the product and the sum."""
    return a + (b - a) * t


def _bilinear_weights(loc, in_size, scale):
    """compute_interpolation_weights: lower, upper, lerp of each output coordinate."""
    x = legacy_loc(loc, scale)
    x_f = np.floor(x)
    return np.maximum(x_f.astype(np.int64), 0), np.minimum(np.ceil(x).astype(np.int64), in_size - 1), x - x_f


def resize_bilinear(img, ry, rx, hs, ws):
    y_lo, y_hi, y_l = _bilinear_weights(ry, img.shape[0], hs)
    x_lo, x_hi, x_l = _bilinear_weights(rx, img.shape[1], ws)
    x_l = x_l[None, :, None]
    top = lerp(_gather(img, y_lo, x_lo), _gather(img, y_lo, x_hi), x_l)
    bottom = lerp(_gather(img, y_hi, x_lo), _gather(img, y_hi, x_hi), x_l)
    return lerp(top, bottom, y_l[:, None, None])


# ---- resize_nearest_neighbor_op.cc ------------------------------------------------------------------------------------
def roundf(x):
    """C roundf, halfway cases away from zero, for x >= 0: the fraction x - floor(x) of a float32 is exact."""
    fl = np.floor(x)
    return np.where(x - fl >= F(0.5), fl + F(1.0), fl)


def resize_nearest(img, ry, rx, hs, ws):
    y = np.minimum(roundf(legacy_loc(ry, hs)).astype(np.int64), img.shape[0] - 1)
    x = np.minimum(roundf(legacy_loc(rx, ws)).astype(np.int64), img.shape[1] - 1)
    return _gather(img, y, x)


# ---- resize_bicubic_op.cc ---------------------------------------------------------------------------------------------
TABLE_SIZE = 1024


def _coeffs_table(a=-0.75):
    """InitCoeffsTable: x = i / 1024 stored as float, the polynomials in double (a is a double), each entry stored as float."""
    x = (np.arange(TABLE_SIZE + 1, dtype=np.float64) * 1.0 / TABLE_SIZE).astype(F).astype(np.float64)
    t = np.zeros((TABLE_SIZE + 1) * 2, F)
    t[0::2] = ((a + 2) * x - (a + 3)) * x * x + 1
    x = (x + 1.0).astype(F).astype(np.float64)  # x += 1.0 on a float
    t[1::2] = ((a * x - 5 * a) * x + 8 * a) * x - 4 * a
    return t


COEFFS = _coeffs_table()


def table_offset(delta):
    """lrintf(delta * kTableSize): round half to even under the default rounding mode."""
    return np.rint(delta * F(TABLE_SIZE)).astype(np.int64)


def _cubic_weights(loc, limit, scale):
    """GetWeightsAndIndices<LegacyScaler, use_keys_cubic=false>: four weights and four clamped indices per coordinate."""
    in_loc_f = legacy_loc(loc, scale)
    in_loc = np.floor(in_loc_f)
    off = table_offset(in_loc_f - in_loc)
    w = (COEFFS[off * 2 + 1], COEFFS[off * 2], COEFFS[(TABLE_SIZE - off) * 2], COEFFS[(TABLE_SIZE - off) * 2 + 1])
    i = in_loc.astype(np.int64)
    return w, tuple(bound(i + k, limit) for k in (-1, 0, 1, 2))


def interpolate_1d(w, v):
    """Interpolate1D / Compute: ((v0 w0 + v1 w1) + v2 w2) + v3 w3, tap by tap."""
    acc = v[0] * w[0]
    for k in (1, 2, 3):
        acc = acc + v[k] * w[k]
    return acc


def resize_bicubic(img, ry, rx, hs, ws):
    """interpolate_with_caching: the y interpolation at each of the four x taps, then the x interpolation of those four."""
    yw, yi = _cubic_weights(ry, img.shape[0], hs)
    xw, xi = _cubic_weights(rx, img.shape[1], ws)
    yw = [w[:, None, None] for w in yw]
    cached = [interpolate_1d(yw, [_gather(img, yi[k], xi[j]) for k in range(4)]) for j in range(4)]
    return interpolate_1d([w[None, :, None] for w in xw], cached)


# ---- resize_area_op.cc ------------------------------------------------------------------------------------------------
def cell_scale(v, in0, in1, full):
    """The weight of source cell v in the box [in0, in1) (ResizeAreaOp's start_scale / end_minus_one_scale / scale_y)."""
    vf, v1 = np.asarray(v).astype(F), (np.asarray(v) + 1).astype(F)
    return np.where(vf < in0, np.where(v1 > in1, F(full), v1 - in0), np.where(v1 > in1, in1 - vf, F(1.0))).astype(F)


def area_x_interp(loc, scale):
    """CachedInterpolation of each output column: start, end, start_scale, end_minus_one_scale."""
    in_x, in_x1 = legacy_loc(loc, scale), legacy_loc(np.asarray(loc) + 1, scale)
    start, end = np.floor(in_x).astype(np.int64), np.ceil(in_x1).astype(np.int64)
    return start, end, cell_scale(start, in_x, in_x1, scale), cell_scale(end - 1, in_x, in_x1, scale)


def resize_area(img, ry, rx, hs, ws):
    """ResizeAreaOp::ComputeLoop with ComputePatchSumOf3Channels: per row tap i in y_start..y_end-1, the row's patch sum
    start * start_scale (+ middle cells + end-1 * end_scale when start + 1 != end), accumulated as sum += sum_y * scale_y,
    then times 1 / (height_scale * width_scale)."""
    in_h, in_w = img.shape[:2]
    in_y, in_y1 = legacy_loc(ry, hs), legacy_loc(np.asarray(ry) + 1, hs)
    y_start, y_end = np.floor(in_y).astype(np.int64), np.ceil(in_y1).astype(np.int64)
    xs, xe, xs_scale, xe_scale = area_x_interp(rx, ws)
    xs_scale, xe_scale = xs_scale[None, :, None], xe_scale[None, :, None]
    two_ends = (xs + 1 != xe)[None, :, None]
    total = np.zeros((len(ry), len(rx), 3), F)
    for ky in range(int(max(0, (y_end - y_start).max(initial=0)))):
        i = y_start + ky
        row = bound(i, in_h)
        y_on = (i < y_end)[:, None, None]
        sum_y = _gather(img, row, bound(xs, in_w)) * xs_scale
        for kx in range(1, int(max(0, (xe - xs).max(initial=0))) - 1):
            x = xs + kx
            sum_y = np.where((x < xe - 1)[None, :, None], sum_y + _gather(img, row, bound(x, in_w)), sum_y)
        sum_y = np.where(two_ends, sum_y + _gather(img, row, bound(xe - 1, in_w)) * xe_scale, sum_y)
        total = np.where(y_on, total + sum_y * cell_scale(i, in_y, in_y1, hs)[:, None, None], total)
    with np.errstate(divide="ignore", invalid="ignore"):  # a 1-pixel side upscaled has scale 0: 0 * inf, NaN, as in C++
        norm = F(np.float64(1.0) / np.float64(F(hs) * F(ws)))  # const float scale = 1.0 / (height_scale * width_scale)
        return total * norm


RESIZE = (resize_bilinear, resize_nearest, resize_bicubic, resize_area)


# ---- resize_and_pad + where(isfinite) + lightweight_image_augment -------------------------------------------------------
def to_float(u8):
    """convert_image_dtype(uint8 -> float32): a multiply by float32(1/255)."""
    return np.asarray(u8).astype(F) * INV255


def resize_and_pad(img, out_size, sh, sw, oy, ox, method):
    """The [Hd, Wd, 3] float32 image resize_and_pad leaves for float32 source `img`, with where(isfinite(x), x, 0) applied:
    the crop window [oy, oy + Hd) x [ox, ox + Wd) of the (sh, sw) resize, zero where that window leaves the resized image."""
    Hd, Wd = out_size
    ry, rx = np.arange(oy, min(oy + Hd, sh)), np.arange(ox, min(ox + Wd, sw))
    out = np.zeros((Hd, Wd, 3), F)
    if len(ry) and len(rx):
        v = RESIZE[method](img, ry, rx, resize_scale(img.shape[0], sh), resize_scale(img.shape[1], sw))
        with np.errstate(invalid="ignore"):
            out[:len(ry), :len(rx)] = np.where(np.isfinite(v), v, F(0.0))
    return out


def padded_mean(img):
    """float64 per-channel mean of the padded image: what reduce_mean computes, before its float32 rounding."""
    return np.asarray(img, np.float64).mean((0, 1))


# ---- the float32 contrast mean --------------------------------------------------------------------------------------------
U32 = 2.0 ** -24  # unit roundoff of float32, round to nearest
MEAN_THREADS, WARP = 512, 32


def mean_bound(img, threads=MEAN_THREADS, warp=WARP):
    """Per-channel bound on |float32 mean - exact mean| of the padded [Hd, Wd, 3] image for a reduction of this shape: each of
    `threads` threads sums its ceil(npx / threads) pixels serially from 0 (k - 1 roundings, the first addition is exact), a
    butterfly over each warp (log2(32) = 5 roundings), the threads / warp warp sums added serially from 0 (15 roundings for
    512 threads), then one division by npx.  Every pixel passes through at most d = k - 1 + 5 + 15 roundings, so the float32
    sum S' satisfies |S' - S| <= gamma_d sum|x| with gamma_d = d u / (1 - d u) (Higham, Accuracy and Stability of Numerical
    Algorithms, 2nd ed., section 4.2), and the division adds u |S'| / npx <= u (|S| + gamma_d sum|x|) / npx.  S and sum|x| are taken
    in float64 from the oracle's image; their own error (below npx 2^-53 relative) is covered by a 2^-40 relative margin."""
    x = np.asarray(img, np.float64).reshape(-1, 3)
    npx = len(x)
    k = -(-npx // threads)
    d = (k - 1) + int(np.log2(warp)) + (threads // warp - 1)
    gamma = d * U32 / (1 - d * U32)
    s, sa = np.abs(x.sum(0)), np.abs(x).sum(0)
    return ((gamma * (1 + U32) + 2.0 ** -40) * sa + U32 * s) / npx


def reduction_mean(img, threads=MEAN_THREADS, warp=WARP):
    """float32 mean in one order of that shape: thread t sums pixels t, t + threads, ... of the row-major image, a butterfly
    (lane i adds lane i ^ o for o = 16, 8, ..., 1), lane 0's sums added warp by warp, then the division by the pixel count."""
    v = np.asarray(img, F).reshape(-1, 3)
    npx = len(v)
    acc = np.zeros((threads, 3), F)
    for p0 in range(0, npx, threads):
        blk = v[p0:p0 + threads]
        acc[:len(blk)] = acc[:len(blk)] + blk
    a = acc.reshape(threads // warp, warp, 3)
    o = warp // 2
    while o:
        a = a + a[:, np.arange(warp) ^ o]
        o //= 2
    s = np.zeros(3, F)
    for w in range(threads // warp):
        s = s + a[w, 0]
    return s / F(npx)


def augment(img, transform, factor, mean=None):
    """0: the image unchanged (no clip); 1 brightness x * f; 2 contrast (x - mean) * f + mean with the given float32 per-channel
    mean; 1 and 2 then clip_by_value(0, 1)."""
    if transform == 0:
        return img
    f = np.asarray(factor, F).reshape(1, 1, 3)
    if transform == 1:
        x = img * f
    else:
        m = np.asarray(mean, F).reshape(1, 1, 3)
        x = (img - m) * f + m
    return np.minimum(np.maximum(x, F(0.0)), F(1.0))


# ---- the cases the GPU test runs -----------------------------------------------------------------------------------------
def natural_u8(rng, h, w):
    """Camera-like uint8 content: smooth gradients and a low-frequency wave per channel, sensor noise, and saturated black and
    white blocks, so that brightness and contrast reach both ends of clip_by_value."""
    y = np.linspace(0.0, 1.0, h)[:, None, None]
    x = np.linspace(0.0, 1.0, w)[None, :, None]
    a, b, ph = rng.uniform(-120, 120, (3, 1, 1, 3))
    f = rng.uniform(1.0, 6.0, (1, 1, 3))
    v = 128 + a * (y - 0.5) + b * (x - 0.5) + 40 * np.sin(2 * np.pi * f * (x + y) + ph) + rng.normal(0, 10, (h, w, 3))
    for level in (0, 255, 0, 255):
        bh, bw = max(1, h // rng.integers(3, 8)), max(1, w // rng.integers(3, 8))
        y0, x0 = rng.integers(0, h - bh + 1), rng.integers(0, w - bw + 1)
        v[y0:y0 + bh, x0:x0 + bw] = level
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


def _frames(rng, si, plans):
    """One frame per plan x method x transform of source si, each with its own per-channel factor U[0.68, 1.32)."""
    out = []
    for sh, sw, oy, ox in plans:
        for m in range(4):
            for t in range(3):
                out.append(dict(src=si, scaled_h=int(sh), scaled_w=int(sw), offset_y=int(oy), offset_x=int(ox), method=m,
                                augment=t, factor=rng.uniform(0.68, 1.32, 3).astype(F)))
    return out


def _pretrain_launch(rng):
    """192 x 352 frames under dataloader.plan_frames at the default scale range and at 1.125-1.5, from 360 x 640, 480 x 854,
    720 x 1280 and portrait 640 x 360 sources, and a wide and a tall source whose short side hits the 64-pixel floor."""
    from merlot_b200.dataloader import plan_frames
    out = (192, 352)
    sizes = [(360, 640), (480, 854), (720, 1280), (640, 360), (90, 1600), (1400, 100)]
    srcs = [natural_u8(rng, h, w) for h, w in sizes]
    frames, floored = [], 0
    for si, (h, w) in enumerate(sizes):
        for lo, hi in ((0.95, 1.05), (1.125, 1.5)):
            s = F(lo) + rng.random(dtype=F) * (F(hi) - F(lo))
            p = plan_frames(np.array([h]), np.array([w]), out, np.array([s]), np.array([rng.random(dtype=F)]),
                            np.array([rng.random(dtype=F)]))
            plan = tuple(int(p[k][0]) for k in ("scaled_h", "scaled_w", "offset_y", "offset_x"))
            floored += min(plan[:2]) == 64
            frames += _frames(rng, si, [plan])
    assert floored >= 4, "the wide and tall sources must hit the 64-pixel floor"
    return dict(name="pretrain", out=out, srcs=srcs, frames=frames)


def _eval_launch(rng, out):
    """out-sized frames under dataloader.plan_frames_eval (VCR 384 x 704, sort_story 384 x 384, video_mc/qa/fib 192 x 352):
    video-sized and portrait sources, very wide and very tall ones whose resized short side is a few pixels, and video_mc's
    empty slot (a 1 x 1 black source resized to the whole output)."""
    from merlot_b200.dataloader import plan_frames_eval
    sizes = [(480, 854), (720, 1280), (360, 640), (1000, 700), (12, 3000), (3000, 20)]
    srcs = [natural_u8(rng, h, w) for h, w in sizes] + [np.zeros((1, 1, 3), np.uint8)]
    frames = []
    for si, (h, w) in enumerate(sizes):
        p = plan_frames_eval(np.array([h]), np.array([w]), out)
        plan = tuple(int(p[k][0]) for k in ("scaled_h", "scaled_w", "offset_y", "offset_x"))
        assert min(plan[:2]) >= 1
        frames += _frames(rng, si, [plan])
    thin = [min(f["scaled_h"], f["scaled_w"]) for f in frames]
    assert min(thin) <= 4, "a very wide or tall source must resize to a side of a few pixels"
    frames += _frames(rng, len(sizes), [(out[0], out[1], 0, 0)])
    return dict(name=f"eval {out[0]}x{out[1]}", out=out, srcs=srcs, frames=frames)


def _edge_launch(rng, out):
    """Small outputs (out_h * out_w of 1, just below and just above 256, none a multiple of it) from sources of 1 pixel, one
    row, one column, >= 8x larger and >= 8x smaller than the output, under plans that reach the edges: identity, the whole
    output, 1-pixel resizes, the largest crop offsets (scaled - desired), padding only at the bottom, only at the right."""
    Hd, Wd = out
    sizes = [(1, 1), (1, 7), (9, 1), (2, 3), (13, 11), (61, 90), (8 * Hd + 5, 8 * Wd + 3)]
    srcs = [natural_u8(rng, h, w) for h, w in sizes]
    frames = []
    for si, (h, w) in enumerate(sizes):
        up_h, up_w = 8 * Hd + 3, 8 * Wd + 1  # >= 8x up from the small sources
        plans = {(h, w, 0, 0), (Hd, Wd, 0, 0), (1, 1, 0, 0), (1, Wd + 2, 0, 2), (Hd + 1, 1, 1, 0),
                 (up_h, up_w, up_h - Hd, up_w - Wd),            # crop at the far corner
                 (max(1, Hd - 3), Wd + 4, 0, 4),                 # padding at the bottom only
                 (Hd + 5, max(1, Wd - 2), 5, 0),                 # padding at the right only
                 (max(1, Hd // 2), max(1, Wd // 3), 0, 0)}       # both
        frames += _frames(rng, si, sorted(plans))
    return dict(name=f"edges {Hd}x{Wd}", out=out, srcs=srcs, frames=frames)


def gpu_cases(seed=0):
    """The launches of tests/test_gpu_frames_exact.py: dicts of name, out (Hd, Wd), srcs (uint8 HWC arrays) and frames (dicts
    of src index, scaled_h, scaled_w, offset_y, offset_x, method, augment, factor).  Every launch mixes sizes, methods and
    transforms; the first edge launch holds more than 300 frames (grid.y)."""
    rng = np.random.default_rng(seed)
    launches = [_edge_launch(rng, out) for out in ((15, 17), (1, 1), (7, 37), (1, 257))]
    launches.append(_pretrain_launch(rng))
    launches += [_eval_launch(rng, out) for out in ((384, 704), (384, 384), (192, 352))]
    assert len(launches[0]["frames"]) > 300
    return launches


def launch_plan(launch):
    """(packed uint8 sources, the plan dict ops.frames_prepare takes) of a launch."""
    srcs = launch["srcs"]
    offs = np.concatenate([[0], np.cumsum([s.size for s in srcs])[:-1]]).astype(np.int64)
    packed = np.concatenate([s.reshape(-1) for s in srcs])
    fr = launch["frames"]
    plan = {k: np.array([f[k] for f in fr], np.int64) for k in ("scaled_h", "scaled_w", "offset_y", "offset_x", "method",
                                                                 "augment")}
    plan.update(src_offset=offs[[f["src"] for f in fr]], src_h=np.array([srcs[f["src"]].shape[0] for f in fr]),
                src_w=np.array([srcs[f["src"]].shape[1] for f in fr]), factor=np.stack([f["factor"] for f in fr]))
    return packed, plan


def frame_name(launch, f):
    h, w = launch["srcs"][f["src"]].shape[:2]
    return (f"{launch['name']}: {METHODS[f['method']]} {TRANSFORMS[f['augment']]} {h}x{w} -> "
            f"({f['scaled_h']}, {f['scaled_w']}) at ({f['offset_y']}, {f['offset_x']})")


def resized_frames(launch):
    """{(src, scaled_h, scaled_w, offset_y, offset_x, method): the padded float32 image} of every distinct resize in a launch."""
    imgs = [to_float(s) for s in launch["srcs"]]
    out = {}
    for f in launch["frames"]:
        key = frame_key(f)
        if key not in out:
            out[key] = resize_and_pad(imgs[f["src"]], launch["out"], *key[1:])
    return out


def frame_key(f):
    return (f["src"], f["scaled_h"], f["scaled_w"], f["offset_y"], f["offset_x"], f["method"])
