"""ORACLE -- TEST INFRASTRUCTURE ONLY.  NumPy restatement of the per-example half of the reference's pretraining input:
the text part of `_dataset_parser` (model/dataloader.py:56-126), `resize_and_pad` (utils/model_utils.py:855-940),
`lightweight_image_augment`'s brightness and contrast transforms (:758-835) and the TF 1.15 legacy resize kernels that
`tf.image.resize_images(..., align_corners=True)` runs for the four ResizeMethods (tensorflow/core/kernels/
resize_bilinear_op.cc, resize_nearest_neighbor_op.cc, resize_bicubic_op.cc, resize_area_op.cc, image_resizer_state.h).

Written from the structure of those sources -- per output row, column and pixel, whole-image resize then crop and pad --
and not from csrc/frames.cu.  float32 arithmetic is done on np.float32 values, one rounding per operation, no fused
multiply-add.  PARITY UNPINNED against TensorFlow itself (it cannot be installed here); tests/test_input_host.py pins what
can be derived by hand (corner pixels, constant images, identity resizes, linear ramps, the plan's 64-pixel floor)."""
import math

import numpy as np

from oracle.oracle_np import bf16_round

F = np.float32
INV255 = F(1.0 / 255.0)  # convert_image_dtype: image * (1 / dtype.max) in float32
METHODS = ("bilinear", "nearest", "bicubic", "area")  # tf.image.ResizeMethod (TF1) 0..3


# ---- text features of _dataset_parser (:65-69, :100-125) --------------------------------------------------------------
def encode_string(s: bytes, string_len: int):  # utils/model_utils.py:628-637
    raw = np.frombuffer(s, dtype=np.uint8).astype(np.int32)[:string_len]
    return np.concatenate([raw, np.zeros(string_len - len(raw), np.int32)])


def dataset_parser_text(chunks, chunk_text_len, do_clean):
    """chunks: list of dicts with tokenized_cleaned_asr, tokenized_raw_asr (int lists), youtube_id (bytes), chunk_num,
    mean_time, is_eoc."""
    n = len(chunks)
    caps = [list(c["tokenized_cleaned_asr" if do_clean else "tokenized_raw_asr"]) for c in chunks]
    width = max(len(c) for c in caps)
    asr = np.zeros((n, width), dtype=np.int64)  # tf.ragged.stack(...).to_tensor(default_value=0), squeezed
    for i, c in enumerate(caps):
        asr[i, :len(c)] = c
    asr = asr.astype(np.int32)
    start = 2 if do_clean else 5  # tf.where(do_clean, START, NEXTCAPTION_START)
    asr = np.concatenate([np.full((n, 1), start, np.int32), asr], 1)
    asr = asr[:, :chunk_text_len]  # pad_to_fixed_size(truncate=True, axis=1): truncate, then pad with 0
    asr = np.concatenate([asr, np.zeros((n, chunk_text_len - asr.shape[1]), np.int32)], 1)
    is_eoc = np.array([c["is_eoc"] for c in chunks[:-1]] + [1]).astype(bool)
    delta = np.concatenate([[0], is_eoc[:-1].astype(np.int32)])
    return {"youtube_id": np.stack([encode_string(c["youtube_id"], 64) for c in chunks]),
            "chunk_num": np.array([c["chunk_num"] for c in chunks]).astype(np.int32),
            "mean_time": np.array([c["mean_time"] for c in chunks], dtype=np.float32),
            "input_ids": asr, "is_eoc": is_eoc, "video_src_ids": np.cumsum(delta).astype(np.int32)}


# ---- resize_and_pad's plan (utils/model_utils.py:869-899), one frame, float32 scalars ------------------------------------
def resize_plan(height, width, desired_size, random_scale_factor, u_y, u_x):
    desired_height, desired_width = desired_size
    desired_height_f, desired_width_f = F(desired_height), F(desired_width)
    height, width = F(height), F(width)
    scaled_y = int(F(random_scale_factor) * desired_height_f)  # tf.cast(float -> int32) truncates
    scaled_x = int(F(random_scale_factor) * desired_width_f)
    image_scale_y = F(scaled_y) / height
    image_scale_x = F(scaled_x) / width
    image_scale = min(image_scale_x, image_scale_y)
    image_scale = max(image_scale, F(64.0) / min(height, width))
    scaled_height = int(height * image_scale)
    scaled_width = int(width * image_scale)
    offset_y = F(scaled_height - desired_height)
    offset_x = F(scaled_width - desired_width)
    offset_y = int(max(F(0.0), offset_y) * F(u_y))
    offset_x = int(max(F(0.0), offset_x) * F(u_x))
    return scaled_height, scaled_width, offset_y, offset_x


# ---- TF 1.15 legacy resize kernels, align_corners=True -----------------------------------------------------------------
def calculate_resize_scale(in_size, out_size):  # image_resizer_state.h
    return F(in_size - 1) / F(out_size - 1) if out_size > 1 else F(in_size) / F(out_size)


def resize_bilinear(img, out_h, out_w):
    in_h, in_w, _ = img.shape

    def weights(out_size, in_size, scale):  # compute_interpolation_weights with LegacyScaler
        res = []
        for i in range(out_size):
            inp = F(i) * scale
            in_f = np.floor(inp)
            res.append((max(int(in_f), 0), min(int(np.ceil(inp)), in_size - 1), inp - in_f))
        return res

    ys = weights(out_h, in_h, calculate_resize_scale(in_h, out_h))
    xs = weights(out_w, in_w, calculate_resize_scale(in_w, out_w))
    out = np.zeros((out_h, out_w, 3), F)
    for y, (y_lo, y_hi, y_lerp) in enumerate(ys):
        for x, (x_lo, x_hi, x_lerp) in enumerate(xs):
            for c in range(3):  # compute_lerp
                top_left, top_right = img[y_lo, x_lo, c], img[y_lo, x_hi, c]
                bottom_left, bottom_right = img[y_hi, x_lo, c], img[y_hi, x_hi, c]
                top = top_left + (top_right - top_left) * x_lerp
                bottom = bottom_left + (bottom_right - bottom_left) * x_lerp
                out[y, x, c] = top + (bottom - top) * y_lerp
    return out


def resize_nearest(img, out_h, out_w):
    in_h, in_w, _ = img.shape
    hs, ws = calculate_resize_scale(in_h, out_h), calculate_resize_scale(in_w, out_w)
    out = np.zeros((out_h, out_w, 3), F)
    for y in range(out_h):
        in_y = min(math.floor(float(F(y) * hs) + 0.5), in_h - 1)  # roundf: half away from zero (values are >= 0)
        for x in range(out_w):
            in_x = min(math.floor(float(F(x) * ws) + 0.5), in_w - 1)
            out[y, x] = img[in_y, in_x]
    return out


def _coeffs_table(a=-0.75, table_size=1024):  # InitCoeffsTable: double arithmetic, stored as float
    t = np.zeros((table_size + 1) * 2, F)
    for i in range(table_size + 1):
        x = float(F(i * 1.0 / table_size))
        t[i * 2] = ((a + 2) * x - (a + 3)) * x * x + 1
        x = float(F(x + 1.0))
        t[i * 2 + 1] = ((a * x - 5 * a) * x + 8 * a) * x - 4 * a
    return t


_COEFFS = _coeffs_table()


def _cubic_weights_and_indices(scale, out_loc, limit):  # GetWeightsAndIndices<LegacyScaler, use_keys_cubic=false>
    in_loc_f = F(out_loc) * scale
    in_loc = math.floor(in_loc_f)
    delta = in_loc_f - F(in_loc)
    offset = round(float(delta * F(1024)))  # lrintf: round half to even
    w = (_COEFFS[offset * 2 + 1], _COEFFS[offset * 2], _COEFFS[(1024 - offset) * 2], _COEFFS[(1024 - offset) * 2 + 1])
    idx = tuple(min(limit - 1, max(0, in_loc + k)) for k in (-1, 0, 1, 2))  # Bound
    return w, idx


def _interpolate_1d(w, v):
    return v[0] * w[0] + v[1] * w[1] + v[2] * w[2] + v[3] * w[3]


def resize_bicubic(img, out_h, out_w):  # interpolate_with_caching: y interpolation at each of 4 x taps, then x
    in_h, in_w, _ = img.shape
    hs, ws = calculate_resize_scale(in_h, out_h), calculate_resize_scale(in_w, out_w)
    x_wais = [_cubic_weights_and_indices(ws, x, in_w) for x in range(out_w)]
    out = np.zeros((out_h, out_w, 3), F)
    for y in range(out_h):
        yw, yi = _cubic_weights_and_indices(hs, y, in_h)
        for x in range(out_w):
            xw, xi = x_wais[x]
            for c in range(3):
                cached = [_interpolate_1d(yw, [img[yi[k], xi[j], c] for k in range(4)]) for j in range(4)]
                out[y, x, c] = _interpolate_1d(xw, cached)
    return out


def resize_area(img, out_h, out_w):  # ResizeAreaOp::ComputeLoop, ComputePatchSumOf3Channels
    in_h, in_w, _ = img.shape
    hs, ws = calculate_resize_scale(in_h, out_h), calculate_resize_scale(in_w, out_w)
    bound = lambda v, n: min(n - 1, max(0, v))  # noqa: E731  BOUND

    def cell_scale(v, in0, in1, full):
        if F(v) < in0:
            return full if F(v + 1) > in1 else F(v + 1) - in0
        return in1 - F(v) if F(v + 1) > in1 else F(1.0)

    x_interps = []
    for x in range(out_w):
        in_x, in_x1 = F(x) * ws, F(x + 1) * ws
        start, end = math.floor(in_x), math.ceil(in_x1)
        x_interps.append((start, end, cell_scale(start, in_x, in_x1, ws), cell_scale(end - 1, in_x, in_x1, ws)))
    with np.errstate(divide="ignore"):  # a 1-pixel side resized to more has scale 0: 1.0 / 0.0 is inf in C++
        scale = F(np.float64(1.0) / np.float64(hs * ws))
    out = np.zeros((out_h, out_w, 3), F)
    for y in range(out_h):
        in_y, in_y1 = F(y) * hs, F(y + 1) * hs
        rows = [(bound(i, in_h), cell_scale(i, in_y, in_y1, hs)) for i in range(math.floor(in_y), math.ceil(in_y1))]
        for x, (start, end, start_scale, end_scale) in enumerate(x_interps):
            for c in range(3):
                total = F(0.0)
                for r, y_scale in rows:
                    sum_y = img[r, bound(start, in_w), c] * start_scale
                    if start + 1 != end:
                        for xx in range(start + 1, end - 1):
                            sum_y = sum_y + img[r, bound(xx, in_w), c]
                        sum_y = sum_y + img[r, bound(end - 1, in_w), c] * end_scale
                    total = total + sum_y * y_scale
                with np.errstate(invalid="ignore"):  # 0 * inf when no row contributes: NaN, zeroed by where(isfinite)
                    out[y, x, c] = total * scale
    return out


RESIZE = (resize_bilinear, resize_nearest, resize_bicubic, resize_area)


def resize_and_pad(img, desired_size, scaled_height, scaled_width, offset_y, offset_x, method):
    """The image half of resize_and_pad: resize the whole image, crop, pad_to_bounding_box(0, 0, Hd, Wd)."""
    Hd, Wd = desired_size
    img = RESIZE[method](img, scaled_height, scaled_width)
    img = img[offset_y:offset_y + Hd, offset_x:offset_x + Wd]
    out = np.zeros((Hd, Wd, 3), F)
    out[:img.shape[0], :img.shape[1]] = img
    return out


def augment(img, transform, factor):  # 1 brightness, 2 contrast, then clip_by_value(0, 1); 0 leaves the image alone
    factor = np.asarray(factor, F).reshape(1, 1, 3)
    if transform == 0:
        return img
    if transform == 1:
        x = img * factor
    else:
        x_mean = img.astype(np.float64).mean((0, 1), keepdims=True).astype(F)  # reduce_mean over [0, 1]
        x = (img - x_mean) * factor + x_mean
    return np.minimum(np.maximum(x, F(0.0)), F(1.0))


def load_and_resize_img(u8, desired_size, scale, u_y, u_x, method, transform, factor):
    """`_load_and_resize_img` (:72-89) after the JPEG decode + the bf16 cast (:94-96), as float32 values of bf16."""
    img = u8.astype(F) * INV255
    plan = resize_plan(u8.shape[0], u8.shape[1], desired_size, scale, u_y, u_x)
    img = resize_and_pad(img, desired_size, *plan, method)
    img = np.where(np.isfinite(img), img, F(0.0))
    img = augment(img, transform, factor)
    return bf16_round(img), plan
