"""CPU tests of tests/frames_exact_oracle.py, the reference that tests/test_gpu_frames_exact.py holds K14 (csrc/frames.cu) to
bit for bit: the vectorised restatement equals the per-pixel tests/input_oracle.py exactly over a grid of small shapes; one
wrong reference per plausible kernel slip differs from it in at least one bf16 output of the GPU test's own frames, so an
exact match on the GPU rules each slip out; and the contrast-mean bound the GPU test applies holds for a float32 emulation
of a reduction of that shape while a mean over the unpadded crop breaks it."""
import numpy as np
import pytest

from tests import frames_exact_oracle as X
from tests import input_oracle as O

F = np.float32

# (source h, w, scaled h, w, offset y, x, output h, w): 1-row and 1-column sources, 1 x 1 and 1 x N outputs, identity,
# >= 8x down and >= 8x up, crops at the largest offsets (scaled - desired), padding at the bottom, the right and both
GRID = [(1, 1, 1, 1, 0, 0, 1, 1), (1, 1, 5, 7, 0, 0, 4, 6), (1, 9, 3, 20, 0, 4, 3, 16), (11, 1, 25, 2, 9, 0, 16, 3),
        (1, 6, 1, 1, 0, 0, 1, 5), (7, 9, 1, 13, 0, 2, 1, 11), (7, 9, 7, 9, 0, 0, 7, 9), (7, 9, 7, 9, 0, 0, 10, 12),
        (64, 72, 7, 8, 0, 0, 7, 8), (66, 90, 6, 9, 1, 2, 5, 7), (3, 4, 30, 37, 4, 9, 26, 28), (2, 2, 19, 17, 0, 0, 19, 17),
        (13, 17, 21, 29, 21 - 9, 29 - 11, 9, 11), (20, 31, 5, 40, 0, 40 - 12, 8, 12), (20, 31, 14, 6, 14 - 10, 0, 10, 9),
        (15, 15, 16, 16, 3, 3, 16, 16), (5, 40, 1, 50, 0, 0, 1, 50)]


def _u8(h, w, seed):
    return X.natural_u8(np.random.default_rng(seed), h, w)


@pytest.mark.parametrize("method", range(4), ids=X.METHODS)
def test_vectorised_oracle_equals_per_pixel_oracle(method):
    for g, (h, w, sh, sw, oy, ox, Hd, Wd) in enumerate(GRID):
        u8 = _u8(h, w, g)
        img = u8.astype(F) * O.INV255
        np.testing.assert_array_equal(X.to_float(u8).view(np.uint32), img.view(np.uint32))
        with np.errstate(invalid="ignore"):
            want = O.resize_and_pad(img, (Hd, Wd), sh, sw, oy, ox, method)
        want = np.where(np.isfinite(want), want, F(0.0))
        got = X.resize_and_pad(img, (Hd, Wd), sh, sw, oy, ox, method)
        what = f"{X.METHODS[method]} {h}x{w} -> ({sh}, {sw}) at ({oy}, {ox}) in {Hd}x{Wd}"
        assert got.dtype == F and got.shape == (Hd, Wd, 3), what
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=what)  # bits, signs of zero included
        fac = np.random.default_rng(g).uniform(0.68, 1.32, 3).astype(F)
        for t in range(3):
            ref = O.augment(want, t, fac)
            mean = want.astype(np.float64).mean((0, 1)).astype(F)  # input_oracle's own mean, handed to the restatement
            np.testing.assert_array_equal(X.augment(got, t, fac, mean).view(np.uint32), ref.view(np.uint32),
                                          err_msg=f"{what} transform {t}")


def test_area_of_an_upscaled_one_pixel_side_is_zero():
    # scale 0 on that axis: no source row (or column) contributes, 0 * (1 / 0) is NaN and where(isfinite) makes it 0
    img = X.to_float(_u8(1, 5, 0))
    assert (X.resize_and_pad(img, (4, 6), 4, 6, 0, 0, 3) == 0).all()
    assert (X.resize_and_pad(img, (1, 6), 1, 6, 0, 0, 3) != 0).any()


def test_coefficient_table_ends():
    # weights of offset 0 are (k(1), k(0), k(1), k(2)) = (0, 1, 0, 0); every row of four sums to 1 within float rounding
    assert X.COEFFS[0] == 1 and X.COEFFS[1] == 0 and X.COEFFS[2048] == 0 and X.COEFFS[2049] == 0
    off = np.arange(1025)
    s = (X.COEFFS[off * 2 + 1].astype(np.float64) + X.COEFFS[off * 2] + X.COEFFS[(1024 - off) * 2]
         + X.COEFFS[(1024 - off) * 2 + 1])
    assert np.abs(s - 1).max() < 1e-6


# ---- wrong references ---------------------------------------------------------------------------------------------------
def _fma_lerp(a, b, t):  # (b - a) * t + a with the product and the sum rounded once, as an FMA does
    return (np.float64(1.0) * (b - a) * t.astype(np.float64) + a).astype(F)


def _roundf_half_even(x):
    return np.rint(x)


def _scale_half_pixel(in_size, out_size):  # align_corners=False's in / out, which half_pixel_centers uses
    return F(in_size) / F(out_size)


def _table_offset_truncated(delta):
    return (delta * F(X.TABLE_SIZE)).astype(np.int64)


_area_x_interp = X.area_x_interp


def _area_end_from_start(loc, scale):
    start, end, s0, _ = _area_x_interp(loc, scale)
    return start, end, s0, s0


WRONG = {"fma lerp": ("lerp", _fma_lerp, (0,)),
         "nearest rounds half to even": ("roundf", _roundf_half_even, (1,)),
         "half_pixel_centers scale": ("resize_scale", _scale_half_pixel, (0, 1, 2, 3)),
         "bicubic offset truncated": ("table_offset", _table_offset_truncated, (2,)),
         "area end weight from the start cell": ("area_x_interp", _area_end_from_start, (3,))}


@pytest.fixture(scope="module")
def cases():
    return X.gpu_cases()


def _first_difference(cases, methods, wrong):
    """The first frame of the GPU test whose bf16 output under the wrong reference differs from the true one, with its
    transform applied (contrast fed the true padded mean), or None."""
    for launch in cases:
        imgs = [X.to_float(s) for s in launch["srcs"]]
        true = {}
        for f in launch["frames"]:
            if f["method"] not in methods:
                continue
            key = X.frame_key(f)
            if key not in true:
                true[key] = X.resize_and_pad(imgs[f["src"]], launch["out"], *key[1:])
            t = true[key]
            m = X.padded_mean(t).astype(F)
            got, bad_m = wrong(launch, f, t, imgs)
            a = X.bf16_round(X.augment(got, f["augment"], f["factor"], bad_m))
            b = X.bf16_round(X.augment(t, f["augment"], f["factor"], m))
            if (a != b).any():
                return X.frame_name(launch, f), int((a != b).sum())
    return None


@pytest.mark.parametrize("name", sorted(WRONG))
def test_wrong_reference_differs_on_the_gpu_frames(name, cases, monkeypatch):
    attr, fn, methods = WRONG[name]

    def wrong(launch, f, t, imgs):
        with monkeypatch.context() as mp:
            mp.setattr(X, attr, fn)
            return X.resize_and_pad(imgs[f["src"]], launch["out"], *X.frame_key(f)[1:]), X.padded_mean(t).astype(F)

    hit = _first_difference(cases, methods, wrong)
    assert hit is not None, f"{name}: no bf16 output of the GPU test's frames differs"
    print(f"{name}: {hit[1]} elements of {hit[0]}")


def test_contrast_mean_over_the_unpadded_crop_differs(cases):
    def wrong(launch, f, t, imgs):
        vh = max(0, min(launch["out"][0], f["scaled_h"] - f["offset_y"]))
        vw = max(0, min(launch["out"][1], f["scaled_w"] - f["offset_x"]))
        crop = X.padded_mean(t[:vh, :vw]) if vh and vw else np.zeros(3)
        return t, crop.astype(F)

    contrast = [dict(c, frames=[f for f in c["frames"] if f["augment"] == 2]) for c in cases]
    hit = _first_difference(contrast, range(4), wrong)
    assert hit is not None
    print(f"crop mean: {hit[1]} elements of {hit[0]}")


# ---- the contrast mean's bound ------------------------------------------------------------------------------------------
def test_mean_bound_holds_for_the_reduction_shape_and_rejects_the_crop_mean(cases):
    worst = 0.0
    checked = 0
    for launch in cases[4:]:  # the full-size launches
        for (si, sh, sw, oy, ox, m), t in X.resized_frames(launch).items():
            what = f"{launch['name']}: {X.METHODS[m]} source {si} -> ({sh}, {sw}) at ({oy}, {ox})"
            m64 = X.padded_mean(t)
            bound = X.mean_bound(t)
            err = np.abs(X.reduction_mean(t).astype(np.float64) - m64)
            assert (err <= bound).all(), (what, err, bound)
            worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
            checked += 1
            vh, vw = min(launch["out"][0], sh - oy), min(launch["out"][1], sw - ox)
            if (vh, vw) != tuple(launch["out"]) and np.abs(t).sum() > 0:
                crop = X.padded_mean(t[:vh, :vw])
                assert (np.abs(crop - m64) > bound).any(), what
    assert checked >= 100
    print(f"emulated reduction: worst mean error / bound {worst:.3g} over {checked} images")
