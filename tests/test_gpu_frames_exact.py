"""K14 (merlot_frames_prepare, csrc/frames.cu) element by element (pytest -m gpu), against tests/frames_exact_oracle.py at the
sizes the pipelines run and at the edges of the resize kernels' tap arithmetic.  Each launch of X.gpu_cases() goes to the
GPU as one call, with frames of mixed sizes under every method and transform:

- edges at outputs of 15 x 17, 1 x 1, 7 x 37 and 1 x 257 (out_h * out_w of 1, 255, 259 and 257: below and just above the
  256-thread block, never a multiple of it): 1-pixel, 1-row and 1-column sources, >= 8x up and down, crops at offset
  scaled - desired, padding at the bottom only and at the right only; the first launch holds more than 300 frames (grid.y);
- pretraining: dataloader.plan_frames to 192 x 352 at scales 0.95-1.05 and 1.125-1.5 from 360 x 640, 480 x 854,
  720 x 1280 and 640 x 360 frames, and wide and tall ones that hit the 64-pixel floor;
- evaluation: dataloader.plan_frames_eval to 384 x 704 (VCR), 384 x 384 (sort_story) and 192 x 352 (video_mc/qa/fib),
  with sources so wide or tall that one resized side is a few pixels, and video_mc's empty slot.

The bar.  Every operation of the kernel is an explicitly rounded float32 (or double, for the bicubic table) operation in the
TF source's order, and so is every operation of the oracle, so transforms 0 (none) and 1 (brightness) must match bit for bit
in every element, padding included.  Contrast needs the float32 mean of the padded image, a sum whose order TensorFlow leaves
open.  The kernel's mean is read back through `mean_ws` and must lie within X.mean_bound of the float64 mean of the
oracle's padded image: the kernel sums each channel with 512 threads that add ceil(npx / 512) pixels serially, a warp
butterfly (5 levels) and a serial sum of the 16 warp sums, then divides by npx; a pixel meets at most d = ceil(npx / 512) + 19
roundings, so |mean - exact| <= (gamma_d (1 + u) sum|x| + u |sum x|) / npx with u = 2^-24 (basis in X.mean_bound).  The contrast
output must then match the oracle's augment fed that mean bit for bit.

Every measured figure goes into a JSON report: $MERLOT_FRAMES_EXACT_REPORT if set, else a fresh file under the temporary
directory (its path is printed): per launch the frame count, the differing elements, the worst mean error against its bound,
and how many kernel means equal X.reduction_mean (one float32 order of the same shape; not asserted)."""
import json
import os
import tempfile
import time

import numpy as np
import pytest
import torch

from merlot_b200 import ops
from tests import frames_exact_oracle as X

pytestmark = pytest.mark.gpu
DEV = "cuda"
LAUNCHES = ["edges 15x17", "edges 1x1", "edges 7x37", "edges 1x257", "pretrain", "eval 384x704", "eval 384x384",
            "eval 192x352"]
_report = {"path": None, "data": {}}
_cases = []


def record(section, payload):
    if _report["path"] is None:
        _report["path"] = os.environ.get("MERLOT_FRAMES_EXACT_REPORT") or os.path.join(
            tempfile.mkdtemp(prefix="merlot_frames_exact_"), "frames_exact.json")
        print(f"frames-exact report: {_report['path']}")
    _report["data"][section] = payload
    with open(_report["path"], "w") as f:
        json.dump(_report["data"], f, indent=1, sort_keys=True)


def cases():
    if not _cases:
        _cases.extend(X.gpu_cases())
        assert [c["name"] for c in _cases] == LAUNCHES
    return _cases


def _first_difference(got, want):
    y, x, c = (int(v) for v in np.argwhere(got != want)[0])
    return f"first at (y {y}, x {x}, c {c}): got {got[y, x, c]!r}, want {want[y, x, c]!r}"


@pytest.mark.parametrize("name", LAUNCHES)
def test_frames_prepare_bit_exact(name):
    launch = cases()[LAUNCHES.index(name)]
    frames, (Hd, Wd) = launch["frames"], launch["out"]
    n = len(frames)
    packed, plan = X.launch_plan(launch)
    mean_ws = torch.full((n * 3,), float("nan"), dtype=torch.float32, device=DEV)
    t0 = time.perf_counter()
    out = ops.frames_prepare(torch.from_numpy(packed).to(DEV), plan, Hd, Wd, mean_ws=mean_ws)
    got = out.float().cpu().numpy()
    means = mean_ws.cpu().numpy().reshape(n, 3)
    t1 = time.perf_counter()
    resized = X.resized_frames(launch)
    diffs, mean_fails = [], []
    differing = 0
    worst_ratio = worst_abs = 0.0
    contrast = same_order = 0
    for k, f in enumerate(frames):
        img = resized[X.frame_key(f)]
        mean = None
        if f["augment"] == 2:
            contrast += 1
            mean = means[k]
            bound = X.mean_bound(img)
            err = np.abs(mean.astype(np.float64) - X.padded_mean(img))
            if not (err <= bound).all():  # NaN (a mean never written) fails too
                mean_fails.append(f"{X.frame_name(launch, f)}: mean {mean.tolist()} error {err.tolist()} > bound {bound.tolist()}")
            else:
                worst_ratio = max(worst_ratio, float((err / np.maximum(bound, 1e-300)).max()))
                worst_abs = max(worst_abs, float(err.max()))
            same_order += bool((mean == X.reduction_mean(img)).all())
        want = X.bf16_round(X.augment(img, f["augment"], f["factor"], mean))
        bad = got[k] != want  # NaN in the output counts as a difference
        if bad.any():
            differing += int(bad.sum())
            diffs.append(f"{X.frame_name(launch, f)}: {int(bad.sum())} elements, {_first_difference(got[k], want)}")
    record(name, {"frames": n, "out": [Hd, Wd], "elements": int(got.size), "differing_elements": differing,
                  "differing_frames": len(diffs), "first_differences": diffs[:20], "contrast_frames": contrast,
                  "mean_bound_failures": mean_fails[:20], "worst_mean_error_over_bound": worst_ratio,
                  "worst_mean_abs_error": worst_abs, "means_equal_to_reduction_mean": same_order,
                  "gpu_seconds_incl_copies": round(t1 - t0, 3), "oracle_seconds": round(time.perf_counter() - t1, 3)})
    assert not mean_fails, f"{len(mean_fails)} contrast means out of bound:\n" + "\n".join(mean_fails[:10])
    assert not diffs, f"{differing} elements differ in {len(diffs)} frames:\n" + "\n".join(diffs[:10])

