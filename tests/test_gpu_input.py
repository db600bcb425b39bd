"""GPU tests of the pretraining input (pytest -m gpu): K14 (merlot_frames_prepare) against tests/input_oracle.py on frames of
mixed odd sizes for every resize method x {none, brightness, contrast}; tfrecords -> input_fn_builder -> one batch against the
oracle pipeline and one training step on it; and the trainer reading tfrecords in a subprocess."""
import io
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import dataloader as D
from merlot_b200 import ops
from merlot_b200.config import NeatConfig
from oracle.oracle_np import process_example_np
from tests import frames_exact_oracle as X
from tests import input_oracle as O
from tests import tfrecord_writer as W
from tests.gemm_exact_oracle import bf16_ulps

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(got, ref, what):
    # every operation of K14 and of the oracle is one float32 rounding in the TF source's order, so the outputs are equal
    # bit for bit; contrast frames are checked against the oracle fed the kernel's own mean (_contrast_mean bounds it)
    bad = got != ref
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ, first at {np.argwhere(bad)[0].tolist()}"


def _contrast_mean(mean, img, what):
    """The kernel's float32 contrast mean against the float64 mean of the oracle's padded image, within the bound of its
    reduction (tests/frames_exact_oracle.py:mean_bound)."""
    err = np.abs(mean.astype(np.float64) - X.padded_mean(img))
    assert (err <= X.mean_bound(img)).all(), f"{what}: mean {mean.tolist()} error {err.tolist()}"
    return mean


# ---- K14 against the oracle -------------------------------------------------------------------------------------------
OUT = (24, 40)
SOURCES = [(37, 53), (61, 29), (20, 90), (9, 13), (48, 64), (31, 47)]


def _frames():
    """(source index, scaled_h, scaled_w, offset_y, offset_x): upscaling with a non-zero crop, downscaling with padding on
    both sides, 1-pixel resizes, a same-size resize, and plans of resize_and_pad (incl. the 64-pixel floor of the wide frame)."""
    explicit = [(0, 55, 80, 7, 13), (1, 30, 15, 0, 0), (3, 1, 1, 0, 0), (3, 1, 50, 0, 5), (3, 40, 1, 9, 0), (4, 48, 64, 5, 3),
                (5, 23, 70, 0, 21)]
    planned = []
    for si, s in [(2, 1.0), (0, 1.3), (5, 0.7), (1, 1.125)]:
        h, w = SOURCES[si]
        p = O.resize_plan(h, w, OUT, s, 0.37, 0.81)
        planned.append((si,) + p)
    assert planned[0][1] == 64  # the wide 20 x 90 frame hits the 64-pixel floor
    return explicit + planned


def test_frames_prepare_matches_oracle():
    rng = np.random.default_rng(5)
    srcs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in SOURCES]
    offs = np.concatenate([[0], np.cumsum([s.size for s in srcs])[:-1]])
    packed = torch.from_numpy(np.concatenate([s.reshape(-1) for s in srcs])).cuda()
    frames = _frames()
    rows = []  # every frame under every method and transform, all in ONE launch (mixed sizes)
    for m in range(4):
        for t in range(3):
            for f in frames:
                rows.append((m, t) + f + (tuple(rng.uniform(0.68, 1.32, 3).astype(np.float32)),))
    plan = {k: [] for k in ops.FRAME_FIELDS + ("factor",)}
    for m, t, si, sh, sw, oy, ox, fac in rows:
        for k, v in zip(ops.FRAME_FIELDS + ("factor",), (offs[si], *SOURCES[si], sh, sw, oy, ox, m, t, fac)):
            plan[k].append(v)
    mean_ws = torch.full((len(rows) * 3,), float("nan"), dtype=torch.float32, device="cuda")
    got = ops.frames_prepare(packed, plan, *OUT, mean_ws=mean_ws).float().cpu().numpy()
    means = mean_ws.cpu().numpy().reshape(-1, 3)
    assert got.shape == (len(rows),) + OUT + (3,)
    resized = {}
    for i, (m, t, si, sh, sw, oy, ox, fac) in enumerate(rows):
        key = (m, si, sh, sw, oy, ox)
        if key not in resized:
            resized[key] = O.resize_and_pad(srcs[si].astype(np.float32) * O.INV255, OUT, sh, sw, oy, ox, m)
        ref = np.where(np.isfinite(resized[key]), resized[key], np.float32(0))
        what = f"{O.METHODS[m]} transform {t} source {SOURCES[si]} -> ({sh}, {sw}) at ({oy}, {ox})"
        if t == 2:
            ref = X.augment(ref, t, fac, _contrast_mean(means[i], ref, what))
        else:
            ref = O.augment(ref, t, fac)
        _check(got[i], O.bf16_round(ref), what)
        if t == 0 and (sh < OUT[0] or sw < OUT[1]):
            assert (got[i][sh - oy:] == 0).all() and (got[i][:, sw - ox:] == 0).all()  # zero padding, bottom and right


# ---- tfrecords -> input_fn_builder -> batch, against the oracle pipeline ----------------------------------------------
def _write_dataset(tmp_path, files=3, per_file=3, num_chunks=4, vocab=1000):
    rng = np.random.default_rng(17)
    sizes = [(70, 100), (66, 99), (81, 123), (64, 96)]
    by_record = {}
    for fi in range(files):
        recs = []
        for e in range(per_file):
            chunks = W.video_chunks(rng, num_chunks, frame_hw=lambda i: sizes[(i + e) % len(sizes)], max_caption=24,
                                    video=f"f{fi}e{e}", vocab=vocab)
            rec = W.chunks_example(chunks)
            by_record[rec] = chunks
            recs.append(rec)
        W.write_records(tmp_path / f"train-{fi:02d}.tfrecord", recs)
    return by_record


def _config(tmp_path, tiny_cfg, steps=3):
    model = dict(tiny_cfg, image_size=[64, 96], num_chunks_in_group=2)
    return {"data": {"train_file": str(tmp_path / "train-*.tfrecord"), "num_chunks": 4, "chunk_text_len": 16,
                     "random_scale_min": 1.125, "random_scale_max": 1.5, "augment_prob": 0.8, "clean_asr_prob": 0.5,
                     "shuffle_chunks": True, "num_threads": 4, "shuffle_buffer_size": 4},
            "model": model,
            "optimizer": {"type": "adam_optimizer", "learning_rate": 3e-4, "num_train_steps": steps, "num_warmup_steps": 1,
                          "weight_decay_rate": 0.1, "beta_2": 0.98, "clip_norm": 0.0, "use_bfloat16_adam": True},
            "device": {"output_dir": str(tmp_path / "out"), "train_batch_size": 2}}


def _oracle_batch(info, by_record, data, model):
    from PIL import Image
    n, L, out = data["num_chunks"], data["chunk_text_len"], tuple(model["image_size"])
    fd = info["frame_draws"]
    texts, images = [], []
    for e, rec in enumerate(info["records"]):
        chunks = by_record[rec]
        texts.append(O.dataset_parser_text(chunks, L, bool(info["do_clean"][e])))
        for j, c in enumerate(chunks):
            k = e * n + j
            u8 = np.asarray(Image.open(io.BytesIO(c["image/encoded"])).convert("RGB"))
            img, _ = O.load_and_resize_img(u8, out, fd["scale"][k], fd["u_y"][k], fd["u_x"][k], fd["method"][k], fd["augment"][k],
                                           fd["factor"][k])
            images.append(img)
    feats = {k: np.stack([t[k] for t in texts]) for k in texts[0]}
    feats["images"] = np.stack(images).reshape(len(texts), n, *out, 3)
    feats["contrast"] = (np.asarray(fd["augment"]) == 2).reshape(len(texts), n)  # follows its frame through the shuffle
    pd = {k: v.numpy() for k, v in info["process_draws"].items()}
    idx, shuffled = process_example_np(feats["input_ids"], feats["video_src_ids"], pd["chunk_u"], pd["num_shuffle"], pd["pick_u"],
                                       pd["order_u"], model["num_chunks_in_group"], model["image_shuffle_prob"],
                                       data["shuffle_chunks"])
    feats = {k: np.take_along_axis(v, idx.reshape(idx.shape + (1,) * (v.ndim - 2)), 1) for k, v in feats.items()}
    feats["images"] = feats["images"].reshape(-1, *out, 3)
    feats["contrast"] = feats["contrast"].reshape(-1)
    feats["shuffled_idx_img"] = shuffled
    return feats


def test_input_pipeline_batch_matches_oracle_and_trains(tmp_path, tiny_cfg):
    from merlot_b200.train import model_fn_builder
    by_record = _write_dataset(tmp_path)
    cfg = _config(tmp_path, tiny_cfg)
    config = NeatConfig.from_dict(cfg)
    with D.input_fn_builder(config, True, seed=5) as pipe:
        feats = next(pipe)
        info = pipe.last_info
        torch.cuda.synchronize()
        ref = _oracle_batch(info, by_record, cfg["data"], cfg["model"])
        assert feats["images"].shape == (2 * 4, 64, 96, 3) and feats["images"].dtype == torch.bfloat16
        assert feats["input_ids"].shape == (2, 4, 16)
        for k in ("input_ids", "video_src_ids", "youtube_id", "chunk_num", "mean_time", "is_eoc", "shuffled_idx_img"):
            np.testing.assert_array_equal(feats[k].cpu().numpy(), ref[k], err_msg=k)
        got = feats["images"].float().cpu().numpy()
        d = bf16_ulps(got, ref["images"])
        c = ref["contrast"]
        assert d[~c].max(initial=0) == 0, int((d[~c] > 0).sum())  # bit-exact, as in the K14 test
        if c.any():  # the oracle's contrast mean is the float64 one, the kernel's a float32 sum
            assert d[c].max() <= 1 and (d[c] > 0).mean() <= 0.005, (int(d[c].max()), float((d[c] > 0).mean()))
        model_fn = model_fn_builder(config, device="cuda")
        spec = model_fn(feats, None, "train", None)
        spec.train_op()
        torch.cuda.synchronize()
        losses = [float(x) for x in spec.loss_parts]
        assert all(np.isfinite(losses)), losses
        next(pipe)  # a second batch is ready behind the first
    assert not [t.name for t in threading.enumerate() if t.name.startswith("merlot-")]


def test_trainer_reads_tfrecords(tmp_path, tiny_cfg):
    _write_dataset(tmp_path)
    path = tmp_path / "tiny.yaml"
    path.write_text(yaml.safe_dump(_config(tmp_path, tiny_cfg, steps=3)))
    code = ("import runpy, sys, threading\n"
            f"sys.argv = ['merlot_b200.train', {str(path)!r}]\n"
            "runpy.run_module('merlot_b200.train', run_name='__main__')\n"
            "print('LEFT', [t.name for t in threading.enumerate() if t.name.startswith('merlot-')])\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "step 0 loss" in r.stdout and "synthetic" not in r.stdout, r.stdout
    assert "LEFT []" in r.stdout, r.stdout
