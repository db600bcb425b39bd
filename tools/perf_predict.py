"""Measure model_fn's PREDICT mode on one GPU at merlot.yaml's sizes (hybrid stem, 16 segments of 192 x 352 frames per
video, 32-token captions, val_batch_size 16), per batch of 16 videos on one resident evaluation batch:

  1. forward: MerlotModel as eval / predict build it (is_training=True, mask_input=True, nothing saved for backward)
     without an attention export, with the per-layer export (export_attention_probs=True) and with the layer-mean export
     ("layer_mean"), CUDA events over --iters forwards each; the export time is the difference to the forward without.
     (The layer-mean variant also takes attention_log from the exported map instead of K4's column sums.)
  2. max_memory_allocated above the memory held before each of the three forwards
  3. model_fn(..., "predict") end to end, and inside it the device-to-host copy (train.predictions) and the file write
     (predict.write_batch), host wall clock after a device synchronize

    python tools/perf_predict.py [--iters 5] [--out perf_predict.json]

Prints one JSON object with the card's name and power limit (queried in the same run).  Several GPUs are not measured.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

VAL_BATCH = 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_predict.py measures on a CUDA device")
    from perf_pretrain_validate import config_for
    from perf_input import SRC_HW
    from merlot_b200 import dataloader as D
    from merlot_b200 import predict as PR
    from merlot_b200 import train as T
    from merlot_b200.modeling import MerlotModel
    from tests import tfrecord_writer as W
    res = {"card": card(), "val_batch_size": VAL_BATCH, "multi_gpu": "not measured"}
    with tempfile.TemporaryDirectory() as tmp:
        rng = np.random.default_rng(0)
        recs = [W.chunks_example(W.video_chunks(rng, 16, frame_hw=SRC_HW, max_caption=40, video=f"v{e}"))
                for e in range(VAL_BATCH)]
        W.write_records(os.path.join(tmp, "val-000.tfrecord"), recs)
        config = config_for("hybrid", os.path.join(tmp, "val-*.tfrecord"), tmp)
        fn = T.model_fn_builder(config, seed=0)
        store = fn.store
        with torch.no_grad(), D.input_fn_builder(config, is_training=False, batch_size=VAL_BATCH) as pipe:
            batch = next(pipe)
        torch.cuda.synchronize()

        def forward(export):
            return MerlotModel(config.model, is_training=True, use_tpu=False, image=batch["images"],
                               input_ids=batch["input_ids"], shuffled_idx_img=batch["shuffled_idx_img"], mask_input=True,
                               params=store, save_for_backward=False, export_attention_probs=export)

        fwd = {}
        with torch.no_grad():
            for name, export in (("none", False), ("per_layer", True), ("layer_mean", "layer_mean")):
                forward(export)  # warm-up: buffers of this variant on the store
                torch.cuda.synchronize()
                before = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    m = forward(export)
                e1.record()
                torch.cuda.synchronize()
                if export == "layer_mean":
                    res["joint_map_shape"] = list(m.encoder_info["self_attn_probs"].shape)
                del m
                fwd[name] = {"forward_ms": round(e0.elapsed_time(e1) / args.iters, 2),
                             "peak_above_held_gib": round((torch.cuda.max_memory_allocated() - before) / 2 ** 30, 3),
                             "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)}
                store._bufs = {k: v for k, v in store._bufs.items() if not (isinstance(k, tuple) and k[0] == "joint.probs")}
                torch.cuda.empty_cache()
        for name in ("per_layer", "layer_mean"):
            fwd[name]["export_ms"] = round(fwd[name]["forward_ms"] - fwd["none"]["forward_ms"], 2)
        res["forward"] = fwd

        # model_fn "predict" end to end, with its device-to-host copy and the file write timed inside it
        d2h, write, total = [], [], []
        plain = T.predictions

        def timed_predictions(features, bsz):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = plain(features, bsz)
            d2h.append(time.perf_counter() - t0)
            return out
        T.predictions = timed_predictions
        out_dir = os.path.join(tmp, "pred")
        os.makedirs(out_dir)
        try:
            with torch.no_grad():
                for k in range(args.iters + 1):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    arrays = fn(batch, None, "predict", {"eval_batch": k, "batch_size": VAL_BATCH})
                    t1 = time.perf_counter()
                    PR.write_batch(out_dir, k, arrays)
                    t2 = time.perf_counter()
                    total.append(t1 - t0)
                    write.append(t2 - t1)
        finally:
            T.predictions = plain
        size = os.path.getsize(os.path.join(out_dir, PR.BATCH_FILE.format(0)))
        ms = lambda xs: round(1e3 * statistics.median(xs[1:]), 1)  # the first is a warm-up
        res["predict"] = {"model_fn_ms": ms(total), "device_to_host_ms": ms(d2h), "file_write_ms": ms(write),
                          "file_mib": round(size / 2 ** 20, 1),
                          "arrays": {k: list(v.shape) for k, v in arrays.items() if v.ndim > 2}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
