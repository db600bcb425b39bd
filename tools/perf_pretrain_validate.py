"""Measure pretraining validation on one GPU at merlot.yaml's sizes (16 segments of 192 x 352 frames per video from 288 x 512
JPEGs, 32-token captions, val_batch_size 16), with the patch-embed stem and with the hybrid stem:

  1. end to end: pretrain_validate.Validator.evaluate on one checkpoint (restore, evaluation input, eval forwards, means),
     after one warm-up evaluate: videos/s
  2. forward time per batch: model_fn(..., "eval") on one resident batch of 16 videos, CUDA events over --iters calls
  3. memory per batch: the device buffers the eval forward keeps on the store (reused by every later batch) and the
     transient peak of one more forward above them (max_memory_allocated over memory_allocated before it)

    python tools/perf_pretrain_validate.py [--batches 6] [--iters 10] [--out perf_pretrain_validate.json]

The records are generated from a seed in a temporary directory.  Prints one JSON object with the card's name and power
limit (queried in the same run) and the host's CPU count.  Several GPUs are not measured here.
"""
import argparse
import json
import os
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


def config_for(stem, val_glob, out_dir):
    import bench
    from perf_input import MERLOT_DATA
    config = bench.load_config()
    config.model["resnet_layers"] = [3, 4, 9] if stem == "hybrid" else []  # model/configs/merlot.yaml:33
    config.data = dict(MERLOT_DATA, val_file=val_glob)
    config.data.pop("val_file_expanded", None)
    config.device.update(output_dir=out_dir, val_batch_size=VAL_BATCH)
    config.validate = {}
    return config


def forward_buffer_bytes(store):
    """Bytes of the named device buffers the forwards on `store` keep (modeling._Buffers)."""
    def size(x):
        if torch.is_tensor(x):
            return x.numel() * x.element_size() if x.is_cuda else 0
        if isinstance(x, (tuple, list)):
            return sum(size(y) for y in x)
        if isinstance(x, dict):
            return sum(size(y) for y in x.values())
        return 0
    return sum(size(x) for x in getattr(store, "_bufs", {}).values())


def measure(stem, val_glob, tmp, iters):
    from merlot_b200 import dataloader as D
    from merlot_b200.pretrain_validate import Validator
    out_dir = os.path.join(tmp, stem)
    os.makedirs(out_dir)
    config = config_for(stem, val_glob, out_dir)
    v = Validator(config)
    prefix = os.path.join(out_dir, "model.ckpt-0")
    v.store.init_reference(seed=0)
    v.store.save_checkpoint(prefix)
    v.evaluate(prefix)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = v.evaluate(prefix)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    with torch.no_grad(), D.input_fn_builder(config, is_training=False, batch_size=VAL_BATCH) as pipe:
        batch = next(pipe)
        v.model_fn(batch, None, "eval")
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        v.model_fn(batch, None, "eval")
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - before
        held = forward_buffer_bytes(v.store)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(iters):
            v.model_fn(batch, None, "eval", {"eval_batch": k})
        e1.record()
        torch.cuda.synchronize()
        fwd_ms = e0.elapsed_time(e1) / iters
    out = {"stem": stem, "videos": res["videos"], "end_to_end_s": round(seconds, 3),
           "videos_per_s": round(res["videos"] / seconds, 1), "forward_ms_per_batch": round(fwd_ms, 2),
           "forward_buffers_gib": round(held / 2 ** 30, 3), "transient_peak_per_batch_gib": round(peak / 2 ** 30, 3),
           "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), "loss": res["loss"]}
    del v, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=6, help="whole batches of 16 videos in the evaluation records")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_pretrain_validate.py measures on a CUDA device")
    from perf_input import SRC_HW
    from tests import tfrecord_writer as W
    res = {"card": card(), "cpus": len(os.sched_getaffinity(0)), "val_batch_size": VAL_BATCH, "multi_gpu": "not measured",
           "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        rng = np.random.default_rng(0)
        n = args.batches * VAL_BATCH
        recs = [W.chunks_example(W.video_chunks(rng, 16, frame_hw=SRC_HW, max_caption=40, video=f"v{e}")) for e in range(n)]
        for f in range(4):
            W.write_records(os.path.join(tmp, f"val-{f:03d}.tfrecord"), recs[f::4])
        res["records_written_s"] = round(time.perf_counter() - t0, 1)
        for stem in ("patch", "hybrid"):
            res["runs"].append(measure(stem, os.path.join(tmp, "val-*.tfrecord"), tmp, args.iters))
            print(json.dumps(res["runs"][-1]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
