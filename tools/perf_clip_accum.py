"""Cost of per-micro-batch clipping under gradient accumulation on one GPU: bench.py's configs[1] pretraining step (merlot.yaml
sizes, patch-embed ViT-B/16) as A = 4 micro-batches of 2 videos, with clip_norm 0 and 1.0 alternating step by step on two
models in the same process.  Per arm: ms per optimizer step (host clock around steps that end in a device synchronise) and
its own max_memory_allocated (store, step buffers and, when clipping, the accumulator).  And ops.clip_accumulate alone over
a 223.4 M-element arena: ms per call (CUDA events) and bytes/s at 20 B per element against the H100 SXM's 3.35 TB/s.
Prints one JSON line with the card's name and power limit.

    python tools/perf_clip_accum.py [--steps 8] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def steps(A, m, n_steps, warmup):
    import torch
    from bench import load_config
    from merlot_b200.params import ParamStore
    from merlot_b200.train import model_fn_builder, synthetic_batch
    arms = {}
    feats = [synthetic_batch(load_config(), m, seed=j) for j in range(A)]
    for clip in (0.0, 1.0):
        # the arm's own footprint: max_memory_allocated from before its store is built through its first step, less what
        # was allocated before (the other arm's store and buffers)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        config = load_config()
        config.optimizer["clip_norm"] = clip
        store = ParamStore(config.model, device="cuda", optimizer_cfg=config.optimizer)
        store.init_reference(seed=0)
        fn = model_fn_builder(config, store=store, device="cuda")
        fn(feats).train_op()
        torch.cuda.synchronize()
        arms[clip] = dict(fn=fn, ms=[], peak=torch.cuda.max_memory_allocated() - base)
    for i in range(warmup + n_steps):
        for clip, arm in arms.items():  # alternate the two arms step by step
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            spec = arm["fn"](feats)
            spec.train_op()
            torch.cuda.synchronize()
            if i >= warmup:
                arm["ms"].append((time.perf_counter() - t0) * 1e3)
            arm["loss"] = spec.loss
            arm["gradnorm"] = float(spec.metrics["gradnorms/_overall"]) if clip > 0 else None
    out = []
    for clip, arm in arms.items():
        ms = sorted(arm["ms"])
        out.append({"clip_norm": clip, "A": A, "micro_batch": m, "ms_per_step_median": ms[len(ms) // 2],
                    "ms_per_step_min": ms[0], "ms_per_step_max": ms[-1],
                    "max_memory_allocated_gib_of_arm": arm["peak"] / 2 ** 30, "g_acc_allocated": arm["fn"].store.g_acc is not None,
                    "loss": arm["loss"], "gradnorms/_overall": arm["gradnorm"]})
    return out


def kernel(n=223_430_272, iters=20):
    import torch
    from merlot_b200 import ops
    acc = torch.zeros(n, device="cuda")
    g = torch.randn(n, device="cuda")
    scratch = torch.zeros(1, dtype=torch.float64, device="cuda")
    norm = torch.zeros(1, dtype=torch.float32, device="cuda")
    for _ in range(3):
        ops.clip_accumulate(acc, g, 1.0, scratch, norm)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.clip_accumulate(acc, g, 1.0, scratch, norm)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    nbytes = 20 * n
    return {"elements": n, "ms": ms, "bytes": nbytes, "tb_per_s": nbytes / ms / 1e9, "share_of_3.35_tb_per_s": nbytes / ms / 1e9 / 3.35}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_clip_accum.py needs a CUDA device")
    res = {"card": card(), "workload": "configs[1] (bench.py), A = 4 micro-batches of 2 videos x 4 segments per optimizer step",
           "kernel": kernel(), "arms": steps(4, 2, args.steps, args.warmup)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
