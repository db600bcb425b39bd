"""What share_params: False costs the configs[1] training step (bench.py's workload: merlot.yaml sizes, patch-embed ViT-B/16,
12 ViT + 12 language-only + 12 joint layers, 8 videos x 4 segments, hidden dropout 0.1, bf16 Adam moments).

Both stores are built in one process, True first:
1. torch.cuda.max_memory_allocated over each store's construction, warm-up and steps, less what was allocated before it;
2. ms per training step, CUDA events around --steps steps after --warmup, the two settings alternated over --rounds;
3. K10 (fused AdamW) over each arena, as the step runs it (optimizer.apply_gradients, every hyper-parameter group, gradient
   zeroing on): CUDA events over --iters calls, alternated over --rounds, with GB/s at 26 B per element.

Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/perf_share_params.py [--steps 10] [--warmup 3] [--rounds 3] [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BYTES_PER_ELEM = 26  # K10 with bf16 moments: read p, g, m, v; write p, m, v; bf16 copy; gradient zeroing


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def build(share):
    import torch
    from bench import PER_GPU_BATCH, load_config
    from merlot_b200.train import model_fn_builder, synthetic_batch
    config = load_config()
    config.model["share_params"] = share
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn = model_fn_builder(config, device="cuda")
    feats = synthetic_batch(config, PER_GPU_BATCH, seed=0)
    return fn, feats, base


def timed_steps(fn, feats, steps, warmup):
    import torch
    for _ in range(warmup):
        fn(feats).train_op()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        spec = fn(feats)
        spec.train_op()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, float(spec.loss)


def timed_adamw(fn, iters):
    import torch
    opt = fn.optimizer
    opt.apply_gradients(advance=False)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        opt.apply_gradients(advance=False)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_share_params.py needs a CUDA device")
    runs = {}
    for share in (True, False):
        fn, feats, base = build(share)
        timed_steps(fn, feats, args.steps, args.warmup)
        runs[share] = {"fn": fn, "feats": feats, "mem": (torch.cuda.max_memory_allocated() - base) / 2 ** 30}
    step_ms, adam_ms, loss = {True: [], False: []}, {True: [], False: []}, {}
    for _ in range(args.rounds):
        for share in (True, False):
            r = runs[share]
            ms, loss[share] = timed_steps(r["fn"], r["feats"], args.steps, args.warmup)
            step_ms[share].append(ms)
            adam_ms[share].append(timed_adamw(r["fn"], args.iters))
    out = {"card": card(), "workload": "configs[1] training step (bench.py), 8 videos x 4 segments, bf16 Adam moments"}
    for share in (True, False):
        st = runs[share]["fn"].store
        k10 = statistics.median(adam_ms[share])
        out[f"share_params_{share}"] = {
            "params": st.num_params(), "arena_elements": st.total, "max_memory_allocated_gib": round(runs[share]["mem"], 3),
            "ms_per_step": [round(x, 2) for x in step_ms[share]], "ms_per_step_median": round(statistics.median(step_ms[share]), 2),
            "k10_ms": [round(x, 3) for x in adam_ms[share]], "k10_ms_median": round(k10, 3),
            "k10_gb_per_s": round(BYTES_PER_ELEM * st.total / (k10 * 1e-3) / 1e9, 1), "loss_last": round(loss[share], 4)}
    a, b = out["share_params_True"], out["share_params_False"]
    out["delta"] = {"ms_per_step": round(b["ms_per_step_median"] - a["ms_per_step_median"], 2),
                    "k10_ms": round(b["k10_ms_median"] - a["k10_ms_median"], 3),
                    "max_memory_allocated_gib": round(b["max_memory_allocated_gib"] - a["max_memory_allocated_gib"], 3),
                    "params": b["params"] - a["params"]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
