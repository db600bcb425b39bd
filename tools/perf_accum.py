"""Gradient accumulation cost on one GPU: the configs[1] pretraining step (bench.py's workload: merlot.yaml sizes, patch-embed
ViT-B/16, 8 videos of 4 segments) as one batch (A = 1) against A = 4 micro-batches of 2 videos.  Per arm: ms per optimizer
step (host clock around steps that end in a device synchronise), the share of it spent in the features-only first pass
(model_fn), and the peak memory above the parameter store.  And K16, the contrastive head, forward + backward at
(n, nW) = (2048, 16384) (merlot.yaml on 8 GPUs) and (32, 32): us per call and TFLOP/s.  Prints one JSON line with the card's name and power limit.

    python tools/perf_accum.py [--steps 10] [--warmup 3]
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


def measure(A, m, steps, warmup):
    import torch
    from bench import load_config
    from merlot_b200.train import model_fn_builder, synthetic_batch
    config = load_config()
    fn = model_fn_builder(config, device="cuda")
    feats = [synthetic_batch(config, m, seed=j) for j in range(A)]
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    first = total = 0.0
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        spec = fn(feats if A > 1 else feats[0])
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        spec.train_op()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if i >= warmup:
            first += t1 - t0
            total += t2 - t0
    peak = torch.cuda.max_memory_allocated() - base
    out = {"A": A, "micro_batch": m, "ms_per_step": total / steps * 1e3, "peak_gib_above_params": peak / 2 ** 30,
           "loss": spec.loss}
    if A > 1:
        out["pass1_share"] = first / total
    del fn, feats, spec
    torch.cuda.empty_cache()
    return out


def k16(n, world, iters=20):
    """K16 forward + backward (contrastive_head + contrastive_head_bwd) at n local rows x n*world columns, Cs = 768: us per
    call (CUDA events) and TFLOP/s of the six tensor-core GEMMs counted from the shapes (3-term split: K tripled)."""
    import torch
    from merlot_b200.modeling import _Buffers, contrastive_head, contrastive_head_bwd

    class Store:
        device = "cuda"

    class Gather:  # every rank's rows: the all-gather without a collective (the GEMM work of rank 0 of `world`)
        def __init__(self):
            self.world, self.rank = world, 0

        def all_gather_rows(self, x):
            return x.repeat(world, 1)

        def reduce_scatter_rows(self, x_all):
            return x_all[:n]

    Cs = 768
    f = {k: torch.nn.functional.normalize(torch.randn(n, Cs, device="cuda"), dim=1) for k in ("lang", "viz")}
    bufs, dist = _Buffers(Store()), (Gather() if world > 1 else None)

    def once():
        info, _ = contrastive_head(bufs, {"contrast_temp": 0.05, "contrast_coef": 0.25}, dist, f["lang"], f["viz"], n)
        contrastive_head_bwd(bufs, dist, info)

    for _ in range(3):
        once()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        once()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / iters * 1e3
    nW = n * world
    flop = 2 * 2.0 * (n * nW * 3 * Cs + n * Cs * 3 * nW + nW * Cs * 3 * n)
    return {"n": n, "nW": nW, "us": us, "tflops": flop / us / 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_accum.py needs a CUDA device")
    res = {"card": card(), "workload": "configs[1] (bench.py), 8 videos x 4 segments per optimizer step",
           "arms": [measure(1, 8, args.steps, args.warmup), measure(4, 2, args.steps, args.warmup)],
           "k16": [k16(2048, 8), k16(32, 1)]}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
