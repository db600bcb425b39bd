"""K10 (fused AdamW) with bf16 and with fp32 moments, and what use_bfloat16_adam costs a training step.

1. Both K10 instances over the configs[1] arena (merlot.yaml sizes, patch-embed ViT-B/16: the ParamStore's padded element
   count) with the bf16 compute copy and gradient zeroing on, as the training step runs them: CUDA events over --iters
   launches after --warmup, the two instances alternated over --rounds.  Bytes are counted from the element count, 26 B
   (bf16 moments) and 34 B (fp32 moments) per element, and reported as GB/s and as a share of the H100 SXM data sheet's
   3.35 TB/s.
2. The configs[1] training step (bench.py's workload, 8 videos x 4 segments) with use_bfloat16_adam True and False,
   alternated over --rounds: ms per step (host clock around steps that end in a device synchronise) and
   torch.cuda.max_memory_allocated.

Prints one JSON line with the card's name and power limit.

    python tools/perf_adamw.py [--iters 50] [--warmup 5] [--rounds 3] [--steps 10] [--step-warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
BYTES_PER_ELEM = {"bf16": 26, "fp32": 34}  # read p, g, m, v; write p, m, v; bf16 copy 2 B; gradient zeroing 4 B


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def arena_size():
    from bench import load_config
    from merlot_b200.params import ParamStore
    config = load_config()
    return ParamStore(config.model, device="meta", optimizer_cfg=config.optimizer).total


def k10(n, iters, warmup, rounds):
    import torch
    from merlot_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(0)
    p = torch.randn(n, device="cuda", generator=gen) * 0.02
    g = torch.randn(n, device="cuda", generator=gen)
    pb = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    moments = {k: (torch.zeros(n, dtype=dt, device="cuda"), torch.zeros(n, dtype=dt, device="cuda"))
               for k, dt in (("bf16", torch.bfloat16), ("fp32", torch.float32))}

    def launch(kind):
        m, v = moments[kind]
        ops.adamw_step(p, g, m, v, pb, n, 0.9, 0.1, 0.98, 0.02, 1e-6, 1e-4, 0.1, 1.0, True)

    times = {k: [] for k in moments}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for kind in moments:
            for _ in range(warmup):
                launch(kind)
            e0.record()
            for _ in range(iters):
                launch(kind)
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1) / iters)
    out = {}
    for kind, ms in times.items():
        best = statistics.median(ms)
        byts = BYTES_PER_ELEM[kind] * n
        out[kind] = {"ms": ms, "ms_median": best, "bytes": byts, "gb_per_s": byts / best / 1e6,
                     "share_of_3p35_tb_s": byts / (best * 1e-3) / HBM_BYTES_PER_S, "bound_ms": byts / HBM_BYTES_PER_S * 1e3}
    out["fp32_over_bf16_bytes_per_s"] = out["fp32"]["gb_per_s"] / out["bf16"]["gb_per_s"]
    del p, g, pb, moments
    torch.cuda.empty_cache()
    return out


def step(use_bf16_adam, steps, warmup):
    import torch
    from bench import load_config
    from merlot_b200.train import model_fn_builder, synthetic_batch
    config = load_config()
    config.optimizer["use_bfloat16_adam"] = use_bf16_adam
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn = model_fn_builder(config, device="cuda")
    assert fn.store.m.dtype == (torch.bfloat16 if use_bf16_adam else torch.float32)
    feats = synthetic_batch(config, 8, seed=0)
    total = 0.0
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        spec = fn(feats)
        spec.train_op()
        torch.cuda.synchronize()
        if i >= warmup:
            total += time.perf_counter() - t0
    out = {"use_bfloat16_adam": use_bf16_adam, "ms_per_step": total / steps * 1e3,
           "max_memory_allocated_gib": torch.cuda.max_memory_allocated() / 2 ** 30, "loss": float(spec.loss)}
    del fn, feats, spec
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--step-warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_adamw.py needs a CUDA device")
    n = arena_size()
    res = {"card": card(), "arena_elements": n, "k10": k10(n, args.iters, args.warmup, args.rounds),
           "step": [step(flag, args.steps, args.step_warmup) for _ in range(args.rounds) for flag in (True, False)]}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
