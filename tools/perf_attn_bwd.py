"""Time the attention backward (merlot_attention_bwd) alone on the GPU.

At the four shapes the model runs it at -- the ViT (B = 32, S = 266), the joint encoder (B = 8, S = 396), the language-only
stack (B = 8, S = 128) and configs[4]'s joint sequence (B = 16, S = 3608, the long-sequence K3 path) -- each with and without
the token mask (all tokens valid, which selects the masked kernel instances) and with attention-probability dropout p = 0 and
0.1.  12 heads of 64.  Each timing replays a CUDA graph of many backward calls after a warm-up, so host launch cost is out of
the number; CUDA events around the replays.  Prints microseconds per call and algorithmic TFLOP/s (10 B h S^2 64: S, dP, dV,
dK and dQ over all S keys, no discount for padding or masks), with the card's name, power limit and SM clock.

Usage: python tools/perf_attn_bwd.py [--reps 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from merlot_b200 import ops  # noqa: E402

DEV = "cuda"
HEADS, H = 12, 768
SHAPES = [("ViT", 32, 266), ("joint", 8, 396), ("lang-only", 8, 128), ("configs[4] joint", 16, 3608)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return (q.stdout.strip().splitlines() or [torch.cuda.get_device_name()])[0]


def time_graph(fn, calls, reps):
    """us per call: the median over `reps` replays of a graph of `calls` calls."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    g.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / calls * 1e3)
    del g
    return statistics.median(out), min(out), max(out)


def shape_rows(name, B, S, reps):
    g = torch.Generator().manual_seed(S)
    qkv = (torch.randn(B * S, 3 * H, generator=g) * 0.5).bfloat16().to(DEV)
    dctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16().to(DEV)
    dqkv = torch.empty(B * S, 3 * H, dtype=torch.bfloat16, device=DEV)
    ws = ops.attention_bwd_workspace(B, S, HEADS, DEV)
    dsum = torch.empty(B, HEADS, S, device=DEV)
    flops = 10.0 * B * HEADS * S * S * 64
    calls = max(3, min(200, int(40e-3 / (flops / 150e12))))  # about 40 ms of work per replay
    for masked in (False, True):
        valid = torch.ones(B * S, dtype=torch.uint8, device=DEV) if masked else None
        for p in (0.0, 0.1):
            drop = (p, 2 ** 32 + 1, 5)
            ctx, lse = ops.attention_fwd(qkv, B, S, HEADS, valid, dropout=drop)
            med, lo, hi = time_graph(lambda: ops.attention_bwd(qkv, ctx, dctx, lse, B, S, HEADS, valid, dqkv=dqkv, dq_accum=ws,
                                                               dsum=dsum, dropout=drop), calls, reps)
            print(f"{name:17s} B={B:2d} S={S:4d} mask={'on ' if masked else 'off'} p={p:.1f}: {med:9.1f} us "
                  f"(min {lo:.1f}, max {hi:.1f})  {flops / (med * 1e-6) / 1e12:6.1f} TFLOP/s", flush=True)
    del qkv, dctx, dqkv, ws, dsum


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    for name, B, S in SHAPES:
        shape_rows(name, B, S, args.reps)


if __name__ == "__main__":
    main()
