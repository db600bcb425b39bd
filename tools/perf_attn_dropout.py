"""Cost of attention-probability dropout (attention_probs_dropout_prob) on the GPU.

1. K2 (forward), K3 (backward: dsum + K3 + dq finish, as merlot_attention_bwd launches them) and K4 (column sums) alone,
   CUDA-event timed, with p = 0 and p = 0.1, at the attention shapes of the configs[1] training step (ViT, language-only
   and joint stacks, read off one real step) and at S = 3608 (configs[4]'s joint sequence, B = 16).  The language-only and
   joint shapes run with an all-valid token mask, which selects the masked kernel instances the step uses there.
2. The configs[1] training step (bench.py's workload, fwd + bwd + AdamW) with attention_probs_dropout_prob 0.1 against
   0.0, alternated round by round on one parameter store.

Prints the card name and power limit with the numbers.  Usage: python tools/perf_attn_dropout.py [--rounds 4 --steps 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from merlot_b200 import ops  # noqa: E402

DEV = "cuda"
P_DROP = 0.1


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return (q.stdout.strip().splitlines() or [torch.cuda.get_device_name()])[0]


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us


def kernel_rows(name, B, S, masked, iters):
    heads, H = 12, 768
    g = torch.Generator().manual_seed(S)
    qkv = (torch.randn(B * S, 3 * H, generator=g) * 0.5).bfloat16().to(DEV)
    dctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16().to(DEV)
    valid = torch.ones(B * S, dtype=torch.uint8, device=DEV) if masked else None
    ctx = torch.empty(B * S, H, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, heads, S, device=DEV)
    dqkv = torch.empty(B * S, 3 * H, dtype=torch.bfloat16, device=DEV)
    ws = ops.attention_bwd_workspace(B, S, heads, DEV)
    dsum = torch.empty(B, heads, S, device=DEV)
    colsum = torch.zeros(B, S, device=DEV)
    res = {}
    for p in (0.0, P_DROP):
        drop = (p, 2 ** 32 + 1, 5)
        res[p] = (timed(lambda: ops.attention_fwd(qkv, B, S, heads, valid, ctx=ctx, lse=lse, dropout=drop), iters),
                  timed(lambda: ops.attention_bwd(qkv, ctx, dctx, lse, B, S, heads, valid, dqkv=dqkv, dq_accum=ws, dsum=dsum,
                                                  dropout=drop), iters),
                  timed(lambda: ops.attention_colsum(qkv, lse, colsum, B, S, heads, valid, dropout=drop), iters))
    for i, k in enumerate(("K2 fwd", "K3 bwd", "K4 colsum")):
        a, b = res[0.0][i], res[P_DROP][i]
        print(f"{name:34s} {k:10s} p=0: {a:9.1f} us   p={P_DROP}: {b:9.1f} us   +{(b / a - 1) * 100:5.1f} %", flush=True)
    del qkv, dctx, ctx, dqkv, ws


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    from merlot_b200.train import model_fn_builder, synthetic_batch
    config = bench.load_config()
    model_fn = model_fn_builder(config)
    feats = synthetic_batch(config, bench.PER_GPU_BATCH, seed=0, device=DEV)

    def step():
        spec = model_fn(feats, None, "train", None)
        spec.train_op()
        return spec

    config.model["attention_probs_dropout_prob"] = 0.0
    m = step().model
    torch.cuda.synchronize()
    d = m._dims
    lo = m.lang_transformer_info["hidden_state"].shape
    shapes = [(f"ViT B={d['N']} S={d['Sv']} (B*h={d['N'] * 12})", d["N"], d["Sv"], False, 20),
              (f"lang-only B={lo[0]} S={lo[1]}", lo[0], lo[1], True, 20),
              (f"joint B={m.B} S={d['Sj']}", m.B, d["Sj"], True, 20),
              ("configs[4] joint B=16 S=3608", 16, 3608, True, 3)]
    del m
    for name, B, S, masked, iters in shapes:
        kernel_rows(name, B, S, masked, iters)

    times = {0.0: [], P_DROP: []}
    for p in (0.0, P_DROP):  # warm both arms
        config.model["attention_probs_dropout_prob"] = p
        for _ in range(2):
            step()
    torch.cuda.synchronize()
    for r in range(args.rounds):
        for p in ((0.0, P_DROP) if r % 2 == 0 else (P_DROP, 0.0)):
            config.model["attention_probs_dropout_prob"] = p
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            times[p].append(e0.elapsed_time(e1) / args.steps)
    segs = bench.PER_GPU_BATCH * config.model["num_chunks_in_group"]
    for p, ts in times.items():
        print(f"configs[1] step attention_probs_dropout_prob={p}: median {statistics.median(ts):.2f} ms "
              f"(rounds {', '.join(f'{t:.2f}' for t in ts)}) = {segs / statistics.median(ts) * 1e3:.0f} segments/s", flush=True)
    a, b = statistics.median(times[0.0]), statistics.median(times[P_DROP])
    print(f"step cost of p={P_DROP}: +{b - a:.2f} ms (+{(b / a - 1) * 100:.1f} %)", flush=True)


if __name__ == "__main__":
    main()
