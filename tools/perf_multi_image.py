"""Time one forward + backward of the joint encoder with several frames per text, at a size close to multi-frame video QA.

2 questions of 6 frames of 192x352 each (67 viz tokens per frame after the 2x2 pool), one frame of question 1 masked, 4
candidate texts of 64 tokens per question: B = 8 joint rows of P * num_imgs + L = 402 + 64 = 466 tokens; merlot.yaml's widths
(ViT-B over the patch-embed stem, 12 joint layers, hidden dropout 0.1).  One step = MerlotModel(is_training=True, img_mask=...)
then backward(d_hidden_state=...) from a fixed bf16 gradient, the pattern of a downstream head.  CUDA events around `--steps`
steps after `--warmup`; prints one JSON line with ms/step, torch.cuda.max_memory_allocated and the card's name and power limit
read in the same run.

Usage: python tools/perf_multi_image.py [--steps 10 --warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return (q.stdout.strip().splitlines() or [torch.cuda.get_device_name()])[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_multi_image.py needs a CUDA device")
    import bench
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import ParamStore
    questions, frames, texts, L = 2, 6, 4, 64
    cfg = dict(bench.load_config().model, num_imgs=frames, num_texts=texts, num_chunks_in_group=1)
    store = ParamStore(cfg, device="cuda")
    g = torch.Generator().manual_seed(0)
    image = torch.rand(questions * frames, 192, 352, 3, generator=g).to("cuda", torch.bfloat16)
    ids = torch.randint(100, 50357, (questions * texts, L), generator=g)
    ids[:, 48:] = 0
    ids = ids.int().cuda()
    mask = torch.ones(questions, frames, dtype=torch.bool)
    mask[1, 4] = False
    mask = mask.cuda()
    Sj, H = frames * 67 + L, cfg["hidden_size"]
    d_hidden = (torch.randn(questions * texts, Sj, H, generator=g) * 1e-3).to("cuda", torch.bfloat16)

    def step(i):
        m = MerlotModel(cfg, is_training=True, use_tpu=False, image=image, input_ids=ids, img_mask=mask, params=store,
                        dropout_seed=i)
        store.g.zero_()
        m.backward(d_hidden_state=d_hidden)
        return m

    for i in range(args.warmup):
        m = step(i)
    assert m._dims["Sj"] == Sj
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        step(args.warmup + i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    print(json.dumps({"workload": f"MerlotModel forward + backward(d_hidden_state), merlot.yaml widths: {questions} questions x "
                                  f"{frames} frames 192x352 (patch-embed stem), {questions * texts} texts x {L} tokens, Sj {Sj}",
                      "ms_per_step": round(ms, 2), "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                      "grad_norm_finite": bool(torch.isfinite(store.g).all()), "card": card()}))


if __name__ == "__main__":
    main()
