"""Time multiple-choice video QA (downstream.task: video_mc) on one GPU: the training step and the validator's forward.

One realistic size: 8 questions per GPU, 5 candidate answers, 6 frames of 192x352 per question (6 x 67 viz tokens), texts of
128 tokens, so the joint sequence is 6 * 67 + 128 = 530 tokens (past the attention backward's 512-token split); merlot.yaml
widths, hidden dropout 0.1, with the patch embedding and with the hybrid ResNet stem ([3, 4, 9]).  Every question holds all
six frames.  Per stem: the train step (video_mc_model_fn_builder "train": forward, head, backward, AdamW) and the eval
forward the validator runs ("eval", no dropout, loss and accuracy), CUDA events around `--steps` calls after `--warmup`;
questions/s and torch.cuda.max_memory_allocated of each, and the card's name, power limit and maximum SM clock read in the
same run.  Prints one JSON line per measurement.

Usage: python tools/perf_video_mc.py [--questions 8 --steps 10 --warmup 3 --stem patch,hybrid]
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


def video_mc_config(questions: int, stem: str):
    from merlot_b200.config import NeatConfig
    model = dict(transpose_input=False, num_imgs=6, num_texts=5, image_size=[192, 352], patch_size=16, spatial_pool_size=2,
                 use_bfloat16=True, vocab_size=50370, hidden_size=768, resnet_layers=[3, 4, 9] if stem == "hybrid" else [],
                 attention_probs_dropout_prob=0.0, hidden_dropout_prob=0.1, hidden_act="gelu", initializer_range=0.02,
                 intermediate_size=3072, max_position_embeddings=1024, num_attention_heads=12, num_hidden_layers=12,
                 num_vision_transformer_hidden_layers=12, num_lang_transformer_hidden_layers=12, share_params=True)
    optimizer = dict(type="adam_optimizer", learning_rate=0.000012, num_train_steps=60000, num_warmup_steps=6000,
                     weight_decay_rate=0.01, beta_2=0.98, clip_norm=0.0, adafactor=False, use_bfloat16_adam=True, verbose=False,
                     param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"],
                                       {"weight_decay_rate": 0}]])
    return NeatConfig.from_dict({"data": {}, "model": model, "optimizer": optimizer,
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_video_mc", "train_batch_size": questions},
                                 "downstream": {"task": "video_mc", "max_text_len": 128}})


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--stem", default="patch,hybrid")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_video_mc.py needs a CUDA device")
    from merlot_b200.train import synthetic_video_mc_batch
    from merlot_b200.video_mc import video_mc_model_fn_builder
    name = card()
    for stem in args.stem.split(","):
        cfg = video_mc_config(args.questions, stem)
        fn = video_mc_model_fn_builder(cfg)
        feats = synthetic_video_mc_batch(cfg, args.questions, seed=0)
        feats["img_mask"].fill_(True)  # every question holds six frames
        losses = []

        def train():
            spec = fn(feats)
            spec.train_op()
            losses.append(spec.metrics["loss"])

        def evaluate():
            with torch.no_grad():
                fn(feats, None, "eval")

        for what, f in (("train step", train), ("validator eval forward", evaluate)):
            ms, peak = timed(f, args.steps, args.warmup)
            out = {"workload": f"video_mc {what}, {stem} stem: {args.questions} questions x 6 frames 192x352, 5 choices x 128 "
                               f"tokens (Sj = 530)", "ms_per_call": round(ms, 2),
                   "questions_per_s": round(1e3 * args.questions / ms, 1),
                   "max_memory_allocated_gib": round(peak / 2 ** 30, 2), "card": name}
            if what == "train step":
                out.update(loss_first=round(float(losses[0]), 4), loss_last=round(float(losses[-1]), 4))
            print(json.dumps(out), flush=True)
        del fn, feats
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
