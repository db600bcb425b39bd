"""Time the VCR fine-tuning step at merlot_vcr.yaml's per-GPU sizes on one GPU.

The step is vcr_model_fn_builder's train step exactly as `python -m merlot_b200.train merlot_vcr.yaml` runs it on one of the
8 GPUs of the reference's batch: 8 questions = 16 images of 384x704 through the hybrid ResNet stem ([3, 4, 9]) and the ViT,
64 candidate texts of 184 tokens through the joint encoder (265 + 184 tokens), the answer / rationale towers, backward and
AdamW, hidden dropout 0.1.  CUDA events around `--steps` steps after `--warmup` steps; prints one JSON line with ms/step,
questions/s, torch.cuda.max_memory_allocated and the card's name and power limit read in the same run.

Usage: python tools/perf_vcr_step.py [--questions 8 --steps 10 --warmup 3]
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


def vcr_config(train_batch_size):
    """merlot_vcr.yaml's model / optimizer / downstream sections (init_checkpoint left out: weights are the initialisers)."""
    from merlot_b200.config import NeatConfig
    model = dict(transpose_input=True, num_texts=4, image_size=[384, 704], patch_size=16, spatial_pool_size=2, use_bfloat16=True,
                 vocab_size=50370, hidden_size=768, resnet_layers=[3, 4, 9], attention_probs_dropout_prob=0.0,
                 hidden_dropout_prob=0.1, hidden_act="gelu", initializer_range=0.02, intermediate_size=3072,
                 max_position_embeddings=1024, num_attention_heads=12, num_hidden_layers=12,
                 num_vision_transformer_hidden_layers=12, num_lang_transformer_hidden_layers=12, share_params=True)
    optimizer = dict(type="adam_optimizer", learning_rate=0.000012, num_train_steps=60000, num_warmup_steps=6000,
                     weight_decay_rate=0.01, beta_2=0.98, clip_norm=0.0, adafactor=False, use_bfloat16_adam=True, verbose=False,
                     param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"],
                                       {"weight_decay_rate": 0}]])
    return NeatConfig.from_dict({"data": {}, "model": model, "optimizer": optimizer,
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_vcr", "train_batch_size": train_batch_size},
                                 "downstream": {"task": "vcr", "mode": "answer"}})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_vcr_step.py needs a CUDA device")
    from merlot_b200.train import synthetic_vcr_batch
    from merlot_b200.vcr import vcr_model_fn_builder
    cfg = vcr_config(args.questions)
    fn = vcr_model_fn_builder(cfg)
    feats = synthetic_vcr_batch(cfg, args.questions, seed=0)
    losses = []

    def step():
        spec = fn(feats)
        spec.train_op()
        losses.append(spec.metrics["loss"])

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    print(json.dumps({"workload": f"VCR train step, merlot_vcr.yaml per-GPU sizes: {args.questions} questions, "
                                  f"{2 * args.questions} images 384x704 (hybrid stem), {8 * args.questions} texts x 184 tokens",
                      "ms_per_step": round(ms, 2), "questions_per_s": round(1e3 * args.questions / ms, 1),
                      "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                      "loss_first": round(float(losses[0]), 4), "loss_last": round(float(losses[-1]), 4), "card": card()}))


if __name__ == "__main__":
    main()
