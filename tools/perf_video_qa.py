"""Time open-ended video QA (downstream.task: video_qa) on one GPU: the training step, the head's share of it and the
validator's forward.

One realistic size: 8 questions per GPU, 6 frames of 192x352 per question (6 x 67 viz tokens), question texts of 64 tokens,
so the joint sequence is 6 * 67 + 64 = 466 tokens; A = 1500 answers (the tower's output layer stored as 1504 columns);
merlot.yaml widths, hidden dropout 0.1, the patch embedding (or the hybrid ResNet stem with --stem hybrid).  Every question
holds all six frames.  Measured with CUDA events around `--steps` calls after `--warmup`:
  * the train step (video_qa_model_fn_builder "train": forward, head, backward, AdamW), with max_memory_allocated;
  * the head alone on the step's hidden state: qa_head + qa_loss (forward) and qa_head_backward (backward), and their share
    of the train step;
  * the eval forward the validator runs per batch ("eval": no dropout, loss, accuracy and the counts).
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line per measurement.

Usage: python tools/perf_video_qa.py [--questions 8 --answers 1500 --steps 10 --warmup 3 --stem patch]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.perf_video_mc import card, timed  # noqa: E402


def video_qa_config(questions: int, answers: int, stem: str):
    from merlot_b200.config import NeatConfig
    from tools.perf_video_mc import video_mc_config
    cfg = video_mc_config(questions, stem)
    model = dict(cfg.model, num_texts=1)
    return NeatConfig.from_dict({"data": {}, "model": model, "optimizer": dict(cfg.optimizer),
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_video_qa", "train_batch_size": questions},
                                 "downstream": {"task": "video_qa", "max_text_len": 64, "num_answers": answers}})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=8)
    ap.add_argument("--answers", type=int, default=1500)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--stem", default="patch")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_video_qa.py needs a CUDA device")
    from merlot_b200 import video_qa as VQ
    from merlot_b200.train import synthetic_video_qa_batch
    name = card()
    for stem in args.stem.split(","):
        cfg = video_qa_config(args.questions, args.answers, stem)
        fn = VQ.video_qa_model_fn_builder(cfg)
        store = fn.store
        feats = synthetic_video_qa_batch(cfg, args.questions, seed=0)
        feats["img_mask"].fill_(True)  # every question holds six frames
        what = (f"{args.questions} questions x 6 frames 192x352, 64-token texts (Sj = 466), A = {args.answers}, {stem} stem")
        losses = []

        def train():
            spec = fn(feats)
            spec.train_op()
            losses.append(spec.metrics["loss"])

        step_ms, peak = timed(train, args.steps, args.warmup)
        print(json.dumps({"workload": f"video_qa train step: {what}", "ms_per_call": round(step_ms, 2),
                          "questions_per_s": round(1e3 * args.questions / step_ms, 1),
                          "max_memory_allocated_gib": round(peak / 2 ** 30, 2), "loss_first": round(float(losses[0]), 4),
                          "loss_last": round(float(losses[-1]), 4), "card": name}), flush=True)

        spec = fn(feats)  # a training forward whose hidden state the head runs on
        model, p = spec.model, float(cfg.model["hidden_dropout_prob"])

        def head_forward():
            VQ.qa_head(model, store, dropout=(p, 1))
            VQ.qa_loss(model, feats["lm_targets"])

        def head_backward():
            VQ.qa_head_backward(model, store)

        fwd_ms, _ = timed(head_forward, args.steps, args.warmup)
        bwd_ms, _ = timed(head_backward, args.steps, args.warmup)
        store.g.zero_()
        print(json.dumps({"workload": f"video_qa head: {what}", "forward_ms": round(fwd_ms, 3), "backward_ms": round(bwd_ms, 3),
                          "share_of_train_step": round((fwd_ms + bwd_ms) / step_ms, 4), "card": name}), flush=True)
        del spec, model

        def evaluate():
            with torch.no_grad():
                fn(feats, None, "eval")

        ms, peak = timed(evaluate, args.steps, args.warmup)
        print(json.dumps({"workload": f"video_qa validator eval forward per batch: {what}", "ms_per_call": round(ms, 2),
                          "questions_per_s": round(1e3 * args.questions / ms, 1),
                          "max_memory_allocated_gib": round(peak / 2 ** 30, 2), "card": name}), flush=True)
        del fn, feats
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
