"""Time fill-in-the-blank video QA (downstream.task: video_fib) on one GPU: the training step, the head's share of it and
the validator's forward.

One realistic size: 8 questions per GPU, 6 frames of 192x352 per question (6 x 67 viz tokens), sentence texts of 64 tokens
with one blank each, so the joint sequence is 6 * 67 + 64 = 466 tokens; A answers (`--answers`, default 1000 and 10000;
the answer layer stored as ceil(A/8)*8 columns), derived from the word embeddings of 1- to 3-token answers; merlot.yaml
widths with do_projection (the MLM head's projection and LayerNorm run), hidden dropout 0.1, the patch embedding or the
hybrid ResNet stem (`--stem patch,hybrid`).  Every question holds all six frames.  Measured with CUDA events around
`--steps` calls after `--warmup`:
  * the train step (video_fib_model_fn_builder "train": forward, head, backward, AdamW), with max_memory_allocated;
  * the head alone on the step's hidden state: fib_head + fib_loss (forward) and fib_head_backward (backward), and their
    share of the train step;
  * the eval forward the validator runs per batch ("eval": loss, accuracy and the counts).
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line per measurement.

Usage: python tools/perf_video_fib.py [--questions 8 --answers 1000,10000 --steps 10 --warmup 3 --stem patch,hybrid]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.perf_video_mc import card, timed  # noqa: E402


def answer_tokens(answers: int, vocab: int, directory: str) -> str:
    """A JSON answer vocabulary of `answers` distinct answers of 1 to 3 token ids each, written under `directory`."""
    rng = np.random.default_rng(0)
    out, seen = [], set()
    while len(out) < answers:
        a = tuple(int(t) for t in rng.integers(100, vocab, int(rng.integers(1, 4))))
        if a not in seen:
            seen.add(a)
            out.append(list(a))
    path = os.path.join(directory, f"answers-{answers}.json")
    with open(path, "w") as f:
        json.dump(out, f)
    return path


def video_fib_config(questions: int, answers: int, stem: str, directory: str):
    from merlot_b200.config import NeatConfig
    from tools.perf_video_mc import video_mc_config
    cfg = video_mc_config(questions, stem)
    model = dict(cfg.model, num_texts=1, do_projection=True)
    return NeatConfig.from_dict({"data": {}, "model": model, "optimizer": dict(cfg.optimizer),
                                 "device": {"use_tpu": False, "output_dir": os.path.join(directory, "out"),
                                            "train_batch_size": questions},
                                 "downstream": {"task": "video_fib", "max_text_len": 64,
                                                "answer_tokens": answer_tokens(answers, model["vocab_size"], directory)}})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=8)
    ap.add_argument("--answers", default="1000,10000")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--stem", default="patch,hybrid")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_video_fib.py needs a CUDA device")
    from merlot_b200 import video_fib as VF
    from merlot_b200.train import synthetic_video_fib_batch
    name = card()
    tmp = tempfile.mkdtemp(prefix="merlot_perf_video_fib_")
    for stem in args.stem.split(","):
        for A in (int(a) for a in args.answers.split(",")):
            cfg = video_fib_config(args.questions, A, stem, tmp)
            fn = VF.video_fib_model_fn_builder(cfg)
            store = fn.store
            feats = synthetic_video_fib_batch(cfg, args.questions, seed=0)
            feats["img_mask"].fill_(True)  # every question holds six frames
            what = f"{args.questions} questions x 6 frames 192x352, 64-token texts (Sj = 466), A = {A}, {stem} stem"
            losses = []

            def train():
                spec = fn(feats)
                spec.train_op()
                losses.append(spec.metrics["loss"])

            step_ms, peak = timed(train, args.steps, args.warmup)
            print(json.dumps({"workload": f"video_fib train step: {what}", "ms_per_call": round(step_ms, 2),
                              "questions_per_s": round(1e3 * args.questions / step_ms, 1),
                              "max_memory_allocated_gib": round(peak / 2 ** 30, 2),
                              "loss_first": round(float(losses[0]), 4), "loss_last": round(float(losses[-1]), 4),
                              "card": name}), flush=True)

            spec = fn(feats)  # a training forward whose hidden state the head runs on
            model = spec.model

            def head_forward():
                VF.fib_head(model, store, feats["blank_pos"])
                VF.fib_loss(model, feats["lm_targets"])

            def head_backward():
                VF.fib_head_backward(model, store)

            fwd_ms, _ = timed(head_forward, args.steps, args.warmup)
            bwd_ms, _ = timed(head_backward, args.steps, args.warmup)
            store.g.zero_()
            print(json.dumps({"workload": f"video_fib head: {what}", "forward_ms": round(fwd_ms, 3),
                              "backward_ms": round(bwd_ms, 3), "share_of_train_step": round((fwd_ms + bwd_ms) / step_ms, 4),
                              "card": name}), flush=True)
            del spec, model

            def evaluate():
                with torch.no_grad():
                    fn(feats, None, "eval")

            ms, peak = timed(evaluate, args.steps, args.warmup)
            print(json.dumps({"workload": f"video_fib validator eval forward per batch: {what}", "ms_per_call": round(ms, 2),
                              "questions_per_s": round(1e3 * args.questions / ms, 1),
                              "max_memory_allocated_gib": round(peak / 2 ** 30, 2), "card": name}), flush=True)
            del fn, feats, store
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
