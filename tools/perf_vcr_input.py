"""Measure VCR fine-tuning and validation from records at merlot_vcr.yaml's sizes (384x704 images, hybrid stem, ViT-B +
12-layer joint encoder) on one GPU:

  1. the training pipeline alone (vcr_input, 8 questions = 16 images per batch, the per-GPU share of the YAML's 64 on 8
     GPUs): questions/s, host clock around batches that end in a device synchronise
  2. the VCR train step fed by that pipeline, alternated with the same step on resident synthetic batches (the step of
     tools/perf_vcr_step.py): ms/step of each, CUDA events
  3. the validator (vcr_validate.Validator, val_batch_size 64) on the answer and rationale modes, with every batch in one
     forward and in chunks: questions/s end to end (restore, pipeline, forwards) and the peak allocated memory

    python tools/perf_vcr_input.py [--questions 128] [--steps 10] [--rounds 2] [--chunks 64,16] [--out perf_vcr_input.json]

The records (JPEGs of 720x1280 and 540x960 at quality 95, the sizes of VCR's movie frames) are generated from a seed in a
temporary directory.  Prints one JSON object with the card's name and power limit and the host's CPU count.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from merlot_b200 import vcr_input as VI  # noqa: E402
from merlot_b200 import vcr_validate as VV  # noqa: E402
from perf_vcr_step import vcr_config  # noqa: E402
from tests import vcr_records as R  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return (q.stdout.strip().splitlines() or [torch.cuda.get_device_name()])[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=128, help="questions in the generated records")
    ap.add_argument("--batch", type=int, default=8, help="training questions per step")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--chunks", default="64,16", help="validator chunk sizes to measure")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_vcr_input.py needs a CUDA device")
    from merlot_b200.train import synthetic_vcr_batch
    from merlot_b200.vcr import vcr_model_fn_builder
    res = {"card": card(), "cpus": os.cpu_count()}
    with tempfile.TemporaryDirectory() as tmp:
        from pathlib import Path
        t = Path(tmp)
        t0 = time.perf_counter()
        sizes = [(720, 1280), (540, 960)]
        R.write_questions(t, [args.questions // 4] * 4, prefix="train", seed=0, sizes=sizes)
        R.write_questions(t, [args.questions // 4] * 4, prefix="val", seed=1, sizes=sizes)
        res["records_written_s"] = round(time.perf_counter() - t0, 1)
        cfg = vcr_config(args.batch)
        cfg.data.update(train_file_expanded=sorted(str(p) for p in t.glob("train-*.tfrecord")),
                        val_file_expanded=sorted(str(p) for p in t.glob("val-*.tfrecord")), draw="segm",
                        num_threads=os.cpu_count(), shuffle_buffer_size=64)
        cfg.device.update(output_dir=str(t / "out"), val_batch_size=64)
        cfg.validate = {"eval_samples": args.questions, "eval_timeout": 0}

        # 1. the pipeline alone
        with VI.input_fn_builder(cfg, is_training=True, batch_size=args.batch) as pipe:
            for _ in range(3):
                next(pipe)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = 4 * args.steps
            for _ in range(n):
                next(pipe)
            torch.cuda.synchronize()
            res["pipeline_questions_per_s"] = round(n * args.batch / (time.perf_counter() - t0), 1)

        # 2. the train step from records, alternated with the step on resident synthetic batches
        fn = vcr_model_fn_builder(cfg)
        synth = synthetic_vcr_batch(cfg, args.batch, seed=0)
        times = {"records": [], "synthetic": []}
        with VI.input_fn_builder(cfg, is_training=True, batch_size=args.batch) as pipe:
            for r in range(args.rounds + 1):
                for kind in ("synthetic", "records"):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        fn(next(pipe) if kind == "records" else synth).train_op()
                    e1.record()
                    torch.cuda.synchronize()
                    if r:  # round 0 warms up
                        times[kind].append(round(e0.elapsed_time(e1) / args.steps, 1))
        res["train_step_ms"] = times
        del fn, synth
        torch.cuda.empty_cache()

        # 3. the validator, per mode and chunk size, on a checkpoint of the initial weights
        store_fn = vcr_model_fn_builder(cfg)
        os.makedirs(cfg.device["output_dir"], exist_ok=True)
        prefix = os.path.join(cfg.device["output_dir"], "model.ckpt-0")
        store_fn.store.save_checkpoint(prefix)
        del store_fn
        torch.cuda.empty_cache()
        res["validator"] = []
        for mode in ("answer", "rationale"):
            cfg.downstream["mode"] = mode
            for chunk in [int(c) for c in args.chunks.split(",")]:
                v = VV.Validator(cfg, chunk=chunk)
                try:
                    v.evaluate(prefix)  # warm-up: every shape once
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    out = v.evaluate(prefix)
                    torch.cuda.synchronize()
                    s = time.perf_counter() - t0
                    res["validator"].append({"mode": mode, "chunk": chunk, "questions": out["questions"],
                                             "questions_per_s": round(out["questions"] / s, 1),
                                             "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)})
                except torch.OutOfMemoryError as e:
                    res["validator"].append({"mode": mode, "chunk": chunk, "out_of_memory": str(e).splitlines()[0]})
                del v
                torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
