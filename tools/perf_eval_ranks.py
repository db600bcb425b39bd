"""Measure the evaluation programs end to end on 1, 2 and 4 ranks (one process per rank, as torchrun starts them; the
ranks share the visible GPUs round-robin, so on a one-GPU host they share the card):

  1. VCR validation: vcr_validate.Validator.evaluate on a checkpoint at merlot_vcr.yaml's sizes (hybrid stem, 384x704,
     val_batch_size 64, --chunk 16 so that four ranks fit one 80 GB card), answer mode: questions/s from the start of
     evaluate (restore, pipeline, forwards, gather) to its end on every rank, after one warm-up evaluate
  2. story unshuffling: sort_story.gather_story_rows (restore, pipeline, zero-shot forwards, gather) at merlot_5segments.yaml's
     sizes, 8 stories per batch: stories/s, after one warm-up pass

    python tools/perf_eval_ranks.py [--ranks 1,2,4] [--questions 256] [--stories 192] [--out perf_eval_ranks.json]

data.num_threads is left at its default, so every rank runs 64 // ranks decode threads (eval_decode_threads).  The
records are generated from a seed in a temporary directory (tools/perf_vcr_input.py's and tools/perf_sort_story.py's
JPEG sizes).  Prints one JSON object with the card's name, power limit and SM clock limit, the host's CPU count and the
decode threads per rank.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile
import time
import traceback

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

STORY_BATCH = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines() or [torch.cuda.get_device_name()]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _timed(group, fn):
    """fn() once to warm up, then once timed; every rank starts the timed call after every rank finished the warm-up."""
    fn()
    torch.cuda.synchronize()
    group.agree(None)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def _vcr(group, cfg_dict, prefix, chunk):
    from merlot_b200.config import NeatConfig
    from merlot_b200.vcr_validate import Validator
    v = Validator(NeatConfig.from_dict(cfg_dict), chunk=chunk, group=group)
    res, s = _timed(group, lambda: v.evaluate(prefix))
    return {"questions": res["questions"], "seconds": round(s, 2), "questions_per_s": round(res["questions"] / s, 1),
            "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def _story(group, cfg_dict, prefix):
    from merlot_b200.config import NeatConfig
    from merlot_b200.sort_story import gather_story_rows
    config = NeatConfig.from_dict(cfg_dict)
    (batches, dropped), s = _timed(group, lambda: gather_story_rows(config, prefix, group))
    n = sum(len(b) for b in batches)
    return {"stories": n, "dropped": dropped, "seconds": round(s, 2), "stories_per_s": round(n / s, 1),
            "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def _rank_main(rank, world, port, what, args, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    try:
        from merlot_b200.dataloader import eval_decode_threads
        from merlot_b200.eval_ranks import backend, eval_group
        with eval_group() as group:
            out = {"vcr": _vcr, "story": _story}[what](group, *args)
        out.update(decode_threads=eval_decode_threads(args[0]["data"]), backend=backend() if world > 1 else None,
                   device=torch.cuda.current_device())
        q.put({"rank": rank, "out": out})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


def run_ranks(world, what, *args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_rank_main, args=(r, world, port, what, args, q)) for r in range(world)]
    try:
        for p in ps:
            p.start()
        res = sorted((q.get(timeout=1800) for _ in range(world)), key=lambda r: r["rank"])
    finally:
        for p in ps:
            p.join(timeout=300)
            if p.is_alive():
                p.kill()
                p.join()
    errors = [r["error"] for r in res if "error" in r]
    if errors:
        return {"ranks": world, "error": errors[0].strip().splitlines()[-1]}
    out = dict(res[0]["out"], ranks=world)  # every rank returns the gathered result; rank 0's clock
    out["max_memory_allocated_gib"] = [r["out"]["max_memory_allocated_gib"] for r in res]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", default="1,2,4")
    ap.add_argument("--questions", type=int, default=256, help="VCR validation questions (in batches of 64)")
    ap.add_argument("--stories", type=int, default=192, help="stories (in batches of 8)")
    ap.add_argument("--chunk", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_eval_ranks.py measures on CUDA devices")
    from pathlib import Path
    from merlot_b200.params import ParamStore
    from merlot_b200.tf_checkpoint import update_checkpoint_state
    from merlot_b200.vcr import vcr_model_fn_builder
    from perf_vcr_step import vcr_config
    from tests import story_records as SR
    from tests import tfrecord_writer as W
    from tests import vcr_records as R
    res = {"card": card(), "gpus": torch.cuda.device_count(), "cpus": len(os.sched_getaffinity(0)), "vcr": [], "story": []}
    ranks = [int(x) for x in args.ranks.split(",")]
    with tempfile.TemporaryDirectory() as tmp:
        t = Path(tmp)
        t0 = time.perf_counter()
        R.write_questions(t, [args.questions // 4] * 4, prefix="val", seed=1, sizes=[(720, 1280), (540, 960)])
        rng = np.random.default_rng(0)
        recs = [SR.story_example(SR.story(rng, k, sizes=[(375, 500), (500, 375)], vocab=50000)) for k in range(args.stories)]
        for f in range(4):
            W.write_records(t / f"story-{f:03d}.tfrecord", recs[f::4])
        res["records_written_s"] = round(time.perf_counter() - t0, 1)

        cfg = vcr_config(8)
        cfg.data.update(val_file=str(t / "val-*.tfrecord"), draw="segm")
        cfg.data.pop("num_threads", None)
        cfg.device.update(output_dir=str(t / "vcr"), val_batch_size=64)
        cfg.validate = {"eval_samples": args.questions, "eval_timeout": 0}
        os.makedirs(cfg.device["output_dir"])
        vcr_prefix = str(t / "vcr" / "model.ckpt-0")
        fn = vcr_model_fn_builder(cfg)
        fn.store.save_checkpoint(vcr_prefix)
        del fn
        vcr_dict = {k: dict(getattr(cfg, k)) for k in ("data", "model", "optimizer", "device", "downstream", "validate")}

        model = SR.five_segments_model()
        story_dict = {"data": {"val_file": str(t / "story-*.tfrecord")}, "model": model, "optimizer": {},
                      "device": {"output_dir": str(t / "story"), "val_batch_size": STORY_BATCH}}
        os.makedirs(t / "story")
        story_prefix = str(t / "story" / "model.ckpt-0")
        store = ParamStore(model, device="cuda")  # checkpoints hold the optimizer slots too
        store.init_reference(seed=0)
        store.save_checkpoint(story_prefix)
        update_checkpoint_state(str(t / "story"), story_prefix)
        del store
        torch.cuda.empty_cache()

        for n in ranks:
            res["vcr"].append(run_ranks(n, "vcr", vcr_dict, vcr_prefix, args.chunk))
            print(json.dumps(res["vcr"][-1]), flush=True)
            res["story"].append(run_ranks(n, "story", story_dict, story_prefix))
            print(json.dumps(res["story"][-1]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
