"""Measure zero-shot story unshuffling at merlot_5segments.yaml's sizes (5 x 384 x 384 frames per story, hybrid stem,
ViT-B + 12-layer joint encoder, duplication factor 2, val_batch_size 16), on one GPU:

  1. the zero-shot forward of one batch of 16 stories: frame_copies=2 (one ViT pass per story) against the tiled forward the
     reference runs (every frame through the ViT once per copy), alternated in one process, CUDA events, warm-up first;
     peak memory of each, and how far their probabilities are apart
  2. end to end from story records: input_fn_builder + zero_shot_predict over every batch, host clock around work that
     ends in a device synchronise

    python tools/perf_sort_story.py [--iters 10] [--rounds 3] [--stories 96] [--out perf_sort_story.json]

The records (500 x 375 and 375 x 500 quality-95 JPEGs) are generated from a seed in a temporary directory.  Prints one JSON
object, the card's name and power limit included.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from merlot_b200 import sort_story as S  # noqa: E402
from merlot_b200.config import NeatConfig  # noqa: E402
from merlot_b200.modeling import MerlotModel  # noqa: E402
from merlot_b200.params import ParamStore  # noqa: E402
from tests import story_records as R  # noqa: E402

DUP, BATCH = 2, 16  # get_zero_shot_logits.py:33, merlot_5segments.yaml device.val_batch_size


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def forward_compare(config, store, iters, rounds):
    cfg = config.model
    g = torch.Generator().manual_seed(0)
    images = torch.rand(BATCH * 5, 384, 384, 3, generator=g).to(torch.bfloat16).cuda()
    sents = torch.randint(100, 50357, (BATCH, 5, 32), generator=g, dtype=torch.int32)
    sents[:, :, 0] = 2
    sents[:, :, 24:] = 0
    sents = sents.cuda()
    batch = {"images": images, "sentences": sents, "story_id": np.arange(BATCH), "permutation_identity_encode": np.zeros(BATCH)}
    tiled_images = images.view(BATCH, 5, 384, 384, 3).repeat_interleave(DUP, 0).reshape(BATCH * DUP * 5, 384, 384, 3).contiguous()
    ids, shuf = S.tiled_inputs(sents, DUP)

    def one_pass():
        out = S.zero_shot_predict(config, store, batch, duplication_factor=DUP)
        return out["lang_viz_probs"], out["viz_viz_probs"]

    def tiled():
        m = MerlotModel(cfg, is_training=False, use_tpu=False, image=tiled_images, input_ids=ids, mask_input=False,
                        shuffled_idx_img=shuf, params=store, log_attention_probs=False)
        return S.temporal_probs(m, DUP, "lang_viz_temporal"), S.temporal_probs(m, DUP, "viz_viz_temporal")

    res = {}
    for name, fn in (("frame_copies", one_pass), ("tiled", tiled)):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        for _ in range(3):
            out = fn()
        torch.cuda.synchronize()
        res[f"{name}_peak_GiB"] = torch.cuda.max_memory_allocated() / 2 ** 30
        res[f"{name}_probs"] = [p.clone() for p in out]
    a, b = res.pop("frame_copies_probs"), res.pop("tiled_probs")
    res["probs_max_abs_diff"] = max(float((x - y).abs().max()) for x, y in zip(a, b))
    ms = {"frame_copies": [], "tiled": []}
    for _ in range(rounds):
        for name, fn in (("frame_copies", one_pass), ("tiled", tiled)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / iters)
    for name, v in ms.items():
        res[f"{name}_ms_per_batch"] = v
        res[f"{name}_stories_per_s"] = BATCH / (float(np.median(v)) * 1e-3)
    res["speedup_median"] = float(np.median(ms["tiled"])) / float(np.median(ms["frame_copies"]))
    return res


def end_to_end(config, store, stories):
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        from tests import tfrecord_writer as W
        recs = [R.story_example(R.story(rng, k, sizes=[(375, 500), (500, 375)], vocab=50000)) for k in range(stories)]
        files = 4
        for f in range(files):
            W.write_records(os.path.join(d, f"val-{f:03d}.tfrecord"), recs[f::files])
        config.data.update(val_file=os.path.join(d, "val-*.tfrecord"), num_threads=16)
        config.data.pop("val_file_expanded", None)
        out = {"stories": stories, "tfrecord_bytes": sum(os.path.getsize(os.path.join(d, n)) for n in os.listdir(d))}
        for rep in ("warm", "timed"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = 0
            with torch.no_grad(), S.input_fn_builder(config, batch_size=BATCH) as pipe:
                for batch in pipe:
                    p = S.zero_shot_predict(config, store, batch, duplication_factor=DUP)
                    n += len(batch["story_id"])
                torch.cuda.synchronize()
                dropped = pipe.dropped
            dt = time.perf_counter() - t0
        out.update(scored=n, dropped=dropped, seconds=dt, stories_per_s=n / dt, last_probs_finite=bool(torch.isfinite(p["lang_viz_probs"]).all()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--stories", type=int, default=96)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_sort_story.py measures on a CUDA device")
    cfg = R.five_segments_model()
    config = NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {}, "device": {"output_dir": "/nonexistent"}})
    store = ParamStore(cfg, device="cuda", with_optimizer_state=False)
    store.init_reference(seed=0)
    result = {"card": card(), "cpus": len(os.sched_getaffinity(0)), "batch_stories": BATCH, "duplication_factor": DUP}
    with torch.no_grad():
        result["forward"] = forward_compare(config, store, args.iters, args.rounds)
    result["end_to_end"] = end_to_end(config, store, args.stories)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
