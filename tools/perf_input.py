"""Measure the pretraining input pipeline at merlot.yaml's sizes (192 x 352 frames from 288 x 512 quality-95 JPEGs, the size
data/process.py writes), on one GPU:

  1. host: read + CRC + parse of the records, then JPEG decode in a pool of T threads -> frames/s for each T
  2. K14 (merlot_frames_prepare): CUDA-event time per batch of 32 and 128 frames, against the bytes it has to move
  3. the configs[1]-sized training step (bench.py's model, 8 groups of 4 segments = 32 frames) fed by input_fn_builder
     (2 examples of 16 frames) against the same step on device-resident synthetic inputs, alternated in one process

    python tools/perf_input.py [--steps 20] [--rounds 3] [--out perf_input.json]

The tfrecords are generated from a seed in a temporary directory.  Prints one JSON object (card name and power limit included).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from merlot_b200 import dataloader as D  # noqa: E402
from merlot_b200 import ops  # noqa: E402
from merlot_b200.tfrecord import parse_example, read_records  # noqa: E402
from tests import tfrecord_writer as W  # noqa: E402

MERLOT_DATA = {"num_chunks": 16, "chunk_text_len": 32, "random_scale_min": 1.125, "random_scale_max": 1.5, "augment_prob": 0.8,
               "clean_asr_prob": 0.5, "shuffle_chunks": True}  # model/configs/merlot.yaml data section
SRC_HW, OUT_HW = (288, 512), (192, 352)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def write_dataset(d, files, per_file):
    rng = np.random.default_rng(0)
    for fi in range(files):
        recs = [W.chunks_example(W.video_chunks(rng, 16, frame_hw=SRC_HW, max_caption=40, video=f"v{fi}_{e}"))
                for e in range(per_file)]
        W.write_records(os.path.join(d, f"train-{fi:03d}.tfrecord"), recs)
    return sorted(os.path.join(d, f) for f in os.listdir(d))


def host_rates(files, threads):
    out = {}
    t0 = time.perf_counter()
    examples = [parse_example(r) for f in files for r in read_records(f)]
    t_parse = time.perf_counter() - t0
    jpgs = [j for ex in examples for j in D.frame_bytes(ex, 16)]
    out["frames"] = len(jpgs)
    out["read_crc_parse_frames_per_s_1_thread"] = len(jpgs) / t_parse
    for t in threads:
        with ThreadPoolExecutor(t) as pool:
            list(pool.map(D.decode_jpeg, jpgs[:t]))  # warm
            t0 = time.perf_counter()
            list(pool.map(D.decode_jpeg, jpgs))
            out[f"decode_frames_per_s_{t}_threads"] = len(jpgs) / (time.perf_counter() - t0)
    return out, jpgs


def k14_times(jpgs, sizes, iters=50):
    dev = torch.device("cuda")
    frames = [D.decode_jpeg(j) for j in jpgs[:max(sizes)]]
    out = {}
    for n in sizes:
        fr = frames[:n]
        packed = torch.from_numpy(np.concatenate([f.reshape(-1) for f in fr])).to(dev)
        offs = np.concatenate([[0], np.cumsum([f.size for f in fr])[:-1]])
        dr = D.frame_draws(np.random.default_rng(n), n, MERLOT_DATA)
        plan = D.plan_frames([f.shape[0] for f in fr], [f.shape[1] for f in fr], OUT_HW, dr["scale"], dr["u_y"], dr["u_x"])
        plan.update(src_offset=offs, src_h=[f.shape[0] for f in fr], src_w=[f.shape[1] for f in fr], method=dr["method"],
                    augment=dr["augment"], factor=dr["factor"])
        res = torch.empty((n,) + OUT_HW + (3,), dtype=torch.bfloat16, device=dev)
        for _ in range(5):
            ops.frames_prepare(packed, plan, *OUT_HW, out=res)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            ops.frames_prepare(packed, plan, *OUT_HW, out=res)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        written = res.numel() * 2
        read = sum(f.size for f in fr)  # each source byte at least once (resizes upscale 1.125-1.5x: every source pixel is read)
        out[f"k14_{n}_frames_us"] = us
        out[f"k14_{n}_frames_bytes"] = written + read
        out[f"k14_{n}_frames_GB_per_s"] = (written + read) / us / 1e3
        out[f"k14_{n}_frames_share_of_3.35TB_per_s"] = (written + read) / us / 1e3 / 3350
    return out


def step_compare(files, steps, rounds):
    import bench
    from merlot_b200.train import model_fn_builder, synthetic_batch
    config = bench.load_config()
    config.data.update(MERLOT_DATA, train_file_expanded=files, num_threads=8, shuffle_buffer_size=16)
    model_fn = model_fn_builder(config, device="cuda")
    resident = synthetic_batch(config, bench.PER_GPU_BATCH, seed=0, device="cuda")  # 8 x 4 segments
    per_step = bench.PER_GPU_BATCH * config.model["num_chunks_in_group"] // MERLOT_DATA["num_chunks"]  # 2 examples x 16 frames

    def run(next_feats, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(k):
            spec = model_fn(next_feats(), None, "train", None)
            spec.train_op()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / k

    res = {"synthetic_ms": [], "real_ms": []}
    with D.input_fn_builder(config, True, seed=0, batch_size=per_step) as pipe:
        run(lambda: resident, 3)
        run(lambda: next(pipe), 3)
        for _ in range(rounds):
            res["synthetic_ms"].append(run(lambda: resident, steps))
            res["real_ms"].append(run(lambda: next(pipe), steps))
    res["segments_per_step"] = bench.PER_GPU_BATCH * config.model["num_chunks_in_group"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--files", type=int, default=4)
    ap.add_argument("--per-file", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_input.py measures on a CUDA device")
    result = {"card": card(), "cpus": len(os.sched_getaffinity(0))}
    with tempfile.TemporaryDirectory() as d:
        files = write_dataset(d, args.files, args.per_file)
        result["tfrecord_bytes"] = sum(os.path.getsize(f) for f in files)
        host, jpgs = host_rates(files, [1, 2, 4, 8])
        result.update(host)
        result["mean_jpeg_bytes"] = float(np.mean([len(j) for j in jpgs]))
        result.update(k14_times(jpgs, [32, 128]))
        result.update(step_compare(files, args.steps, args.rounds))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
