"""Checkpoint cost at merlot.yaml sizes: K15 (merlot_crc32c_multi) throughput over every tensor of a pretraining checkpoint,
save time split into staging / CRC / device-to-host / file write, restore time, peak extra device memory, and the NumPy
CRC-32C rate on the same host.  Needs an H100; prints the results as JSON and also writes them to --out if given.

  python tools/perf_checkpoint.py [--stem patch|hybrid] [--dir /tmp/...] [--out results.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stem", choices=("patch", "hybrid"), default="patch")
    ap.add_argument("--dir", default=None, help="where the checkpoint is written (default: a temporary directory)")
    ap.add_argument("--out", default=None, help="also write the JSON results to this file")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_checkpoint needs a GPU"
    import bench
    from merlot_b200 import ops
    from merlot_b200.params import ParamStore
    from merlot_b200.tf_checkpoint import crc32c
    bench.STEM = args.stem
    cfg = bench.load_config()
    store = ParamStore(cfg.model, device="cuda", optimizer_cfg=cfg.optimizer)
    g = torch.Generator(device="cuda").manual_seed(0)
    store.p.normal_(generator=g)
    store.m.copy_(torch.randn(store.total, device="cuda", generator=g).bfloat16())
    store.v.copy_(torch.rand(store.total, device="cuda", generator=g).bfloat16())
    store.global_step = 1000
    res = {"card": card(), "stem": args.stem, "params": store.num_params()}

    # K15 alone over the checkpoint's tensors, staged back to back as in save_checkpoint
    tensors = store._checkpoint_tensors(())
    sizes = [t.numel() * t.element_size() for _, _, t in tensors]
    offs = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    stage = torch.empty(offs[-1], dtype=torch.uint8, device="cuda")
    views = [stage[o:o + s] for o, s in zip(offs, sizes)]
    for (_, _, t), v in zip(tensors, views):
        v.view(t.dtype).view(t.shape).copy_(t)
    out = torch.empty(len(views), dtype=torch.int32, device="cuda")
    for _ in range(3):
        ops.crc32c_multi(views, out=out)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.reps):
        ops.crc32c_multi(views, out=out)
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / args.reps
    res["k15"] = {"tensors": len(views), "bytes": offs[-1], "ms": ms, "GB_per_s": offs[-1] / ms / 1e6,
                  "share_of_hbm_peak": offs[-1] / (ms * 1e-3) / HBM_PEAK}
    # spot check against the host CRC on a few tensors
    host = out.cpu().numpy().view(np.uint32)
    for i in (0, 1, len(views) // 2, len(views) - 1):
        assert int(host[i]) == crc32c(views[i].cpu().numpy()), i
    del stage, views

    d = args.dir or tempfile.mkdtemp(prefix="merlot_ckpt_")
    os.makedirs(d, exist_ok=True)
    try:
        prefix = os.path.join(d, "model.ckpt-1000")
        runs = []
        for _ in range(2):
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            split = store.save_checkpoint(prefix)
            split["total_s"] = time.perf_counter() - t0
            split["peak_extra_device_bytes"] = torch.cuda.max_memory_allocated() - base
            runs.append(split)
        res["save"] = runs
        res["file_bytes"] = os.path.getsize(prefix + ".data-00000-of-00001") + os.path.getsize(prefix + ".index")
        ref_p = store.p.clone()
        rruns = []
        for _ in range(2):
            store.p.zero_()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            store.restore_checkpoint(prefix)
            torch.cuda.synchronize()
            rruns.append({"total_s": time.perf_counter() - t0,
                          "peak_extra_device_bytes": torch.cuda.max_memory_allocated() - base})
        res["restore"] = rruns
        # every variable's values come back (the generated p also had values in the padding, which restores as zero)
        name = "word_embeddings/word_embeddings"
        e = store.entries[name]
        res["restore_matches"] = bool(torch.equal(store.P(name), ref_p[e.offset:e.offset + e.numel].view(e.shape)))
        del ref_p
    finally:
        if args.dir is None:
            shutil.rmtree(d, ignore_errors=True)

    sample = np.random.default_rng(0).integers(0, 256, 64 << 20, dtype=np.uint8)
    crc32c(sample[:1 << 20])  # builds the lane tables
    t0 = time.perf_counter()
    crc32c(sample)
    res["numpy_crc_MB_per_s"] = sample.nbytes / (time.perf_counter() - t0) / 1e6
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
