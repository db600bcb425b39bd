"""Measure frame <-> transcript retrieval (merlot_b200.retrieval_validate) on one GPU at merlot.yaml's sizes:

  1. the feature pass: MerlotModel(is_training=False, mask_input=True, features_only=True) + contrastive_features() on one
     resident evaluation batch of 16 videos x 16 segments (192 x 352 frames, 32-token captions), CUDA events over --iters
     calls, with the patch-embed stem and with the hybrid stem; the time of N segments is N / 256 batches at that rate
  2. the scores: K16's split of both arenas and one K1 GEMM per query chunk [chunk, N] (K = 3 Cs), CUDA events over every
     chunk of one direction, at N = 16,384 (merlot.yaml's global batch, 1024 videos x 16 segments) and N = 163,840
  3. K17 on the same score blocks: time per direction, and its HBM rate, chunk * N * 4 bytes read per chunk over its time,
     against the H100 SXM data sheet's 3.35 TB/s
  4. rank_chunks end to end (split, GEMMs, K17 and the host copies) for one direction

    python tools/perf_retrieval.py [--iters 5] [--chunk 1024] [--out perf_retrieval.json]

Prints one JSON object with the card's name and power limit, queried in the same run.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_GBS = 3350.0
SIZES = (16384, 163840)


def events(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()  # warm-up
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def feature_pass(stem, val_glob, tmp, iters):
    from perf_pretrain_validate import VAL_BATCH, config_for
    from merlot_b200 import dataloader as D
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import ParamStore
    config = config_for(stem, val_glob, os.path.join(tmp, stem))
    store = ParamStore(config.model, device="cuda", optimizer_cfg=config.optimizer)
    store.init_reference(seed=0)
    with torch.no_grad(), D.input_fn_builder(config, is_training=False, batch_size=VAL_BATCH) as pipe:
        batch = next(pipe)

        def run():
            m = MerlotModel(config.model, is_training=False, use_tpu=False, image=batch["images"], input_ids=batch["input_ids"],
                            mask_input=True, shuffled_idx_img=batch["shuffled_idx_img"], params=store, features_only=True,
                            log_attention_probs=False)
            m.contrastive_features()
        ms = events(run, iters)
    rows = VAL_BATCH * batch["input_ids"].shape[1]
    out = {"stem": stem, "segments_per_batch": rows, "ms_per_batch": round(ms, 2),
           "s_at_N": {str(n): round(ms * n / rows / 1e3, 2) for n in SIZES}}
    del store, batch
    torch.cuda.empty_cache()
    return out, int(config.model.get("contrastive_size", config.model["hidden_size"]))


def ranking(n, Cs, chunk, iters):
    from merlot_b200 import ops
    from merlot_b200 import retrieval_validate as RV
    g = torch.Generator(device="cuda").manual_seed(n)
    lang = torch.nn.functional.normalize(torch.randn(n, Cs, device="cuda", generator=g), dim=1)
    viz = torch.nn.functional.normalize(lang + torch.randn(n, Cs, device="cuda", generator=g), dim=1)
    xc = torch.empty((n, 3 * Cs), dtype=torch.bfloat16, device="cuda")
    yc = torch.empty((n, 3 * Cs), dtype=torch.bfloat16, device="cuda")
    block = torch.empty((chunk, RV.pad8(n)), dtype=torch.float32, device="cuda")
    chunks = RV.query_chunks(n, chunk)
    outs = [(torch.empty(e - s, dtype=torch.int32, device="cuda"), torch.empty(e - s, dtype=torch.int32, device="cuda"),
             torch.empty((e - s, 10), dtype=torch.int32, device="cuda"), torch.empty((e - s, 10), device="cuda"),
             torch.arange(s, e, dtype=torch.int32, device="cuda")) for s, e in chunks]

    def split():
        ops.ctr_split(lang, xc, 3 * Cs, Cs, 0b100)
        ops.ctr_split(viz, yc, 3 * Cs, Cs, 0b010)

    def gemms():
        for s, e in chunks:
            ops.gemm(xc[s:e], yc, out=block[:e - s, :n], alpha=1.0, M=e - s, N=n, K=3 * Cs)

    def k17():
        for (s, e), (gr, ti, ix, va, pos) in zip(chunks, outs):
            ops.rank_topk(block[:e - s, :n], pos, 10, gr, ti, ix, va)

    split_ms = events(split, iters)
    gemm_ms = events(gemms, iters)
    k17_ms = events(k17, iters)
    k17_bytes = n * n * 4
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    RV.rank_chunks(lang, viz, [(c, s, e) for c, (s, e) in enumerate(chunks)], chunk)
    torch.cuda.synchronize()
    e2e = time.perf_counter() - t0
    flops = 2.0 * n * n * 3 * Cs
    res = {"N": n, "Cs": Cs, "chunk": chunk, "split_ms": round(split_ms, 3), "gemm_ms_per_direction": round(gemm_ms, 2),
           "gemm_tflops": round(flops / gemm_ms / 1e9, 1), "k17_ms_per_direction": round(k17_ms, 2),
           "k17_gbs": round(k17_bytes / k17_ms / 1e6, 1), "k17_share_of_hbm": round(k17_bytes / k17_ms / 1e6 / HBM_GBS, 3),
           "rank_chunks_s_per_direction": round(e2e, 3)}
    del lang, viz, xc, yc, block, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=1024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_retrieval.py measures on a CUDA device")
    from perf_input import SRC_HW
    from perf_pretrain_validate import VAL_BATCH, card
    from tests import tfrecord_writer as W
    res = {"card": card(), "features": [], "ranking": []}
    with tempfile.TemporaryDirectory() as tmp:
        rng = np.random.default_rng(0)
        recs = [W.chunks_example(W.video_chunks(rng, 16, frame_hw=SRC_HW, max_caption=40, video=f"v{e}")) for e in range(VAL_BATCH)]
        W.write_records(os.path.join(tmp, "val-000.tfrecord"), recs)
        Cs = None
        for stem in ("patch", "hybrid"):
            f, Cs = feature_pass(stem, os.path.join(tmp, "val-*.tfrecord"), tmp, args.iters)
            res["features"].append(f)
            print(json.dumps(f), flush=True)
    for n in SIZES:
        res["ranking"].append(ranking(n, Cs, args.chunk, args.iters))
        print(json.dumps(res["ranking"][-1]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
