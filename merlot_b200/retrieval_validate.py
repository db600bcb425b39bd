"""`python -m merlot_b200.retrieval_validate CONFIG`: zero-shot frame <-> transcript retrieval over the whole held-out set, the
contrastive head (model/modeling.py:491-526) measured against every held-out segment instead of one batch.

Features.  Per checkpoint the trainer's pretraining store is restored and MerlotModel(is_training=False, mask_input=True,
features_only=True) runs on the batches pretrain_validate reads: the evaluation input (dataloader.EvalInputPipeline), batch
k with parser draws keyed by (--seed, k) and masking seed train.eval_seed(--seed, k), the first validate.eval_samples //
device.val_batch_size batches (every whole batch without eval_samples).  Dropout is off, so the features depend on the
weights and pixels only.  contrastive_features() gives each batch's l2-normalised lang and viz rows, copied into two
[N, Cs] fp32 arenas in global row order: row i = (batch k, video v, chunk c) with i = (k * val_batch_size + v) * num_chunks + c.
Segment i's transcript and frame are the pair the contrastive loss trains (label = row).

Scores and ranks.  In each direction (lang_to_viz: transcript queries against frame keys; viz_to_lang the reverse) the
queries run in chunks of --chunk rows.  A chunk's cosine similarities with all N keys are one K1 GEMM over K16's split-bf16
operands, [xh | xh | xl] . [yh | yl | yh]^T with alpha 1 (dividing by contrast_temp would not change the order but would merge
near ties), into a [chunk, pad8(N)] fp32 block that K17 (csrc/retrieval.cu) ranks exactly: rank = 1 + the number of keys
scoring strictly above the positive, so ties count in the query's favour.

Output.  One JSON line per checkpoint appended to output_dir/eval/retrieval.jsonl: {global_step, segments, lang_to_viz:
{r1, r5, r10, median_rank, mean_rank, tied}, viz_to_lang: {...}}, where r@K is the fraction of queries of rank <= K,
median_rank is np.median of the ranks, and tied counts the queries whose positive ties another key.  A NaN positive
raises and names the segment.  `--predictions OUT.npz` (with `--checkpoint`) stores, per direction, every query's rank and
its --top-k keys with their scores.

Under torchrun with WORLD_SIZE > 1 (eval_ranks): rank 0 follows device.output_dir and broadcasts each prefix; every rank
computes the features of the global batches k with k % world == rank; the arenas are gathered to every rank in global order
(NCCL on the device, or through host memory under gloo); query chunk c is ranked on rank c % world, so every GEMM has the
one-GPU shape; the per-query results are gathered in chunk order and rank 0 writes the line one GPU writes.
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import time
from typing import Callable, Dict, List, Sequence, Tuple

import numpy as np

from .pretrain_validate import check_val_file, eval_batch_count
from .vcr_validate import follow_checkpoints

RETRIEVAL_FILE = os.path.join("eval", "retrieval.jsonl")
DIRECTIONS = ("lang_to_viz", "viz_to_lang")
MAX_TOP_K = 32
FINETUNING_TASKS = ("vcr", "video_mc", "video_qa", "video_fib")


def pad8(n: int) -> int:
    return (n + 7) // 8 * 8


def segment_of(row: int, batch_size: int, num_chunks: int) -> Tuple[int, int, int]:
    """Feature row -> (global batch, video in the batch, chunk in the video)."""
    video, chunk = divmod(int(row), num_chunks)
    batch, video = divmod(video, batch_size)
    return batch, video, chunk


def query_chunks(n: int, chunk: int) -> List[Tuple[int, int]]:
    """[start, stop) of every query chunk of n rows."""
    return [(s, min(s + chunk, n)) for s in range(0, n, chunk)]


def chunk_owner(c: int, world: int) -> int:
    """The rank that ranks query chunk c."""
    return c % world


def direction_metrics(greater: np.ndarray, ties: np.ndarray) -> Dict:
    """{r1, r5, r10, median_rank, mean_rank, tied} of one direction from K17's per-query counts; rank = 1 + greater."""
    ranks = 1 + np.asarray(greater, np.int64)
    out = {f"r{k}": float(np.mean(ranks <= k)) for k in (1, 5, 10)}
    out.update(median_rank=float(np.median(ranks)), mean_rank=float(np.mean(ranks)), tied=int(np.sum(np.asarray(ties) > 0)))
    return out


def results_line(global_step: int, segments: int, per_direction: Dict[str, Tuple[np.ndarray, np.ndarray]]) -> Dict:
    res = {"global_step": int(global_step), "segments": int(segments)}
    for d in DIRECTIONS:
        res[d] = direction_metrics(*per_direction[d])
    return res


def check_nan_positives(greater: Dict[str, np.ndarray], batch_size: int, num_chunks: int) -> None:
    """K17 reports a NaN positive score as greater = -1: raise ValueError naming the first such segment."""
    for d in DIRECTIONS:
        bad = np.flatnonzero(np.asarray(greater[d]) == -1)
        if bad.size:
            k, v, c = segment_of(bad[0], batch_size, num_chunks)
            raise ValueError(f"{d}: the positive score of segment {int(bad[0])} (global batch {k}, video {v}, chunk {c}) is "
                             f"NaN; {bad.size} queries in all")


def check_config(config, chunk: int, top_k: int, predictions=None, checkpoint=None) -> None:
    """Every refusal that needs no GPU: a fine-tuning task, an empty data.val_file, fewer than one batch, --chunk < 1, --top-k
    outside [1, 32], --predictions without --checkpoint."""
    task = config.downstream.get("task")
    if task in FINETUNING_TASKS:
        raise ValueError(f"downstream.task is {task!r}: frame-transcript retrieval ranks a pretraining checkpoint's contrastive "
                         f"head; validate {'VCR' if task == 'vcr' else task} fine-tuning with merlot_b200.{task}_validate")
    if chunk < 1:
        raise ValueError(f"--chunk {chunk}: need at least one query row per chunk")
    if not 1 <= top_k <= MAX_TOP_K:
        raise ValueError(f"--top-k {top_k}: need 1 <= top_k <= {MAX_TOP_K}")
    if predictions and not checkpoint:
        raise ValueError("--predictions needs --checkpoint: the file holds one checkpoint's per-query results")
    output_dir = str(config.device["output_dir"])
    if "://" in output_dir:
        raise ValueError(f"device.output_dir {output_dir!r}: only local directories are supported for checkpoints")
    check_val_file(config)
    eval_batch_count(config)


def rank_chunks(queries, keys, chunks: Sequence[Tuple[int, int, int]], chunk: int, top_k: int = 0) -> Dict:
    """K16 scores + K17 ranks of the given query chunks (c, start, stop) of `queries` [N, Cs] against all of `keys` [N, Cs]
    (both fp32, l2-normalised, on the device); query i's positive is key i.  Returns {c: (greater, ties, topk_idx,
    topk_val)} as host arrays (the top-k pair is None when top_k is 0)."""
    import torch
    from . import ops
    n, Cs = keys.shape
    if Cs % 8 != 0:
        raise ValueError(f"contrastive_size {Cs} must be a multiple of 8 (K16's bf16 operand rows)")
    dev = keys.device
    xc = torch.empty((n, 3 * Cs), dtype=torch.bfloat16, device=dev)
    yc = torch.empty((n, 3 * Cs), dtype=torch.bfloat16, device=dev)
    ops.ctr_split(queries, xc, 3 * Cs, Cs, 0b100)  # [xh | xh | xl]
    ops.ctr_split(keys, yc, 3 * Cs, Cs, 0b010)     # [yh | yl | yh]
    block = torch.empty((min(chunk, n), pad8(n)), dtype=torch.float32, device=dev)
    k = max(top_k, 1)
    out = {}
    for c, start, stop in chunks:  # stream-ordered reuse of one block; the host copies wait until every chunk is queued
        q = stop - start
        scores = block[:q, :n]
        ops.gemm(xc[start:stop], yc, out=scores, alpha=1.0, M=q, N=n, K=3 * Cs)
        pos = torch.arange(start, stop, dtype=torch.int32, device=dev)
        out[c] = ops.rank_topk(scores, pos, k)
    return {c: tuple(t.cpu().numpy() if (i < 2 or top_k) else None for i, t in enumerate(res)) for c, res in out.items()}


class Validator:
    """Ranks the held-out segments of data.val_file against each other under one checkpoint after another.  With an
    eval_ranks.EvalGroup of several ranks, each rank computes the features of the global batches k with k % world == rank
    and ranks the query chunks c with c % world == rank; every rank gets the result one rank computes."""

    def __init__(self, config, seed: int = 0, device="cuda", group=None, chunk: int = 1024, top_k: int = 0):
        from .eval_ranks import EvalGroup
        from .params import ParamStore
        from .train import variables_without_gradient
        self.group = group if group is not None else EvalGroup()
        self.config, self.seed, self.device, self.chunk, self.top_k = config, seed, device, int(chunk), int(top_k)
        self.batch_size = int(config.device.get("val_batch_size", 16))
        self.num_chunks = int(config.data.get("num_chunks", config.model.get("num_chunks_in_group", 4)))
        self.Cs = int(config.model.get("contrastive_size", config.model["hidden_size"]))
        self.num_batches = eval_batch_count(config)
        check_val_file(config)
        self.store = ParamStore(config.model, device=device, optimizer_cfg=config.optimizer)
        self.skip = variables_without_gradient(config.model, self.store)
        self.predictions = None  # per-query results of the last evaluate(): {direction: (greater, ties, topk_idx, topk_val)}

    @property
    def rows_per_batch(self) -> int:
        return self.batch_size * self.num_chunks

    def _own_features(self) -> List:
        """This rank's batches' (lang, viz) feature rows, [2, rows_per_batch, Cs] fp32 on the device per batch, in the order
        of its global batches."""
        import torch
        from .dataloader import input_fn_builder
        from .modeling import MerlotModel
        from .train import eval_seed
        g, cfg = self.group, self.config
        out = []
        with torch.no_grad(), input_fn_builder(cfg, is_training=False, rank=g.rank, world=g.world, seed=self.seed,
                                               batch_size=self.batch_size, device=self.device) as pipe:
            own = pipe if self.num_batches is None else itertools.islice(pipe, len(range(g.rank, self.num_batches, g.world)))
            for batch in own:
                k = pipe.last_info["batch"]
                m = MerlotModel(cfg.model, is_training=False, use_tpu=cfg.device.get("use_tpu", False), image=batch["images"],
                                input_ids=batch["input_ids"], mask_input=True, shuffled_idx_img=batch["shuffled_idx_img"],
                                params=self.store, dropout_seed=eval_seed(self.seed, k), log_attention_probs=False,
                                features_only=True)
                lang, viz = m.contrastive_features()
                if lang.n != self.rows_per_batch or lang.Cs != self.Cs:
                    raise RuntimeError(f"batch {k}: {lang.n} x {lang.Cs} features, expected {self.rows_per_batch} x {self.Cs}")
                out.append(torch.stack([lang.feat, viz.feat]))
        return out

    def features(self, prefix: str):
        """Restore `prefix` and compute the (lang, viz) arenas [N, Cs] fp32 of every held-out segment, in global row order,
        on every rank."""
        import torch
        g = self.group
        self.store.restore_checkpoint(prefix, skip=self.skip)
        if g.world == 1:
            own = self._own_features()
            if not own:
                raise ValueError(f"data.val_file holds no whole batch of {self.batch_size} videos")
            arena = torch.cat(own, dim=1)  # [2, N, Cs]: batch k's rows at [k * rows_per_batch, (k + 1) * rows_per_batch)
            return arena[0], arena[1]
        own, error = [], None
        try:
            own = self._own_features()
        except Exception as e:  # handed to every rank by agree()
            error = f"{type(e).__name__}: {e}"
        g.agree(error)
        counts = g.all_gather(len(own))
        nb, per = sum(counts), max(counts)
        if nb == 0:
            raise ValueError(f"data.val_file holds no whole batch of {self.batch_size} videos")
        on_device = g.dist.get_backend() == "nccl"
        where = self.device if on_device else "cpu"
        shape = (per, 2, self.rows_per_batch, self.Cs)
        mine = torch.zeros(shape, dtype=torch.float32, device=where)
        for j, f in enumerate(own):
            mine[j].copy_(f)
        parts = [torch.empty(shape, dtype=torch.float32, device=where) for _ in range(g.world)]
        g.dist.all_gather(parts, mine)
        arena = torch.empty((2, nb * self.rows_per_batch, self.Cs), dtype=torch.float32, device=self.device)
        for k in range(nb):  # global batch k was computed by rank k % world as its (k // world)-th batch
            arena[:, k * self.rows_per_batch:(k + 1) * self.rows_per_batch].copy_(parts[k % g.world][k // g.world])
        return arena[0], arena[1]

    def evaluate(self, prefix: str) -> Dict:
        """Restore `prefix`, rank every segment in both directions and return the results line; self.predictions keeps the
        per-query arrays.  With several ranks every rank returns the same result; a failure on any rank raises RankFailure
        on every rank."""
        g = self.group
        lang, viz = self.features(prefix)
        n = lang.shape[0]
        chunks = query_chunks(n, self.chunk)
        mine = [(c, s, e) for c, (s, e) in enumerate(chunks) if chunk_owner(c, g.world) == g.rank]

        def own_ranks():
            return {d: rank_chunks(q, k, mine, self.chunk, self.top_k) for d, q, k in
                    (("lang_to_viz", lang, viz), ("viz_to_lang", viz, lang))}

        per_rank = g.run_and_gather(own_ranks)
        merged = {}
        for d in DIRECTIONS:
            parts = [per_rank[chunk_owner(c, g.world)][d][c] for c in range(len(chunks))]
            merged[d] = tuple(None if parts[0][i] is None else np.concatenate([p[i] for p in parts]) for i in range(4))
        check_nan_positives({d: merged[d][0] for d in DIRECTIONS}, self.batch_size, self.num_chunks)
        self.predictions = merged
        return results_line(self.store.global_step, n, {d: merged[d][:2] for d in DIRECTIONS})


def write_predictions(path: str, predictions: Dict, batch_size: int, num_chunks: int) -> str:
    """OUT.npz: segment [N] (the feature row), batch / video / chunk [N], and per direction <d>_rank [N],
    <d>_topk_idx [N, K] (key segments, -1 past the non-NaN scores) and <d>_topk_score [N, K] (their cosine scores)."""
    n = len(predictions[DIRECTIONS[0]][0])
    seg = np.arange(n, dtype=np.int64)
    video, chunk = np.divmod(seg, num_chunks)
    batch, video = np.divmod(video, batch_size)
    arrays = {"segment": seg, "batch": batch, "video": video, "chunk": chunk}
    for d in DIRECTIONS:
        greater, _, idx, val = predictions[d]
        arrays[f"{d}_rank"] = 1 + greater.astype(np.int64)
        arrays[f"{d}_topk_idx"] = idx
        arrays[f"{d}_topk_score"] = val
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        np.savez(f, **arrays)
    return path


def append_result(output_dir: str, res: Dict) -> str:
    """Append the result dict as one JSON line to output_dir/eval/retrieval.jsonl; returns its path."""
    path = os.path.join(output_dir, RETRIEVAL_FILE)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "a", encoding="utf-8") as f:
        f.write(json.dumps(res) + "\n")
    return path


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Rank every held-out segment's frame and transcript against all the others")
    ap.add_argument("config_file")
    ap.add_argument("--checkpoint", help="evaluate this checkpoint prefix once instead of following device.output_dir")
    ap.add_argument("--poll-interval", type=float, default=60.0, help="seconds between looks at device.output_dir")
    ap.add_argument("--seed", type=int, default=0, help="seed of the evaluation draws (parser and masking)")
    ap.add_argument("--chunk", type=int, default=1024, help="query rows per score block [chunk, N]")
    ap.add_argument("--predictions", help="with --checkpoint: write every query's rank and top-k keys to this .npz")
    ap.add_argument("--top-k", type=int, default=10, help=f"keys per query in --predictions (1 to {MAX_TOP_K})")
    return ap.parse_args(argv)


def main(argv=None, clock: Callable[[], float] = time.monotonic, sleep: Callable[[float], None] = time.sleep) -> List[Dict]:
    """Returns the result dict of every evaluated checkpoint, in order."""
    from .config import NeatConfig
    from .eval_ranks import eval_group
    args = parse_args(argv)
    config = NeatConfig.from_yaml(args.config_file)
    check_config(config, args.chunk, args.top_k, args.predictions, args.checkpoint)
    output_dir = str(config.device["output_dir"])

    def follow(sleep_fn):
        if args.checkpoint:
            return iter([args.checkpoint])
        return follow_checkpoints(output_dir, int(config.optimizer.get("num_train_steps", 10)),
                                  float(config.validate.get("eval_timeout", 72000)), args.poll_interval, clock, sleep_fn)

    def write(prefix, res, v):
        path = append_result(output_dir, res)
        l2v, v2l = res["lang_to_viz"], res["viz_to_lang"]
        print(f"{prefix}: global_step {res['global_step']} over {res['segments']} segments: lang_to_viz R@1 {l2v['r1']:.4f} "
              f"median rank {l2v['median_rank']:g}, viz_to_lang R@1 {v2l['r1']:.4f} median rank {v2l['median_rank']:g} -> "
              f"{path}", flush=True)
        if args.predictions:
            write_predictions(args.predictions, v.predictions, v.batch_size, v.num_chunks)

    results = []
    with eval_group() as group:  # WORLD_SIZE > 1: rank 0 follows the checkpoints and writes, every rank evaluates
        v = Validator(config, seed=args.seed, group=group, chunk=args.chunk, top_k=args.top_k if args.predictions else 0)
        for prefix in group.shared_prefixes(follow, sleep):
            res = v.evaluate(prefix)
            group.on_rank0(lambda: write(prefix, res, v))
            results.append(res)
    return results


if __name__ == "__main__":
    main()
