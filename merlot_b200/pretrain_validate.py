"""`python -m merlot_b200.pretrain_validate CONFIG`: held-out evaluation of a pretraining run, the role of the reference's
Estimator EVAL on data.val_file (model/dataloader.py:129-278 with is_training=False, model/modeling.py:691-711,788-798).

It follows device.output_dir with vcr_validate.follow_checkpoints: every checkpoint newer than the last one evaluated, oldest
first, until the one whose global_step reaches optimizer.num_train_steps or until validate.eval_timeout seconds (default
72000) pass without a new one.  `--checkpoint PREFIX` evaluates one prefix and exits.

Per checkpoint the trainer's pretraining store is restored (ParamStore.restore_checkpoint) and model_fn's "eval" mode runs
on the first validate.eval_samples // device.val_batch_size batches of the evaluation input (dataloader.EvalInputPipeline),
or on every whole batch when validate.eval_samples is absent.  Batch k is evaluated with the dropout and masking seed
train.eval_seed(--seed, k) and parser draws keyed by (--seed, k), so successive checkpoints see the same pixels, texts and
masks.  One JSON line per checkpoint, {global_step, loss, videos, every lang/ attn/ contr/ temporal/ key}, is appended to
output_dir/eval/results.jsonl; each value is the mean over batches of the per-batch value, as tf.metrics.mean computes it
from the reference's per-example tiles.  The per-batch values stay on the device until the checkpoint's last batch.

Under torchrun with WORLD_SIZE > 1 (eval_ranks): rank 0 follows device.output_dir and broadcasts each prefix, every rank
evaluates the global batches k with k % world == rank, the per-batch values are gathered in global batch order and reduced
with the one-process operations, and rank 0 appends the line.  No collective runs inside a batch.
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import time
from typing import Callable, Dict, List, Optional, Sequence

from .vcr_validate import RESULTS_FILE, follow_checkpoints

METRIC_PREFIXES = ("lang/", "attn/", "contr/", "temporal/")


def eval_batch_count(config) -> Optional[int]:
    """validate.eval_samples // device.val_batch_size (None when eval_samples is absent: every whole batch).  Raises
    ValueError when that is less than one batch."""
    batch_size = int(config.device.get("val_batch_size", 16))
    if "eval_samples" not in config.validate:
        return None
    n = int(config.validate["eval_samples"]) // batch_size
    if n < 1:
        raise ValueError(f"validate.eval_samples {config.validate['eval_samples']!r} is less than one batch of "
                         f"device.val_batch_size {batch_size}")
    return n


def check_val_file(config) -> List[str]:
    """The files of data.val_file; raises ValueError naming the key when it is empty or matches nothing."""
    from .sort_story import val_files
    files = val_files(config)
    if not files:
        raise ValueError(f"data.val_file {config.data.get('val_file')!r} matches no file: pretraining validation needs "
                         f"held-out records")
    return files


def reduce_batches(keys: Sequence[str], batches: Sequence, batch_size: int, global_step: int, device=None) -> Dict:
    """The results line of one checkpoint from its per-batch vectors [loss, *keys] in global batch order: the mean over
    batches of every entry (one stack and one mean on `device`, the same operations whatever the number of ranks)."""
    import torch
    if not batches:
        raise ValueError(f"data.val_file holds no whole batch of {batch_size} videos")
    means = torch.stack([b.to(device) if device is not None else b for b in batches]).mean(0).tolist()
    res = {"global_step": int(global_step), "loss": means[0], "videos": len(batches) * batch_size}
    res.update(zip(keys, means[1:]))
    return res


class Validator:
    """Evaluates checkpoints of a pretraining run on data.val_file.  With an eval_ranks.EvalGroup of several ranks, each rank
    evaluates the global batches k with k % world == rank, and every rank gets the result one rank computes."""

    def __init__(self, config, seed: int = 0, device="cuda", group=None):
        from .eval_ranks import EvalGroup
        from .params import ParamStore
        from .train import model_fn_builder, variables_without_gradient
        self.group = group if group is not None else EvalGroup()
        self.config, self.seed, self.device = config, seed, device
        self.batch_size = int(config.device.get("val_batch_size", 16))
        self.num_batches = eval_batch_count(config)
        check_val_file(config)
        self.store = ParamStore(config.model, device=device, optimizer_cfg=config.optimizer)
        self.model_fn = model_fn_builder(config, store=self.store, device=device, seed=seed)
        self.skip = variables_without_gradient(config.model, self.store)

    def _own_batches(self, prefix: str):
        """Restore `prefix` and evaluate this rank's batches.  Returns (metric keys, or None without a batch; one fp32 vector
        [loss, *keys] per batch -- on the device with one rank, host copies for the gather with several)."""
        import torch
        from .dataloader import input_fn_builder
        g = self.group
        self.store.restore_checkpoint(prefix, skip=self.skip)
        keys, out = None, []
        with torch.no_grad(), input_fn_builder(self.config, is_training=False, rank=g.rank, world=g.world, seed=self.seed,
                                               batch_size=self.batch_size, device=self.device) as pipe:
            own = pipe if self.num_batches is None else itertools.islice(pipe, len(range(g.rank, self.num_batches, g.world)))
            for batch in own:
                spec = self.model_fn(batch, None, "eval", {"eval_batch": pipe.last_info["batch"]})
                if keys is None:
                    keys = sorted(k for k in spec.metrics if k.startswith(METRIC_PREFIXES))
                out.append(torch.stack([spec.total_loss.float()] + [spec.metrics[k].float() for k in keys]))
        if g.world > 1:
            out = [v.cpu() for v in out]
        return keys, out

    def evaluate(self, prefix: str) -> Dict:
        """Restore `prefix` and evaluate: {global_step, loss, videos, <metric>: mean, ...}.  With several ranks every rank
        returns the same result; a failure on any rank raises RankFailure on every rank."""
        from .eval_ranks import in_batch_order
        per_rank = self.group.run_and_gather(lambda: self._own_batches(prefix))
        keys = next((k for k, _ in per_rank if k is not None), [])
        return reduce_batches(keys, in_batch_order([vecs for _, vecs in per_rank]), self.batch_size, self.store.global_step,
                              self.device)


def append_result(output_dir: str, res: Dict) -> str:
    """Append the result dict as one JSON line to output_dir/eval/results.jsonl; returns its path."""
    path = os.path.join(output_dir, RESULTS_FILE)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "a", encoding="utf-8") as f:
        f.write(json.dumps(res) + "\n")
    return path


def main(argv=None, clock: Callable[[], float] = time.monotonic, sleep: Callable[[float], None] = time.sleep) -> List[Dict]:
    """Returns the result dict of every evaluated checkpoint, in order."""
    from .config import NeatConfig
    from .eval_ranks import eval_group
    ap = argparse.ArgumentParser(description="Validate pretraining checkpoints on data.val_file")
    ap.add_argument("config_file")
    ap.add_argument("--checkpoint", help="evaluate this checkpoint prefix once instead of following device.output_dir")
    ap.add_argument("--poll-interval", type=float, default=60.0, help="seconds between looks at device.output_dir")
    ap.add_argument("--seed", type=int, default=0, help="seed of the evaluation draws (parser, dropout and masking)")
    args = ap.parse_args(argv)
    config = NeatConfig.from_yaml(args.config_file)
    if config.downstream.get("task") in ("vcr", "video_mc", "video_qa", "video_fib"):
        task = config.downstream.get("task")
        raise ValueError(f"downstream.task is {task!r}: validate {'VCR' if task == 'vcr' else task} fine-tuning with "
                         f"merlot_b200.{task}_validate")
    output_dir = str(config.device["output_dir"])
    if "://" in output_dir:
        raise ValueError(f"device.output_dir {output_dir!r}: only local directories are supported for checkpoints")
    check_val_file(config)
    eval_batch_count(config)

    def follow(sleep_fn):
        if args.checkpoint:
            return iter([args.checkpoint])
        return follow_checkpoints(output_dir, int(config.optimizer.get("num_train_steps", 10)),
                                  float(config.validate.get("eval_timeout", 72000)), args.poll_interval, clock, sleep_fn)

    def write(prefix, res):
        path = append_result(output_dir, res)
        print(f"{prefix}: global_step {res['global_step']} loss {res['loss']:.4f} over {res['videos']} videos -> {path}",
              flush=True)

    results = []
    with eval_group() as group:  # WORLD_SIZE > 1: rank 0 follows the checkpoints and writes, every rank evaluates
        v = Validator(config, seed=args.seed, group=group)
        for prefix in group.shared_prefixes(follow, sleep):
            res = v.evaluate(prefix)
            group.on_rank0(lambda: write(prefix, res))
            results.append(res)
    return results


if __name__ == "__main__":
    main()
