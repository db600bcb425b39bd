"""`python -m merlot_b200.predict CONFIG --out DIR [--checkpoint PREFIX] [--seed N]`: model_fn's PREDICT mode on
data.val_file, the role of the reference's Estimator.predict on the pretraining model (model/modeling.py:760-787).

It restores `--checkpoint`, or else the latest checkpoint of device.output_dir (Estimator.predict's default), and runs
model_fn's "predict" mode on the evaluation input (dataloader.EvalInputPipeline): the first validate.eval_samples //
device.val_batch_size batches, or every whole batch when validate.eval_samples is absent (pretrain_validate.eval_batch_count).
Batch k runs with the dropout and masking seed train.eval_seed(--seed, k) and parser draws keyed by (--seed, k), as
pretrain_validate evaluates it, so its losses are the ones pretrain_validate averages.

Global batch k is written to DIR/batch-{k:06d}.npz, the arrays of train.predictions() by name: self_attn_probs (the joint
encoder's attention maps, mean over layers and heads), lang_attn_probs (the language-only encoder's, per layer), masked_ids,
every lang/ attn/ contr/ temporal/ loss and the batch's features other than the images, each leading with the batch's
videos.  read_predictions(DIR) yields them video by video in global order.

Under torchrun with WORLD_SIZE > 1 (eval_ranks) rank r runs and writes the batches k with k % world == r; the ranks exchange
the checkpoint prefix and their status only, never arrays.  A batch's file does not depend on the number of ranks: the same
seeds give the same draws, and the joint maps and attn/ values are summed in a fixed order.  (With masking_use_attn on,
mask_inputs ranks tokens by attention sums added with float atomics, so a near tie may mask another token in any two runs.)
"""
from __future__ import annotations

import argparse
import glob
import itertools
import os
import re
from typing import Dict, Iterator, List, Optional

BATCH_FILE = "batch-{:06d}.npz"
_BATCH_RE = re.compile(r"batch-(\d{6})\.npz")


def batch_files(out_dir: str) -> List[str]:
    """The batch files of `out_dir` in global batch order; raises ValueError when the batch indices are not 0, 1, ..."""
    found = sorted((int(m.group(1)), p) for p in glob.glob(os.path.join(out_dir, "batch-*.npz"))
                   if (m := _BATCH_RE.fullmatch(os.path.basename(p))))
    ks = [k for k, _ in found]
    if ks != list(range(len(ks))):
        raise ValueError(f"{out_dir}: batch files {ks} are not batches 0 .. {len(ks) - 1}")
    return [p for _, p in found]


def read_predictions(out_dir: str) -> Iterator[Dict]:
    """The predictions of `out_dir`, one dict per video in global order: batch by batch, video i of a batch = entry i of
    every array of its file."""
    import numpy as np
    for path in batch_files(out_dir):
        with np.load(path) as z:
            arrays = {name: z[name] for name in z.files}
        n = len(next(iter(arrays.values())))
        for i in range(n):
            yield {name: a[i] for name, a in arrays.items()}


def write_batch(out_dir: str, k: int, arrays: Dict) -> str:
    """DIR/batch-{k:06d}.npz from the arrays by sorted name, through a temporary name so that a file under the final name is
    always whole."""
    import numpy as np
    path = os.path.join(out_dir, BATCH_FILE.format(k))
    tmp = path + ".part"
    with open(tmp, "wb") as f:
        np.savez(f, **{name: arrays[name] for name in sorted(arrays)})
    os.replace(tmp, path)
    return path


class Predictor:
    """model_fn's "predict" mode over this rank's batches of data.val_file (global batches k with k % world == rank)."""

    def __init__(self, config, seed: int = 0, device="cuda", group=None):
        from .eval_ranks import EvalGroup
        from .params import ParamStore
        from .pretrain_validate import check_val_file, eval_batch_count
        from .train import model_fn_builder, variables_without_gradient
        self.group = group if group is not None else EvalGroup()
        self.config, self.seed, self.device = config, seed, device
        self.batch_size = int(config.device.get("val_batch_size", 16))
        self.num_batches = eval_batch_count(config)
        check_val_file(config)
        self.store = ParamStore(config.model, device=device, optimizer_cfg=config.optimizer)
        self.model_fn = model_fn_builder(config, store=self.store, device=device, seed=seed)
        self.skip = variables_without_gradient(config.model, self.store)

    def batches(self, prefix: str) -> Iterator:
        """Restore `prefix`; yield (k, predictions of global batch k) for this rank's batches."""
        import torch
        from .dataloader import input_fn_builder
        g = self.group
        self.store.restore_checkpoint(prefix, skip=self.skip)
        with torch.no_grad(), input_fn_builder(self.config, is_training=False, rank=g.rank, world=g.world, seed=self.seed,
                                               batch_size=self.batch_size, device=self.device) as pipe:
            own = pipe if self.num_batches is None else itertools.islice(pipe, len(range(g.rank, self.num_batches, g.world)))
            for batch in own:
                k = pipe.last_info["batch"]
                yield k, self.model_fn(batch, None, "predict", {"eval_batch": k, "batch_size": self.batch_size})

    def write(self, prefix: str, out_dir: str) -> int:
        """Restore `prefix` and write this rank's batch files into out_dir; returns how many it wrote."""
        n = 0
        for k, arrays in self.batches(prefix):
            write_batch(out_dir, k, arrays)
            n += 1
        return n


def main(argv=None) -> Optional[List[str]]:
    """Returns the batch files of --out in global order (on every rank)."""
    from .config import NeatConfig
    from .eval_ranks import eval_group
    from .pretrain_validate import check_val_file, eval_batch_count
    from .tf_checkpoint import latest_checkpoint
    ap = argparse.ArgumentParser(description="Predict with a pretraining checkpoint on data.val_file (model_fn PREDICT)")
    ap.add_argument("config_file")
    ap.add_argument("--out", required=True, help="directory of the batch-{k:06d}.npz files")
    ap.add_argument("--checkpoint", help="checkpoint prefix (default: the latest checkpoint of device.output_dir)")
    ap.add_argument("--seed", type=int, default=0, help="seed of the evaluation draws (parser, dropout and masking)")
    args = ap.parse_args(argv)
    config = NeatConfig.from_yaml(args.config_file)
    if config.downstream.get("task") in ("vcr", "video_mc", "video_qa", "video_fib"):
        raise ValueError(f"downstream.task is {config.downstream.get('task')!r}: PREDICT runs on the pretraining model")
    check_val_file(config)
    eval_batch_count(config)
    prefix = args.checkpoint
    if not prefix:
        output_dir = str(config.device["output_dir"])
        if "://" in output_dir:
            raise ValueError(f"device.output_dir {output_dir!r}: only local directories are supported for checkpoints")
        prefix = latest_checkpoint(output_dir)
        if prefix is None:
            raise ValueError(f"device.output_dir {output_dir!r} holds no checkpoint: pass --checkpoint PREFIX")
    elif not os.path.exists(prefix + ".index"):
        raise ValueError(f"--checkpoint {prefix!r}: no {prefix}.index")
    if glob.glob(os.path.join(args.out, "batch-*.npz")):
        raise ValueError(f"--out {args.out!r} already holds batch files: give an empty or new directory")
    os.makedirs(args.out, exist_ok=True)

    with eval_group() as group:  # WORLD_SIZE > 1: every rank writes its own batches
        prefix = group.broadcast(prefix)
        p = Predictor(config, seed=args.seed, group=group)
        written = sum(group.run_and_gather(lambda: p.write(prefix, args.out)))
        files = batch_files(args.out)
        if len(files) != written:
            raise RuntimeError(f"{args.out}: {len(files)} batch files after writing {written}")
        group.on_rank0(lambda: print(f"{prefix}: {written} batches of {p.batch_size} videos -> {args.out}", flush=True))
    return files


if __name__ == "__main__":
    main()
