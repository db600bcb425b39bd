"""`python -m merlot_b200.vcr_validate CONFIG`: VCR validation, the role of downstream/vcr/validate.py.

It follows device.output_dir the way tf.contrib.training.checkpoints_iterator does and evaluates every checkpoint newer than
the last one it evaluated, oldest first.  It stops after the checkpoint whose global_step reaches optimizer.num_train_steps,
or once validate.eval_timeout seconds pass without a new checkpoint.  `--checkpoint PREFIX` evaluates one prefix and exits.

Per checkpoint the trainer's restore path (ParamStore.restore_checkpoint, with its name, shape, dtype and checksum checks)
fills a ParamStore(task="vcr"), and the downstream.mode tower is evaluated through vcr_model_fn_builder's "eval" mode on
the first validate.eval_samples // device.val_batch_size batches of the evaluation input (vcr_input).  Like the
reference's `steps=`, the remainder is not evaluated.  A batch can be run in chunks of `--chunk` questions: evaluation has
no dropout and no term across questions, so the means do not change.  One JSON line per checkpoint, {global_step, avg
(mean accuracy, the reference's metric name), loss (mean of the per-batch losses), questions}, is appended to
output_dir/eval/results.jsonl.  `--predictions PATH.npz` (with --checkpoint) also writes, per question, annot_id, img_id,
log_prob [4], prediction and label: the reference's cls_metric / PREDICT dict.  `--unlabelled` scores records without
labels: forward and head only, no loss, no accuracy and no results line.

Under torchrun with WORLD_SIZE > 1 (eval_ranks): rank 0 alone follows device.output_dir and broadcasts each prefix it
chooses, then "stop"; every rank restores the prefix and evaluates the global batches k with k % world == rank; every rank
gathers the per-batch results in global batch order and computes the one-process result from them; rank 0 alone appends
the results line and writes the predictions.  `--checkpoint`, `--chunk` and `--unlabelled` mean what they mean on one GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import time
from typing import Callable, Dict, Iterator, List

import numpy as np

RESULTS_FILE = os.path.join("eval", "results.jsonl")


def checkpoint_step(prefix: str) -> int:
    """The global step in a model.ckpt-<step> prefix (validate.py:48)."""
    m = re.search(r"-(\d+)$", os.path.basename(prefix))
    if m is None:
        raise ValueError(f"{prefix!r} is not a model.ckpt-<global_step> prefix")
    return int(m.group(1))


def follow_checkpoints(directory: str, num_train_steps: int, timeout: float, poll_interval: float = 60.0,
                       clock: Callable[[], float] = time.monotonic,
                       sleep: Callable[[float], None] = time.sleep) -> Iterator[str]:
    """Yield the checkpoint prefixes of `directory` (those its state file lists) as they appear, each one newer than the
    last yielded, oldest first.  Ends after a checkpoint whose step is >= num_train_steps, or when `timeout` seconds of
    `clock` pass after the last yield (or the start) without a new checkpoint.  Polls every `poll_interval` seconds."""
    from .tf_checkpoint import checkpoint_prefixes
    last = -1
    deadline = clock() + timeout
    while True:
        new = sorted((checkpoint_step(p), p) for p in checkpoint_prefixes(directory) if checkpoint_step(p) > last)
        if new:
            for step, prefix in new:
                yield prefix
                last = step
                if step >= num_train_steps:
                    return
            deadline = clock() + timeout
            continue
        if clock() >= deadline:
            return
        sleep(poll_interval)


def log_softmax(logits: np.ndarray) -> np.ndarray:
    """cls_metric's log_prob of fp32 logits [n, 4], computed in float64 and returned as float32."""
    x = np.asarray(logits, np.float64)
    x = x - x.max(-1, keepdims=True)
    return (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)


class Validator:
    """Evaluates checkpoints of a VCR run on the evaluation input of config (data.val_file, downstream.mode).  With an
    eval_ranks.EvalGroup of several ranks, each rank evaluates the global batches k with k % world == rank, and every rank
    gets the result one rank would compute.  video_mc_validate.Validator, video_qa_validate.Validator and
    video_fib_validate.Validator are this class over other tasks: the class attributes and the methods between __init__ and
    _own_batches are what a task sets."""
    TASK = "vcr"
    METRIC = "avg"                     # the results line's name of the mean accuracy
    ID_KEYS = ("annot_id", "img_id")   # per-question host strings of a batch, kept in the predictions
    EXTRA_KEYS = ()                    # results-line entries after global_step, METRIC, loss and questions

    def __init__(self, config, chunk: int = 0, device="cuda", group=None):
        from .eval_ranks import EvalGroup
        from .params import ParamStore
        self.group = group if group is not None else EvalGroup()
        self.config = config
        self.batch_size = int(config.device.get("val_batch_size", 64))
        self.chunk = chunk if chunk > 0 else self.batch_size
        self.num_batches = int(config.validate.get("eval_samples", 0)) // self.batch_size
        if self.num_batches < 1:
            raise ValueError(f"validate.eval_samples {config.validate.get('eval_samples')!r} is less than one batch of "
                             f"device.val_batch_size {self.batch_size}")
        self.store = ParamStore(config.model, device=device, optimizer_cfg=config.optimizer, task=self.TASK,
                                **self._store_options())
        self.model_fn = self._model_fn_builder()(config, store=self.store, device=device)
        self.device = device

    @classmethod
    def add_arguments(cls, ap: argparse.ArgumentParser) -> None:
        """Add the task's own command-line options to `run`'s parser."""

    @classmethod
    def options(cls, args) -> Dict:
        """Keyword arguments of the constructor from the parsed command line besides config, chunk and group."""
        return {}

    def _store_options(self) -> Dict:
        """Keyword arguments of the task's ParamStore besides the model config and the task."""
        return {}

    def _restore(self, prefix: str) -> None:
        """Fill self.store from checkpoint `prefix`: the trainer's strict restore (parameters, slots, global_step)."""
        self.store.restore_checkpoint(prefix)

    def _model_fn_builder(self):
        from .vcr import vcr_model_fn_builder
        return vcr_model_fn_builder

    def _input(self, labelled: bool):
        from . import vcr_input
        g = self.group
        return vcr_input.input_fn_builder(self.config, is_training=False, rank=g.rank, world=g.world,
                                          batch_size=self.batch_size, device=self.device, labelled=labelled)

    def _chunk(self, batch, a: int, n: int) -> Dict:
        """The features of questions a .. a+n-1 of an evaluation batch."""
        return {k: batch[k][a:a + n] for k in ("images", "lm_input", "lm_targets")}

    def _score(self, res: Dict, metrics: Dict, n: int) -> None:
        """Add the eval metrics of a labelled chunk of n questions to its batch's `res` (res['loss'], a device scalar, and
        the lists of device scalars in res)."""
        res["loss"] += metrics["loss"] * (n / self.batch_size)  # cls_loss gives chunk means; weigh them by the chunk's share
        res["correct"].append(metrics["accuracy"] * n)

    def _metrics(self, batches: List[Dict], questions: int) -> Dict:
        """{METRIC, loss} of the labelled batches in global batch order, on this rank's device."""
        import torch
        dev = self.device
        losses = [b["loss"].to(dev) for b in batches]
        correct = [c.to(dev) for b in batches for c in b["correct"]]
        return {self.METRIC: float(torch.stack(correct).sum()) / questions, "loss": float(torch.stack(losses).mean())}

    def _prediction_arrays(self, logits: np.ndarray) -> Dict[str, np.ndarray]:
        """The per-question arrays of the predictions file computed from the fp32 logits [n, classes]."""
        lp = log_softmax(logits)
        return {"log_prob": lp, "prediction": lp.argmax(-1).astype(np.int64)}

    def _own_batches(self, prefix: str, labelled: bool, keep_predictions: bool) -> List[Dict]:
        """Restore `prefix` and evaluate this rank's batches among the first num_batches.  Per batch: its loss (a device
        scalar), the correct count of every chunk, and with keep_predictions every chunk's logits and the batch's ids and
        labels.  With several ranks the tensors are copied to the host for the gather."""
        import torch
        g = self.group
        self._restore(prefix)
        mode = "eval" if labelled else "predict"
        out = []
        with torch.no_grad(), self._input(labelled) as pipe:
            for _, batch in zip(range(len(range(g.rank, self.num_batches, g.world))), pipe):
                res = {"loss": torch.zeros((), dtype=torch.float32, device=self.device), "correct": [], "logits": []}
                for a in range(0, self.batch_size, self.chunk):
                    feats = self._chunk(batch, a, self.chunk)
                    spec = self.model_fn(feats, None, mode)
                    n = feats["lm_targets"].shape[0]
                    if labelled:
                        self._score(res, spec.metrics, n)
                    if keep_predictions:
                        res["logits"].append(spec.metrics["logits"].clone())
                if keep_predictions:
                    res.update({k: batch[k] for k in self.ID_KEYS}, label=batch["lm_targets"].cpu().numpy())
                out.append(res)
        if g.world > 1:  # host copies for the gather
            for b in out:
                for k, v in b.items():
                    if torch.is_tensor(v):
                        b[k] = v.cpu()
                    elif isinstance(v, list) and v and torch.is_tensor(v[0]):
                        b[k] = [x.cpu() for x in v]
        return out

    def evaluate(self, prefix: str, labelled: bool = True, keep_predictions: bool = False) -> Dict:
        """Restore `prefix` and evaluate.  Returns {global_step, METRIC, loss, questions} (METRIC and loss None when not
        labelled), plus per-question arrays under 'predictions' when keep_predictions.  With several ranks every rank
        returns the same result, reduced in global batch order on this rank's device by the same operations one rank
        runs; a failure on any rank raises RankFailure on every rank."""
        import torch
        from .eval_ranks import in_batch_order
        per_rank = self.group.run_and_gather(lambda: self._own_batches(prefix, labelled, keep_predictions))
        batches = in_batch_order(per_rank)
        dev = self.device
        logits = [x.to(dev) for b in batches for x in b["logits"]]
        rows = {k: [a for b in batches for a in b.get(k, [])] for k in self.ID_KEYS}
        rows["label"] = [b["label"] for b in batches if "label" in b]
        questions = len(batches) * self.batch_size
        if questions == 0:
            raise ValueError(f"data.val_file holds no whole batch of {self.batch_size} questions")
        res = {"global_step": self.store.global_step, self.METRIC: None, "loss": None, "questions": questions}
        res.update({k: None for k in self.EXTRA_KEYS})
        if labelled:
            res.update(self._metrics(batches, questions))
        if keep_predictions:
            lg = torch.cat(logits).float().cpu().numpy()
            res["predictions"] = dict({k: np.array(rows[k]) for k in self.ID_KEYS}, **self._prediction_arrays(lg),
                                      label=np.concatenate(rows["label"]).astype(np.int64))
        return res


def append_result(output_dir: str, res: Dict, metric: str = "avg", extra=()) -> str:
    """Append {global_step, <metric>, loss, questions, *extra} as one JSON line to output_dir/eval/results.jsonl; returns
    its path."""
    path = os.path.join(output_dir, RESULTS_FILE)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "a", encoding="utf-8") as f:
        f.write(json.dumps({k: res[k] for k in ("global_step", metric, "loss", "questions") + tuple(extra)}) + "\n")
    return path


def write_predictions(path: str, predictions: Dict[str, np.ndarray]) -> None:
    np.savez(path, **predictions)


def main(argv=None, clock: Callable[[], float] = time.monotonic, sleep: Callable[[float], None] = time.sleep):
    """Returns the result dict of every evaluated checkpoint, in order."""
    return run(Validator, "Validate VCR fine-tuning checkpoints (downstream/vcr/validate.py)", "VCR", argv, clock, sleep)


def run(validator_cls, description: str, task_name: str, argv=None, clock: Callable[[], float] = time.monotonic,
        sleep: Callable[[float], None] = time.sleep):
    """The command line of a validator: follow device.output_dir (or evaluate --checkpoint) with `validator_cls` on every
    rank, rank 0 writing the results lines and predictions.  Returns the result dict of every evaluated checkpoint."""
    from .config import NeatConfig
    ap = argparse.ArgumentParser(description=description)
    ap.add_argument("config_file")
    ap.add_argument("--checkpoint", help="evaluate this checkpoint prefix once instead of following device.output_dir")
    ap.add_argument("--predictions", help="write per-question predictions to this .npz (needs --checkpoint)")
    ap.add_argument("--unlabelled", action="store_true",
                    help="the records have no labels: predictions only, no loss or accuracy (needs --predictions)")
    ap.add_argument("--chunk", type=int, default=0, help="questions per forward (default: device.val_batch_size)")
    ap.add_argument("--poll-interval", type=float, default=60.0, help="seconds between looks at device.output_dir")
    validator_cls.add_arguments(ap)
    args = ap.parse_args(argv)
    if args.predictions and not args.checkpoint:
        raise ValueError("--predictions writes one checkpoint's predictions: pass --checkpoint PREFIX")
    if args.predictions and not args.predictions.endswith(".npz"):
        raise ValueError(f"--predictions {args.predictions!r}: the file must be an .npz")
    if args.unlabelled and not args.predictions:
        raise ValueError("--unlabelled computes no metrics: pass --predictions PATH.npz")
    if args.chunk < 0:
        raise ValueError(f"--chunk {args.chunk} must be >= 0")
    options = validator_cls.options(args)
    config = NeatConfig.from_yaml(args.config_file)
    if config.downstream.get("task") != validator_cls.TASK:
        raise ValueError(f"downstream.task is {config.downstream.get('task')!r}, {task_name} validation needs "
                         f"{validator_cls.TASK!r}")
    output_dir = str(config.device["output_dir"])
    if "://" in output_dir:
        raise ValueError(f"device.output_dir {output_dir!r}: only local directories are supported for checkpoints")
    from .eval_ranks import eval_group

    def follow(sleep_fn):
        if args.checkpoint:
            return iter([args.checkpoint])
        return follow_checkpoints(output_dir, int(config.optimizer.get("num_train_steps", 10)),
                                  float(config.validate.get("eval_timeout", 72000)), args.poll_interval, clock, sleep_fn)

    def write(prefix, res):
        if args.predictions:
            write_predictions(args.predictions, res["predictions"])
        if not args.unlabelled:
            metric = validator_cls.METRIC
            path = append_result(output_dir, res, metric, validator_cls.EXTRA_KEYS)
            loss = "none" if res["loss"] is None else f"{res['loss']:.4f}"  # video_qa: no in-vocabulary question
            print(f"{prefix}: global_step {res['global_step']} {metric} {res[metric]:.4f} loss {loss} over "
                  f"{res['questions']} questions -> {path}", flush=True)
        else:
            print(f"{prefix}: predictions of {res['questions']} questions -> {args.predictions}", flush=True)

    results = []
    with eval_group() as group:  # WORLD_SIZE > 1: rank 0 follows the checkpoints and writes, every rank evaluates
        v = validator_cls(config, chunk=args.chunk, group=group, **options)
        for prefix in group.shared_prefixes(follow, sleep):
            res = v.evaluate(prefix, labelled=not args.unlabelled, keep_predictions=bool(args.predictions))
            group.on_rank0(lambda: write(prefix, res))
            res.pop("predictions", None)
            results.append(res)
    return results


if __name__ == "__main__":
    main()
