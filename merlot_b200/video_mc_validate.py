"""`python -m merlot_b200.video_mc_validate CONFIG`: validation of multiple-choice video QA fine-tuning (downstream.task:
video_mc), with the behaviour of vcr_validate.

It follows device.output_dir and evaluates every checkpoint newer than the last one it evaluated, oldest first, until the
checkpoint whose global_step reaches optimizer.num_train_steps or validate.eval_timeout seconds without a new one
(vcr_validate.follow_checkpoints); `--checkpoint PREFIX` evaluates one prefix and exits.  Per checkpoint the trainer's
restore path fills a ParamStore(task="video_mc"), and video_mc_model_fn_builder's "eval" mode runs on the first
validate.eval_samples // device.val_batch_size batches of the evaluation input (video_mc_input); the remainder is not
evaluated.  `--chunk N` runs a batch N questions at a time (no dropout, no term across questions: the means do not change).
One JSON line per checkpoint, {global_step, accuracy, loss (mean of the per-batch losses), questions}, is appended to
output_dir/eval/results.jsonl.  `--predictions PATH.npz` (with --checkpoint) also writes, per question, id, log_prob [C],
prediction and label.  `--unlabelled` scores records without labels: forward and head only, no loss, no accuracy and no
results line.  Under torchrun with WORLD_SIZE > 1 the ranks share the work as vcr_validate's do (eval_ranks), and the
results line and the predictions are those of one process.
"""
from __future__ import annotations

import time
from typing import Callable, Dict

from . import vcr_validate


class Validator(vcr_validate.Validator):
    """vcr_validate.Validator over a video_mc run: ParamStore(task="video_mc"), the video_mc step and input, batches of
    b questions with F frames and C candidates each."""
    TASK = "video_mc"
    METRIC = "accuracy"
    ID_KEYS = ("id",)

    def _model_fn_builder(self):
        from .video_mc import check_config, video_mc_model_fn_builder
        self.num_frames, self.num_choices = check_config(self.config.model)
        return video_mc_model_fn_builder

    def _input(self, labelled: bool):
        from . import video_mc_input
        g = self.group
        return video_mc_input.input_fn_builder(self.config, is_training=False, rank=g.rank, world=g.world,
                                               batch_size=self.batch_size, device=self.device, labelled=labelled)

    def _chunk(self, batch, a: int, n: int) -> Dict:
        F, C = self.num_frames, self.num_choices
        return {"images": batch["images"][a * F:(a + n) * F], "img_mask": batch["img_mask"][a:a + n],
                "lm_input": batch["lm_input"][a * C:(a + n) * C], "lm_targets": batch["lm_targets"][a:a + n]}


def main(argv=None, clock: Callable[[], float] = time.monotonic, sleep: Callable[[float], None] = time.sleep):
    """Returns the result dict of every evaluated checkpoint, in order."""
    return vcr_validate.run(Validator, "Validate multiple-choice video QA fine-tuning checkpoints", "video_mc", argv, clock,
                            sleep)


if __name__ == "__main__":
    main()
