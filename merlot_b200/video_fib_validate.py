"""`python -m merlot_b200.video_fib_validate CONFIG`: validation of fill-in-the-blank video QA (downstream.task:
video_fib), with the behaviour, options and results line of video_qa_validate.

It follows device.output_dir and evaluates every checkpoint newer than the last one it evaluated (or `--checkpoint PREFIX`
once), restoring a ParamStore(task="video_fib") and running video_fib_model_fn_builder's "eval" mode on the first
validate.eval_samples // device.val_batch_size batches of the evaluation input (video_fib_input), `--chunk N` questions
per forward.  One JSON line per checkpoint is appended to output_dir/eval/results.jsonl:
  {global_step, accuracy, loss, questions, oov}
with video_qa_validate's arithmetic (accuracy over every question with OOV ones wrong, loss over the in-vocabulary ones).
`--predictions PATH.npz` (with --checkpoint) writes id, prediction, label and the top min(5, A) answers with their
log-probabilities; `--unlabelled` scores records without answers.

`--zero-shot` (with --checkpoint) evaluates a *pretraining* checkpoint without fine-tuning: the encoder and lm_head are
restored by name (ParamStore.load_checkpoint) and the answer layer is derived from the checkpoint's word embeddings and
output bias (video_fib.init_answer_layer), so the logits are the pretrained MLM's restricted to the answer vocabulary.
global_step is the checkpoint's.  Under torchrun the ranks share the work as vcr_validate's do.
"""
from __future__ import annotations

import time
from typing import Callable, Dict

from . import vcr_validate, video_qa_validate


class Validator(video_qa_validate.Validator):
    """video_qa_validate.Validator over a video_fib run: ParamStore(task="video_fib", num_answers=A), the video_fib step
    and input, batches with blank_pos; zero_shot=True restores pretraining checkpoints by name and derives the answer
    layer."""
    TASK = "video_fib"

    def __init__(self, config, chunk: int = 0, device="cuda", group=None, zero_shot: bool = False):
        self.zero_shot = zero_shot
        super().__init__(config, chunk=chunk, device=device, group=group)

    @classmethod
    def add_arguments(cls, ap) -> None:
        ap.add_argument("--zero-shot", action="store_true",
                        help="evaluate the pretraining checkpoint --checkpoint without fine-tuning: restore it by name and "
                             "derive the answer layer from its word embeddings")

    @classmethod
    def options(cls, args) -> Dict:
        if args.zero_shot and not args.checkpoint:
            raise ValueError("--zero-shot evaluates one pretraining checkpoint: pass --checkpoint PREFIX")
        return {"zero_shot": bool(args.zero_shot)}

    def _store_options(self) -> Dict:
        from .video_fib import check_config
        self.num_frames, self.answers = check_config(self.config.model, self.config.downstream)
        self.num_answers = len(self.answers)
        return {"num_answers": self.num_answers}

    def _model_fn_builder(self):
        from .video_fib import video_fib_model_fn_builder
        return video_fib_model_fn_builder

    def _input(self, labelled: bool):
        from . import video_fib_input
        g = self.group
        return video_fib_input.input_fn_builder(self.config, is_training=False, rank=g.rank, world=g.world,
                                                batch_size=self.batch_size, device=self.device, labelled=labelled)

    def _chunk(self, batch, a: int, n: int) -> Dict:
        return dict(super()._chunk(batch, a, n), blank_pos=batch["blank_pos"][a:a + n])

    def _restore(self, prefix: str) -> None:
        if not self.zero_shot:
            return super()._restore(prefix)
        from .params import VIDEO_FIB_ANSWERS
        from .tf_checkpoint import list_variables, load_checkpoint
        if any(n.startswith(VIDEO_FIB_ANSWERS + "/") for n, _ in list_variables(prefix)):
            raise ValueError(f"--zero-shot {prefix}: the checkpoint holds {VIDEO_FIB_ANSWERS}, a fine-tuned video_fib "
                             f"checkpoint; validate it without --zero-shot")
        from .video_fib import init_answer_layer
        self.store.init_reference(seed=0)
        init_answer_layer(self.store, self.answers, prefix)
        step = load_checkpoint(prefix, names=["global_step"]).get("global_step")
        self.store.global_step = int(step) if step is not None else 0


def main(argv=None, clock: Callable[[], float] = time.monotonic, sleep: Callable[[float], None] = time.sleep):
    """Returns the result dict of every evaluated checkpoint, in order."""
    return vcr_validate.run(Validator, "Validate fill-in-the-blank video QA checkpoints", "video_fib", argv, clock, sleep)


if __name__ == "__main__":
    main()
