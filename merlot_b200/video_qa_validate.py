"""`python -m merlot_b200.video_qa_validate CONFIG`: validation of open-ended video QA fine-tuning (downstream.task:
video_qa), with the behaviour and options of video_mc_validate.

It follows device.output_dir and evaluates every checkpoint newer than the last one it evaluated (or `--checkpoint PREFIX`
once), restoring a ParamStore(task="video_qa") and running video_qa_model_fn_builder's "eval" mode on the first
validate.eval_samples // device.val_batch_size batches of the evaluation input (video_qa_input), `--chunk N` questions per
forward.  Questions whose answer is outside the vocabulary (answer -1, OOV) are evaluated too, as these benchmarks are
scored.  One JSON line per checkpoint is appended to output_dir/eval/results.jsonl:
  {global_step, accuracy, loss, questions, oov}
accuracy = correct / questions with every OOV question counted wrong; loss = the cross entropy summed over the
in-vocabulary questions divided by their number (a sum and a count over every chunk of every batch, so neither --chunk
nor the number of ranks changes it); oov = questions - in-vocabulary questions.  `--predictions PATH.npz` (with
--checkpoint) writes, per question, id, prediction (the argmax answer), label, and the top k = min(5, A) answers
(`top_k`, int64 [n, k], best first) with their log-probabilities (`top_k_log_prob`).  `--unlabelled` scores records
without answers: no loss, no accuracy, no results line.  Under torchrun the ranks share the work as vcr_validate's do.
"""
from __future__ import annotations

import time
from typing import Callable, Dict, List

import numpy as np

from . import vcr_validate

TOP_K = 5


def top_k(logits: np.ndarray, k: int = TOP_K):
    """(indices int64 [n, min(k, A)], log-probabilities fp32 [n, min(k, A)]) of the most probable answers of fp32 logits
    [n, A], best first (ties: the lower index first)."""
    lp = vcr_validate.log_softmax(logits)
    k = min(k, lp.shape[1])
    idx = np.argsort(-lp, axis=1, kind="stable")[:, :k].astype(np.int64)
    return idx, np.take_along_axis(lp, idx, axis=1)


def results(loss_sums, in_vocab, correct, questions: int) -> Dict:
    """The results line's numbers from the per-chunk sums of every evaluated chunk (any chunking, any rank count):
    accuracy = sum(correct) / questions (OOV questions are never correct), loss = sum(loss_sums) / sum(in_vocab) (None
    without an in-vocabulary question), oov = questions - sum(in_vocab).  Sums in float64."""
    n_iv = float(np.sum(np.asarray(in_vocab, np.float64)))
    loss = float(np.sum(np.asarray(loss_sums, np.float64))) / n_iv if n_iv > 0 else None
    return {"accuracy": float(np.sum(np.asarray(correct, np.float64))) / questions, "loss": loss,
            "oov": questions - int(round(n_iv))}


class Validator(vcr_validate.Validator):
    """vcr_validate.Validator over a video_qa run: ParamStore(task="video_qa", num_answers=A), the video_qa step and
    input, batches of b questions with F frames and one text each; the results line adds `oov`."""
    TASK = "video_qa"
    METRIC = "accuracy"
    ID_KEYS = ("id",)
    EXTRA_KEYS = ("oov",)

    def _store_options(self) -> Dict:
        from .video_qa import check_config
        self.num_frames, self.num_answers = check_config(self.config.model, self.config.downstream)
        return {"num_answers": self.num_answers}

    def _model_fn_builder(self):
        from .video_qa import video_qa_model_fn_builder
        return video_qa_model_fn_builder

    def _input(self, labelled: bool):
        from . import video_qa_input
        g = self.group
        return video_qa_input.input_fn_builder(self.config, is_training=False, rank=g.rank, world=g.world,
                                               batch_size=self.batch_size, device=self.device, labelled=labelled)

    def _chunk(self, batch, a: int, n: int) -> Dict:
        F = self.num_frames
        return {"images": batch["images"][a * F:(a + n) * F], "img_mask": batch["img_mask"][a:a + n],
                "lm_input": batch["lm_input"][a:a + n], "lm_targets": batch["lm_targets"][a:a + n]}

    def _score(self, res: Dict, metrics: Dict, n: int) -> None:
        for k in ("loss_sum", "in_vocab", "correct"):
            res.setdefault(k, []).append(metrics[k].reshape(()))

    def _metrics(self, batches: List[Dict], questions: int) -> Dict:
        import torch
        sums = {k: torch.stack([c.float().cpu() for b in batches for c in b[k]]).double().numpy()
                for k in ("loss_sum", "in_vocab", "correct")}
        return results(sums["loss_sum"], sums["in_vocab"], sums["correct"], questions)

    def _prediction_arrays(self, logits: np.ndarray) -> Dict[str, np.ndarray]:
        idx, lp = top_k(logits)
        return {"prediction": idx[:, 0].copy(), "top_k": idx, "top_k_log_prob": lp}


def main(argv=None, clock: Callable[[], float] = time.monotonic, sleep: Callable[[float], None] = time.sleep):
    """Returns the result dict of every evaluated checkpoint, in order."""
    return vcr_validate.run(Validator, "Validate open-ended video QA fine-tuning checkpoints", "video_qa", argv, clock,
                            sleep)


if __name__ == "__main__":
    main()
