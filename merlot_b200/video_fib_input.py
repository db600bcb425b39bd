"""Fill-in-the-blank video QA records to batches (downstream.task: video_fib), on video_mc_input's frame path as
video_qa_input is.

A record is one tf.train.Example per question (INTEGRATION.md, "Fill-in-the-blank video QA"):
  id               bytes
  frames/encoded   bytes list: 1..F JPEGs in time order (F = model.num_imgs)
  question         int64 token ids of the sentence, holding the blank as one MASK (id 1)
  answer           int64: the answer's index in the vocabulary [0, A), or -1 when it is not in it (OOV); absent in an
                   unlabelled run

  * parse   -- `parse_question`: the text is [START] + question + [END], int64 -> int32, padded with PADDING and
               truncated to downstream.max_text_len.  A question without a MASK or with more than one, a MASK lost to the
               truncation, and video_qa_input's frame and token errors raise ValueError naming the record's id.
  * answers -- video_qa_input.check_answers: in a labelled run a missing answer, or one outside [-1, A), raises.
  * OOV     -- training skips questions whose answer is -1; evaluation keeps them (video_qa_input's rules).
  * batches -- video_qa_input's fields (images, img_mask, lm_input, lm_targets, id) and blank_pos [b] int32, the MASK's
               position in lm_input.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from .modeling import MASK
from .tfrecord import parse_example
from .video_fib import check_config
from .video_mc_input import VideoMCEvalPipeline, _input_fn
from .video_qa_input import VideoQATrainPipeline, check_answers, labels
from .video_qa_input import parse_question as parse_qa_question


def parse_question(example, num_frames: int, max_len: int, vocab_size: int) -> Dict:
    """One parsed record without its pixels: video_qa_input.parse_question's {id, jpegs, answer, lm_input} and blank_pos
    (int), the MASK's position in lm_input.  Raises ValueError naming the id on the record errors the module lists."""
    q = parse_qa_question(example, num_frames, max_len, vocab_size, task="video_fib")
    words = example.get("question")
    n = int(np.count_nonzero(np.asarray([] if words is None else words, dtype=np.int64) == MASK))
    if n != 1:
        raise ValueError(f"video_fib record id={q['id']!r}: question holds {n} MASK tokens (id {MASK}), expected exactly one "
                         f"blank")
    pos = np.flatnonzero(q["lm_input"] == MASK)
    if len(pos) != 1:
        raise ValueError(f"video_fib record id={q['id']!r}: the MASK (the blank) is cut off by downstream.max_text_len "
                         f"{max_len}")
    q["blank_pos"] = int(pos[0])
    return q


class _FiB:
    """video_fib's records on video_mc_input's pipelines: the parser and the text and label fields of a batch."""
    TASK = "video_fib"

    def _configure(self, config):
        self.num_frames, answers = check_config(config.model, config.downstream)
        self.num_answers = len(answers)

    def _parse(self, record) -> Dict:
        return parse_question(parse_example(record), self.num_frames, self.max_len, self.vocab_size)

    def _text_fields(self, qs) -> Dict[str, np.ndarray]:
        if self.labelled:
            check_answers(qs, self.num_answers, self.TASK)
        return {"lm_input": np.stack([q["lm_input"] for q in qs]), "lm_targets": labels(qs),
                "blank_pos": np.array([q["blank_pos"] for q in qs], dtype=np.int32)}


class VideoFiBTrainPipeline(_FiB, VideoQATrainPipeline):
    """video_qa_input.VideoQATrainPipeline over video_fib records: shuffled, repeated, OOV questions left out and counted
    in `skipped`."""


class VideoFiBEvalPipeline(_FiB, VideoMCEvalPipeline):
    """video_qa_input.VideoQAEvalPipeline over video_fib records: files in order, OOV questions kept, global batch k on
    rank k % world; `labelled=False` lets records without an answer through."""


def input_fn_builder(config, is_training: bool = True, rank: int = 0, world: int = 1, seed: int = 0,
                     batch_size: Optional[int] = None, device=None, labelled: bool = True):
    """video_mc_input.input_fn_builder over video_fib records: data.train_file sharded by rank, or data.val_file in sorted
    glob order.  Returns the running pipeline (close() it)."""
    return _input_fn(VideoFiBTrainPipeline, VideoFiBEvalPipeline, config, is_training, rank, world, seed, batch_size, device,
                     labelled)
