"""Open-ended video QA records to batches (downstream.task: video_qa), on video_mc_input's frame path.

A record is one tf.train.Example per question (INTEGRATION.md, "Open-ended video QA"):
  id               bytes
  frames/encoded   bytes list: 1..F JPEGs in time order (F = model.num_imgs)
  question         int64 token ids
  answer           int64: the answer's index in the vocabulary [0, A), or -1 when it is not in it (OOV); absent in an
                   unlabelled run

  * parse   -- `parse_question`: the text is [START] + question + [END], int64 -> int32, padded with PADDING and
               truncated to downstream.max_text_len.  Zero frames, more than F frames or a token id outside
               [0, vocab_size) raise ValueError naming the record's id (video_mc_input's rules).
  * answers -- `check_answers`: in a labelled run a missing answer, or one outside [-1, A), raises naming the id.
  * OOV     -- training skips questions whose answer is -1 (`take_answerable`; the pipeline counts them in `skipped`);
               evaluation keeps them, and the step gives them weight 0 (video_qa.qa_loss).
  * pixels  -- video_mc_input's: Pillow decode, one K14 launch per batch, one random-scale draw per question in training,
               empty frame slots all zero with img_mask False.
  * batches -- images [b*F, H, W, 3] bf16 (question-major, frame-minor), img_mask [b, F] bool, lm_input [b, L] int32,
               lm_targets [b] int32 (-1 for OOV, and for every question of an unlabelled run), and id (host strings).
"""
from __future__ import annotations

from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from .dataloader import shuffled_records
from .tfrecord import parse_example
from .vcr_input import END, PADDING, START
from .video_mc_input import VideoMCEvalPipeline, VideoMCTrainPipeline, _id, _input_fn, _tokens, train_draws
from .video_qa import check_config

def parse_question(example, num_frames: int, max_len: int, vocab_size: int, task: str = "video_qa") -> Dict:
    """One parsed record without its pixels: {id (str), jpegs (list of 1..num_frames bytes), answer (int, None if
    absent), lm_input int32 [max_len]}.  Raises ValueError naming the id (and `task`) on the record errors the module
    lists."""
    rid = _id(example)
    jpegs = [bytes(x) for x in example.get("frames/encoded", [])]
    if not 1 <= len(jpegs) <= num_frames:
        raise ValueError(f"{task} record id={rid!r}: {len(jpegs)} frames, expected 1 to {num_frames} (model.num_imgs)")
    q = _tokens(example, "question", rid, vocab_size, required=False, task=task)
    toks = np.concatenate([[START], q, [END]]).astype(np.int64).astype(np.int32)[:max_len]
    lm = np.full(max_len, PADDING, dtype=np.int32)
    lm[:len(toks)] = toks
    v = example.get("answer")
    if v is not None and len(v) != 1:
        raise ValueError(f"{task} record id={rid!r}: answer has {len(v)} values, expected 1")
    return {"id": rid, "jpegs": jpegs, "answer": int(v[0]) if v is not None else None, "lm_input": lm}


def check_answers(questions: Sequence[Dict], num_answers: int, task: str = "video_qa") -> None:
    """Raise ValueError naming the id (and `task`) of the first question without an answer or with one outside
    [-1, num_answers)."""
    for q in questions:
        if q["answer"] is None:
            raise ValueError(f"{task} record id={q['id']!r}: answer is missing (an unlabelled record can only be scored "
                             f"without a loss)")
        if not -1 <= q["answer"] < num_answers:
            raise ValueError(f"{task} record id={q['id']!r}: answer is {q['answer']}, outside [-1, {num_answers}) "
                             f"(-1 marks an answer outside the vocabulary)")


def labels(questions: Sequence[Dict]) -> np.ndarray:
    """int32 [b]: each question's answer, -1 for OOV and for a question without an answer."""
    return np.array([-1 if q["answer"] is None else q["answer"] for q in questions], dtype=np.int32)


def take_answerable(records: Iterator, n: int, parse, num_answers: int,
                    task: str = "video_qa") -> Tuple[List, List[Dict], int]:
    """The next n records of `records` whose answer is in the vocabulary, their parsed questions, and the number of OOV
    questions passed over on the way.  Every record is parsed and checked (check_answers) first."""
    recs, qs, skipped = [], [], 0
    while len(qs) < n:
        r = next(records)
        q = parse(r)
        check_answers([q], num_answers, task)
        if q["answer"] < 0:
            skipped += 1
            continue
        recs.append(r)
        qs.append(q)
    return recs, qs, skipped


class _QA:
    """video_qa's records on video_mc_input's pipelines: the parser and the text and label fields of a batch."""
    TASK = "video_qa"

    def _configure(self, config):
        self.num_frames, self.num_answers = check_config(config.model, config.downstream)

    def _parse(self, record) -> Dict:
        return parse_question(parse_example(record), self.num_frames, self.max_len, self.vocab_size)

    def _text_fields(self, qs) -> Dict[str, np.ndarray]:
        if self.labelled:
            check_answers(qs, self.num_answers)
        return {"lm_input": np.stack([q["lm_input"] for q in qs]), "lm_targets": labels(qs)}


class VideoQATrainPipeline(_QA, VideoMCTrainPipeline):
    """Iterator of training batches of b questions, as video_mc_input.VideoMCTrainPipeline reads them (shuffled files
    repeated forever, interleaved readers, a shuffle buffer, drop_remainder), that leaves out every OOV question.
    `skipped` counts the OOV questions left out so far."""

    def __init__(self, *args, **kw):
        self.skipped = 0
        super().__init__(*args, **kw)

    def _produce(self):
        recs = shuffled_records(self.files, self.rng, self.cycle_length, self.shuffle_buffer_size, self._stop)
        while not self._stop.is_set():
            records, qs, skipped = take_answerable(recs, self.batch_size, self._parse, self.num_answers, self.TASK)
            self.skipped += skipped
            yield self._batch(records, lambda n: train_draws(self.rng, n), qs=qs)


class VideoQAEvalPipeline(_QA, VideoMCEvalPipeline):
    """Iterator of evaluation batches of b questions, OOV questions included, as video_mc_input.VideoMCEvalPipeline
    reads them (files in order, no shuffle, no repeat, `dropped` the records of a last partial batch, global batch k on
    rank k % world).  `labelled=False` lets records without an answer through (no loss may be computed on them)."""


def input_fn_builder(config, is_training: bool = True, rank: int = 0, world: int = 1, seed: int = 0,
                     batch_size: Optional[int] = None, device=None, labelled: bool = True):
    """video_mc_input.input_fn_builder over video_qa records: data.train_file sharded by rank, or data.val_file in sorted
    glob order.  Returns the running pipeline (close() it)."""
    return _input_fn(VideoQATrainPipeline, VideoQAEvalPipeline, config, is_training, rank, world, seed, batch_size, device,
                     labelled)
