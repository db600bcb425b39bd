"""Multiple-choice video QA records to batches (downstream.task: video_mc), built like vcr_input.py.

A record is one tf.train.Example per question (INTEGRATION.md, "Multiple-choice video QA"):
  id               bytes
  frames/encoded   bytes list: 1..F JPEGs in time order (F = model.num_imgs)
  question         int64 token ids
  choice_0 .. choice_{C-1}   int64 token ids each (C = model.num_texts)
  label            int64; absent reads as -1

  * parse   -- `parse_question`: candidate text i is [START] + question + choice_i + [END], int64 -> int32, padded with
               PADDING and truncated to downstream.max_text_len (a long text loses its END).  Zero frames, more than F
               frames, a missing choice or a token id outside [0, vocab_size) raise ValueError naming the record's id.
  * labels  -- `check_labels`: a label outside [0, C) raises on the host in a labelled run, naming the id.  The CE kernel
               reads the logit of the label unchecked, so an unlabelled record (-1) must never reach it.
  * pixels  -- Pillow decodes the JPEGs in the pipeline's thread pool; K14 (`ops.frames_prepare`) resizes every frame slot
               of the batch in one launch.  Training draws one scale and crop of resize_and_pad(do_random_scale=True, 0.9,
               1.1) per question from NumPy keyed by (seed, rank) and applies it to all of the question's frames; evaluation
               uses the do_random_scale=False plan.  An empty slot (a question with k < F frames, slots k..F-1) is planned
               as a 1x1 black source, which K14 resizes to an all-zero frame.
  * batches -- images [b*F, H, W, 3] bf16 (question-major, frame-minor), img_mask [b, F] bool (False at empty slots),
               lm_input [b*C, L] int32 (question-major), lm_targets [b] int32, and id (host strings): the shapes
               video_mc.video_mc_model_fn_builder takes.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from .config import micro_batching
from .dataloader import (DEFAULT_NUM_THREADS, DevicePipeline, decode_jpeg, eval_decode_threads, plan_frames, plan_frames_eval,
                         shard_files, shuffled_records, stage_frames, train_files)
from .sort_story import eval_batches, val_files
from .tfrecord import parse_example
from .vcr_input import END, PADDING, RANDOM_SCALE_MAX, RANDOM_SCALE_MIN, START, _to_device
from .video_mc import check_config

DEFAULT_MAX_TEXT_LEN = 128


def _id(example) -> str:
    v = example.get("id")
    return bytes(v[0]).decode("utf-8", "replace") if v else ""


def _tokens(example, key: str, rid: str, vocab_size: int, required: bool, task: str = "video_mc") -> np.ndarray:
    v = example.get(key)
    if v is None:
        if required:
            raise ValueError(f"{task} record id={rid!r}: {key} is missing")
        v = []
    t = np.asarray(v, dtype=np.int64)
    bad = np.flatnonzero((t < 0) | (t >= vocab_size))
    if len(bad):
        raise ValueError(f"{task} record id={rid!r}: {key} holds token id {int(t[bad[0]])} outside the vocabulary "
                         f"[0, {vocab_size})")
    return t


def parse_question(example, num_frames: int, num_choices: int, max_len: int, vocab_size: int) -> Dict:
    """One parsed record without its pixels: {id (str), jpegs (list of 1..num_frames bytes), label (int, -1 if absent),
    lm_input int32 [num_choices, max_len]}.  Raises ValueError naming the id on the record errors the module lists."""
    rid = _id(example)
    jpegs = [bytes(x) for x in example.get("frames/encoded", [])]
    if not 1 <= len(jpegs) <= num_frames:
        raise ValueError(f"video_mc record id={rid!r}: {len(jpegs)} frames, expected 1 to {num_frames} (model.num_imgs)")
    q = _tokens(example, "question", rid, vocab_size, required=False)
    lm = np.full((num_choices, max_len), PADDING, dtype=np.int32)
    for i in range(num_choices):
        c = _tokens(example, f"choice_{i}", rid, vocab_size, required=True)
        toks = np.concatenate([[START], q, c, [END]]).astype(np.int64).astype(np.int32)[:max_len]
        lm[i, :len(toks)] = toks
    v = example.get("label")
    if v is not None and len(v) != 1:
        raise ValueError(f"video_mc record id={rid!r}: label has {len(v)} values, expected 1")
    return {"id": rid, "jpegs": jpegs, "label": int(v[0]) if v is not None else -1, "lm_input": lm}


def check_labels(questions: Sequence[Dict], num_choices: int) -> None:
    """Raise ValueError naming the id of the first question whose label is outside [0, num_choices)."""
    for q in questions:
        if not 0 <= q["label"] < num_choices:
            raise ValueError(f"video_mc record id={q['id']!r}: label is {q['label']}, outside [0, {num_choices}) (an "
                             f"unlabelled record can only be scored without a loss)")


def decode_frame(question: Dict, k: int, task: str = "video_mc") -> np.ndarray:
    """Frame k of a parsed question as uint8 [h, w, 3] RGB; an undecodable frame raises naming the id (and `task`)."""
    try:
        return decode_jpeg(question["jpegs"][k])
    except Exception as e:
        raise ValueError(f"{task} record id={question['id']!r}: frame {k} cannot be decoded ({type(e).__name__}: {e})") from e


def img_mask(questions: Sequence[Dict], num_frames: int) -> np.ndarray:
    """bool [b, num_frames]: slot f of question q holds a frame iff f < its frame count."""
    counts = np.array([len(q["jpegs"]) for q in questions])
    return np.arange(num_frames)[None] < counts[:, None]


def train_draws(rng: np.random.Generator, n: int) -> Dict[str, np.ndarray]:
    """VCR's training resize draws (vcr_input.train_plan) for n questions: scale U[0.9, 1.1) and the crop's uniforms."""
    f32 = np.float32
    lo, hi = f32(RANDOM_SCALE_MIN), f32(RANDOM_SCALE_MAX)
    return {"scale": lo + rng.random(n, dtype=f32) * (hi - lo), "u_y": rng.random(n, dtype=f32), "u_x": rng.random(n, dtype=f32)}


def _prepare(pool, device, questions, num_frames, out_size, draws=None, task: str = "video_mc"):
    """Decode every frame in `pool`, plan every slot of the batch (question-major, frame-minor) and run K14 once: bf16
    [b * num_frames, H, W, 3] on `device`, the img_mask [b, num_frames] and the plan.  `draws` (train_draws of the
    questions) selects the training plan, None the evaluation plan.  Errors name the record's id and `task`."""
    from . import ops
    mask = img_mask(questions, num_frames)
    decodes = {(i, k): pool.submit(decode_frame, q, k, task) for i, q in enumerate(questions) for k in range(len(q["jpegs"]))}
    black = np.zeros((1, 1, 3), np.uint8)  # the source of every empty slot
    frames = [decodes[(i, k)].result() if mask[i, k] else black for i in range(len(questions)) for k in range(num_frames)]
    staging, offsets, hw = stage_frames(frames)
    if draws is None:
        plan = plan_frames_eval(hw[:, 0], hw[:, 1], out_size)
    else:
        per_slot = {k: np.repeat(v, num_frames) for k, v in draws.items()}
        plan = dict(plan_frames(hw[:, 0], hw[:, 1], out_size, **per_slot), **per_slot)
    empty = ~mask.reshape(-1)
    plan["scaled_h"][empty], plan["scaled_w"][empty] = out_size[0], out_size[1]
    plan["offset_y"][empty], plan["offset_x"][empty] = 0, 0
    bad = np.flatnonzero((plan["scaled_h"] < 1) | (plan["scaled_w"] < 1))
    if len(bad):
        s = int(bad[0])
        raise ValueError(f"{task} record id={questions[s // num_frames]['id']!r}: frame {s % num_frames} of "
                         f"{hw[s, 0]}x{hw[s, 1]} pixels resizes to {plan['scaled_h'][s]}x{plan['scaled_w'][s]} for "
                         f"image_size {list(out_size)}")
    n = len(hw)
    plan.update(src_offset=offsets, src_h=hw[:, 0], src_w=hw[:, 1], method=np.zeros(n, np.int32),
                augment=np.zeros(n, np.int32), factor=np.ones((n, 3), np.float32))
    return ops.frames_prepare(staging.to(device, non_blocking=True), plan, *out_size), mask, plan


class _Pipeline(DevicePipeline):
    """What the training and evaluation pipelines share: the shapes of the config and the batch of parsed records.  A
    task with other records (video_qa_input) overrides TASK and the three methods after __init__."""
    TASK = "video_mc"

    def __init__(self, config, files, batch_size, labelled, num_threads, device, prefetch):
        self._configure(config)
        self.max_len = int(config.downstream.get("max_text_len", DEFAULT_MAX_TEXT_LEN))
        self.vocab_size = int(config.model["vocab_size"])
        self.out_size = tuple(config.model["image_size"])
        self.files = list(files)
        self.batch_size = batch_size
        self.labelled = labelled
        super().__init__(device, num_threads, prefetch)

    def _configure(self, config):
        self.num_frames, self.num_choices = check_config(config.model)

    def _parse(self, record) -> Dict:
        """One record as its parsed question (parse_question)."""
        return parse_question(parse_example(record), self.num_frames, self.num_choices, self.max_len, self.vocab_size)

    def _text_fields(self, qs) -> Dict[str, np.ndarray]:
        """The batch's host arrays besides the frames: lm_input [b*C, L] and lm_targets [b]; checks labels if labelled."""
        if self.labelled:
            check_labels(qs, self.num_choices)
        return {"lm_input": np.stack([q["lm_input"] for q in qs]).reshape(len(qs) * self.num_choices, self.max_len),
                "lm_targets": np.array([q["label"] for q in qs], dtype=np.int32)}

    def _batch(self, records, draws_fn=None, qs=None):
        if qs is None:
            qs = [self._parse(r) for r in records]
        text = self._text_fields(qs)
        draws = draws_fn(len(qs)) if draws_fn is not None else None
        images, mask, plan = _prepare(self._pool, self.device, qs, self.num_frames, self.out_size, draws, self.TASK)
        feats = {"images": images, "img_mask": _to_device(mask, self.device),
                 **{k: _to_device(v, self.device) for k, v in text.items()}, "id": [q["id"] for q in qs]}
        return feats, {"records": list(records), "id": feats["id"], "plan": plan, "draws": draws}


class VideoMCTrainPipeline(_Pipeline):
    """Iterator of training batches of b questions on `device`: the files listed in a shuffled order, repeated forever,
    interleaved over min(data.num_threads, files) readers, a data.shuffle_buffer_size (default 64) shuffle buffer, batches
    with drop_remainder (as vcr_input.VCRTrainPipeline).  Labels must lie in [0, C).  `last_info` holds the records, ids,
    frame plan and per-question draws behind the batch returned last."""

    def __init__(self, config, files: Sequence[str], batch_size: int, rank: int = 0, seed: int = 0, device=None,
                 prefetch: int = 2):
        num_threads = config.data.get("num_threads", 64)
        self.cycle_length = min(num_threads, len(files))
        self.shuffle_buffer_size = config.data.get("shuffle_buffer_size", 64)
        self.rng = np.random.default_rng([seed, rank])
        super().__init__(config, files, batch_size, True, num_threads, device, prefetch)

    def _produce(self):
        recs = shuffled_records(self.files, self.rng, self.cycle_length, self.shuffle_buffer_size, self._stop)
        while not self._stop.is_set():
            yield self._batch([next(recs) for _ in range(self.batch_size)], lambda n: train_draws(self.rng, n))


class VideoMCEvalPipeline(_Pipeline):
    """Iterator of evaluation batches of b questions: the files in the given order, interleaved over min(data.num_threads,
    files) readers, no shuffle, no repeat, the do_random_scale=False plan.  `labelled=False` lets labels outside [0, C)
    through (no loss may be computed on them).  A last partial batch is not returned; after the iteration ends `dropped` is
    the number of records it held.  As rank `rank` of `world` evaluation processes it returns the global batches k with
    k % world == rank (sort_story.eval_batches); `dropped` stays the global count."""

    def __init__(self, config, files: Sequence[str], batch_size: int, labelled: bool = True, device=None, prefetch: int = 2,
                 rank: int = 0, world: int = 1):
        self.rank, self.world = rank, world
        self.cycle_length = min(config.data.get("num_threads", DEFAULT_NUM_THREADS), len(files))
        self.dropped = None
        super().__init__(config, files, batch_size, labelled, eval_decode_threads(config.data), device, prefetch)

    def _produce(self):
        tail: List = []
        for records in eval_batches(self.files, self.cycle_length, self.batch_size, tail, self._stop, self.rank, self.world):
            yield self._batch(records)
        self.dropped = len(tail)


def input_fn_builder(config, is_training: bool = True, rank: int = 0, world: int = 1, seed: int = 0,
                     batch_size: Optional[int] = None, device=None, labelled: bool = True):
    """Training: the files of data.train_file sharded by rank (shard_files), batches of `batch_size` questions (default:
    the micro-batch of config.micro_batching).  Evaluation: the files of data.val_file in sorted glob order, batches of
    `batch_size` questions (default device.val_batch_size), of which rank `rank` of `world` gets the global batches k with
    k % world == rank.  Returns the running pipeline (close() it)."""
    return _input_fn(VideoMCTrainPipeline, VideoMCEvalPipeline, config, is_training, rank, world, seed, batch_size, device,
                     labelled)


def _input_fn(train_cls, eval_cls, config, is_training, rank, world, seed, batch_size, device, labelled):
    """input_fn_builder with the training and evaluation pipeline classes of a task."""
    if is_training:
        files = train_files(config.data)
        if not files:
            raise ValueError(f"data.train_file {config.data.get('train_file')!r} matches no file")
        files = shard_files(files, rank, world)
        if batch_size is None:
            batch_size = micro_batching(config.device, world, default_batch_size=64)[1]
        return train_cls(config, files, batch_size, rank=rank, seed=seed, device=device)
    files = val_files(config)
    if not files:
        raise ValueError(f"data.val_file {config.data.get('val_file')!r} matches no file")
    if batch_size is None:
        batch_size = config.device.get("val_batch_size", 64)
    return eval_cls(config, files, batch_size, labelled=labelled, device=device, rank=rank, world=world)
