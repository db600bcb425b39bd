"""VCR records to batches: the joint training input (downstream/vcr/dataloader_joint.py) and the per-mode evaluation input
(downstream/vcr/dataloader.py), restated on the host like the pretraining pipeline (dataloader.py).

  * parse   -- `parse_question`: img_id, annot_id, the `{mode}/{data.draw}/image/encoded` JPEG of every mode used, the label
               (`label/{mode}_label`, -1 when absent) and the four candidate texts VCR_PROMPT[mode] + ctx + choice_i + [END],
               int64 -> int32, padded with PADDING and truncated to MAX_NUM_TOKENS (a long text loses its END).  The
               `*_tags` features are never read: the reference parses them and does not use them.
  * labels  -- `check_labels`: a label outside [0, 4) raises on the host, naming the annot_id.  The CE kernel reads the logit
               of the label unchecked, so an unlabelled record (-1) must never reach it; scoring such records is the
               validator's predictions-only mode, which runs no loss.
  * pixels  -- Pillow decodes the JPEGs in the pipeline's thread pool; K14 (`ops.frames_prepare`) does convert_image_dtype,
               resize_and_pad (bilinear, no augmentation) and the bf16 cast in one launch per batch.  Training draws the
               scale and crop of resize_and_pad(do_random_scale=True, 0.9, 1.1) from NumPy keyed by (seed, rank), like the
               pretraining input; evaluation uses the do_random_scale=False plan.
  * batches -- training: images [2b, H, W, 3] in the order [q0 answer, q0 rationale, q1 answer, ...], lm_input [2b*4, 184],
               lm_targets [2b]; evaluation: images [b, H, W, 3], lm_input [b, 4, L_mode], lm_targets [b], plus annot_id and
               img_id as host strings.  These are the shapes vcr.vcr_model_fn_builder takes.

VCR_PROMPT holds the reference tokenizer's encodings as constants (checked against tests/golden/vcr_prompts.json), so
the tokenizer is not needed at run time.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from .dataloader import (DEFAULT_NUM_THREADS, DevicePipeline, decode_jpeg, eval_decode_threads, plan_frames, plan_frames_eval,
                         shard_files, shuffled_records, stage_frames, train_files)
from .config import micro_batching
from .sort_story import eval_batches, val_files
from .tfrecord import parse_example

PADDING, START, END = 0, 2, 3  # utils/encode/encoder.py
MODES = ("answer", "rationale")
VCR_PROMPT = {"answer": (START, 3380, 1908, 125),       # [START] + encode(' answer question:')
              "rationale": (START, 2248, 25838, 125)}   # [START] + encode(' provide rationale:')
JOINT_MAX_NUM_TOKENS = 184                              # dataloader_joint.py:135
EVAL_MAX_NUM_TOKENS = {"answer": 134, "rationale": 184}  # dataloader.py:116
RANDOM_SCALE_MIN, RANDOM_SCALE_MAX = 0.9, 1.1            # the VCR parser's resize_and_pad arguments, not data.random_scale_*
NUM_CHOICES = 4


def _string(example, key: str) -> str:
    """A FixedLenFeature((), tf.string, default_value='') as text."""
    v = example.get(key)
    return bytes(v[0]).decode("utf-8", "replace") if v else ""


def candidate_texts(example, mode: str, max_tokens: int) -> np.ndarray:
    """int32 [4, max_tokens]: VCR_PROMPT[mode] + {mode}/ctx + {mode}/choice_i + [END] per candidate (absent lists are empty),
    cast int64 -> int32, then pad_to_fixed_size(PADDING, truncate=True)."""
    out = np.full((NUM_CHOICES, max_tokens), PADDING, dtype=np.int32)
    ctx = np.asarray(example.get(f"{mode}/ctx", []), dtype=np.int64)
    for i in range(NUM_CHOICES):
        toks = np.concatenate([np.asarray(VCR_PROMPT[mode], np.int64), ctx,
                               np.asarray(example.get(f"{mode}/choice_{i}", []), dtype=np.int64), [END]])
        toks = toks.astype(np.int32)[:max_tokens]
        out[i, :len(toks)] = toks
    return out


def parse_question(example, modes: Sequence[str], draw: str, max_tokens: Dict[str, int]) -> Dict:
    """One parsed VCR record without its pixels: img_id and annot_id (str), and per mode of `modes` its encoded image
    (b'' if absent), its label (-1 if absent) and its candidate texts.  Returns {img_id, annot_id, jpegs [len(modes)],
    labels int64 [len(modes)], lm_input int32 [len(modes), 4, L]} (every mode's L must agree)."""
    labels = []
    for mode in modes:
        v = example.get(f"label/{mode}_label")
        if v is not None and len(v) != 1:
            raise ValueError(f"VCR feature label/{mode}_label has {len(v)} values, expected 1")
        labels.append(int(v[0]) if v is not None else -1)
    return {"img_id": _string(example, "img_id"), "annot_id": _string(example, "annot_id"),
            "jpegs": [bytes(example[k][0]) if example.get(k) else b"" for k in
                      (f"{mode}/{draw}/image/encoded" for mode in modes)],
            "labels": np.array(labels, dtype=np.int64),
            "lm_input": np.stack([candidate_texts(example, mode, max_tokens[mode]) for mode in modes])}


def check_labels(questions: Sequence[Dict], modes: Sequence[str]) -> None:
    """Raise ValueError naming the annot_id of the first question whose label is outside [0, NUM_CHOICES)."""
    for q in questions:
        for mode, lab in zip(modes, q["labels"]):
            if not 0 <= lab < NUM_CHOICES:
                raise ValueError(f"VCR record annot_id={q['annot_id']!r}: label/{mode}_label is {int(lab)}, outside "
                                 f"[0, {NUM_CHOICES}) (an unlabelled record can only be scored without a loss)")


def decode_image(question: Dict, k: int, mode: str) -> np.ndarray:
    """Image k of a parsed question as uint8 [h, w, 3] RGB; a missing or undecodable image raises naming the annot_id."""
    buf = question["jpegs"][k]
    if not buf:
        raise ValueError(f"VCR record annot_id={question['annot_id']!r}: the {mode} image is missing")
    try:
        return decode_jpeg(buf)
    except Exception as e:
        raise ValueError(f"VCR record annot_id={question['annot_id']!r}: the {mode} image cannot be decoded "
                         f"({type(e).__name__}: {e})") from e


def train_plan(rng: np.random.Generator, hw: np.ndarray, out_size: Sequence[int]) -> Dict[str, np.ndarray]:
    """resize_and_pad(do_random_scale=True, random_scale_min=0.9, random_scale_max=1.1)'s plan of frames with heights and
    widths hw [n, 2]: the scale factor U[0.9, 1.1) and the two crop offsets' uniforms drawn from `rng` (kept in the plan as
    scale, u_y, u_x), then dataloader.plan_frames (with its 64-pixel floor)."""
    f32, n = np.float32, len(hw)
    lo, hi = f32(RANDOM_SCALE_MIN), f32(RANDOM_SCALE_MAX)
    draws = {"scale": lo + rng.random(n, dtype=f32) * (hi - lo), "u_y": rng.random(n, dtype=f32), "u_x": rng.random(n, dtype=f32)}
    return dict(plan_frames(hw[:, 0], hw[:, 1], out_size, **draws), **draws)


def _prepare(pool, device, questions, modes, out_size, plan_fn):
    """Decode every question's images (question-major, mode-minor) in `pool`, plan them with plan_fn(hw) and run K14 once:
    bf16 [len(questions) * len(modes), H, W, 3] on `device`, and the plan."""
    from . import ops
    decodes = [pool.submit(decode_image, q, k, mode) for q in questions for k, mode in enumerate(modes)]
    staging, offsets, hw = stage_frames([d.result() for d in decodes])
    plan = plan_fn(hw)
    bad = np.flatnonzero((plan["scaled_h"] < 1) | (plan["scaled_w"] < 1))
    if len(bad):
        k = int(bad[0])
        raise ValueError(f"VCR record annot_id={questions[k // len(modes)]['annot_id']!r}: the {modes[k % len(modes)]} image "
                         f"of {hw[k, 0]}x{hw[k, 1]} pixels resizes to {plan['scaled_h'][k]}x{plan['scaled_w'][k]} for "
                         f"image_size {list(out_size)}")
    n = len(hw)
    plan.update(src_offset=offsets, src_h=hw[:, 0], src_w=hw[:, 1], method=np.zeros(n, np.int32),
                augment=np.zeros(n, np.int32), factor=np.ones((n, 3), np.float32))
    return ops.frames_prepare(staging.to(device, non_blocking=True), plan, *out_size), plan


def _to_device(a: np.ndarray, device):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)


class VCRTrainPipeline(DevicePipeline):
    """Iterator of joint training batches {images bf16 [2b, H, W, 3], lm_input int32 [2b*4, 184], lm_targets int32 [2b]} on
    `device` (dataloader_joint.py:197-277): the files listed in a shuffled order, repeated forever, interleaved over
    min(data.num_threads, files) readers, a data.shuffle_buffer_size (default 64) shuffle buffer, batches of b questions
    with drop_remainder.  `last_info` holds the records, ids and frame plan (with its draws) behind the batch returned last."""

    def __init__(self, config, files: Sequence[str], batch_size: int, rank: int = 0, seed: int = 0, device=None,
                 prefetch: int = 2):
        self.files = list(files)
        self.batch_size = batch_size
        self.draw = config.data.get("draw", "segm")
        self.out_size = tuple(config.model["image_size"])
        num_threads = config.data.get("num_threads", 64)
        self.cycle_length = min(num_threads, len(self.files))
        self.shuffle_buffer_size = config.data.get("shuffle_buffer_size", 64)
        self.rng = np.random.default_rng([seed, rank])
        super().__init__(device, num_threads, prefetch)

    def _batch(self, records):
        qs = [parse_question(parse_example(r), MODES, self.draw, {m: JOINT_MAX_NUM_TOKENS for m in MODES}) for r in records]
        check_labels(qs, MODES)
        n = 2 * len(qs)
        images, plan = _prepare(self._pool, self.device, qs, MODES, self.out_size,
                                lambda hw: train_plan(self.rng, hw, self.out_size))
        feats = {"images": images,
                 "lm_input": _to_device(np.stack([q["lm_input"] for q in qs]).reshape(n * NUM_CHOICES, JOINT_MAX_NUM_TOKENS),
                                        self.device),
                 "lm_targets": _to_device(np.stack([q["labels"] for q in qs]).reshape(n).astype(np.int32), self.device)}
        info = {"records": list(records), "annot_id": [q["annot_id"] for q in qs], "img_id": [q["img_id"] for q in qs],
                "plan": plan}
        return feats, info

    def _produce(self):
        recs = shuffled_records(self.files, self.rng, self.cycle_length, self.shuffle_buffer_size, self._stop)
        while not self._stop.is_set():
            yield self._batch([next(recs) for _ in range(self.batch_size)])


class VCREvalPipeline(DevicePipeline):
    """Iterator of evaluation batches of one mode {images bf16 [b, H, W, 3], lm_input int32 [b, 4, L_mode], lm_targets int32
    [b] (on `device`), annot_id, img_id (lists of str)} (dataloader.py:161-211 with is_training=False): the files in the given
    order, interleaved over min(data.num_threads, files) readers, no shuffle, no repeat.  `labelled=False` lets labels
    outside [0, 4) through (they are returned as read; no loss may be computed on them).  A last partial batch is not
    returned; after the iteration ends `dropped` is the number of records it held.  As rank `rank` of `world` evaluation
    processes it returns the batches k with k % world == rank (sort_story.eval_batches); `dropped` stays the global count."""

    def __init__(self, config, files: Sequence[str], batch_size: int, mode: str, labelled: bool = True, device=None,
                 prefetch: int = 2, rank: int = 0, world: int = 1):
        if mode not in MODES:
            raise ValueError(f"downstream.mode must be one of {MODES}, got {mode!r}")
        self.files = list(files)
        self.batch_size = batch_size
        self.mode, self.labelled = mode, labelled
        self.rank, self.world = rank, world
        self.draw = config.data.get("draw", "segm")
        self.out_size = tuple(config.model["image_size"])
        num_threads = config.data.get("num_threads", DEFAULT_NUM_THREADS)
        self.cycle_length = min(num_threads, len(self.files))
        self.dropped = None
        super().__init__(device, eval_decode_threads(config.data), prefetch)

    def _batch(self, records):
        modes = (self.mode,)
        qs = [parse_question(parse_example(r), modes, self.draw, EVAL_MAX_NUM_TOKENS) for r in records]
        if self.labelled:
            check_labels(qs, modes)
        images, plan = _prepare(self._pool, self.device, qs, modes, self.out_size,
                                lambda hw: plan_frames_eval(hw[:, 0], hw[:, 1], self.out_size))
        feats = {"images": images, "lm_input": _to_device(np.stack([q["lm_input"][0] for q in qs]), self.device),
                 "lm_targets": _to_device(np.array([q["labels"][0] for q in qs], dtype=np.int32), self.device),
                 "annot_id": [q["annot_id"] for q in qs], "img_id": [q["img_id"] for q in qs]}
        return feats, {"records": list(records), "plan": plan}

    def _produce(self):
        tail: List = []
        for records in eval_batches(self.files, self.cycle_length, self.batch_size, tail, self._stop, self.rank, self.world):
            yield self._batch(records)
        self.dropped = len(tail)


def input_fn_builder(config, is_training: bool = True, rank: int = 0, world: int = 1, seed: int = 0,
                     batch_size: Optional[int] = None, device=None, labelled: bool = True):
    """dataloader_joint.input_fn_builder(is_training=True) or dataloader.input_fn_builder(is_training=False).  Training: the
    files of data.train_file sharded by rank (shard_files), batches of `batch_size` questions (default: the micro-batch of
    config.micro_batching, device.train_batch_size // world without device.micro_batch_size).  Evaluation: the files of data.val_file in sorted glob order, the downstream.mode
    input, batches of `batch_size` questions (default device.val_batch_size), of which rank `rank` of `world` gets the
    batches k with k % world == rank.  Returns the running pipeline (close() it)."""
    if is_training:
        files = train_files(config.data)
        if not files:
            raise ValueError(f"data.train_file {config.data.get('train_file')!r} matches no file")
        files = shard_files(files, rank, world)
        if batch_size is None:
            batch_size = micro_batching(config.device, world, default_batch_size=64)[1]
        return VCRTrainPipeline(config, files, batch_size, rank=rank, seed=seed, device=device)
    files = val_files(config)
    if not files:
        raise ValueError(f"data.val_file {config.data.get('val_file')!r} matches no file")
    if batch_size is None:
        batch_size = config.device.get("val_batch_size", 64)
    return VCREvalPipeline(config, files, batch_size, config.downstream.get("mode", "answer"), labelled=labelled,
                           device=device, rank=rank, world=world)
