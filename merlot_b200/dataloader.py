"""The reference's pretraining input pipeline (model/dataloader.py) -- SURVEY.md 8(f) next-row 4.

Per example (`_dataset_parser`, :56-126), on the host: TFRecord reading and tf.train.Example decoding (tfrecord.py), the text
and metadata fields (`parse_text`), JPEG decoding with Pillow in a thread pool (`decode_jpeg`), and the per-frame plan of
resize_and_pad (`frame_draws`, `plan_frames`).  The per-pixel work -- convert, resize, crop, pad, augment, bf16 -- is K14
(csrc/frames.cu, `ops.frames_prepare`) on a data stream of its own.  `input_fn_builder` (:129-278) ties them together.

The random draws come from a NumPy generator keyed by (seed, rank), not from TensorFlow's bit stream, which cannot be
reproduced without TensorFlow: the distributions are the reference's, the individual values are not.

Batch-level step (`_process_example`, :210-272), below.  It runs on whatever device the feature tensors live on (plain index
arithmetic: argsort / gather / where), so the step can stay on the GPU next to the model instead of in a tf.data map on the host.

  * shuffle_chunks (:211-224)   -- permute whole source videos inside a row: [A A A A B B] -> [B B A A A A]
  * frame shuffle (:226-257)    -- per group of `num_chunks_in_group` segments draw how many frames are out of place
                                   (categorical over [1-p, 1e-6, p/(n-1), ...]), pick that many positions, give them the ids
                                   16 + random order; everything else keeps arange(n).  The offset 16 (< 64) is why every
                                   temporal pair weighs 0.01 in pretraining (SURVEY quirk 4).
  * flatten + transpose (:259-264) -- images [b, n, h, w, 3] -> [b*n, h, w, 3] (-> [h, w, 3, b*n] when training with
                                   `transpose_input`, undone by model_fn, modeling.py:683-685)

The reference draws its random numbers with tf.random.*; `draws` injects them so the integer results can be compared bit for
bit with the NumPy restatement in oracle/oracle_np.py (tests/test_host_logic.py).
"""
from __future__ import annotations

import collections
import glob
import io
import math
import queue
import threading
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from .tfrecord import parse_example, read_records

SHUFFLE_OFFSET = 16  # model/dataloader.py:227
_PER_CHUNK_KEYS = ("youtube_id", "chunk_num", "mean_time", "images", "input_ids", "is_eoc", "video_src_ids")  # :222


def num_shuffle_probs(num_chunks_in_group: int, shuffle_prob: float):
    """:243-244 -- P(k frames out of place) for k = 0..n: [1-p, 1e-6, p/(n-1) x (n-1)] (one frame out of place is no shuffle)."""
    n = num_chunks_in_group
    return [1.0 - shuffle_prob, 1e-6] + [shuffle_prob / (n - 1) for _ in range(n - 1)]


def make_draws(batch_size: int, num_chunks: int, num_chunks_in_group: int, shuffle_prob: float, seed: int, device="cpu"):
    """The four random tensors `_process_example` draws, from a seed (tf.random_uniform x3, tf.random.categorical x1)."""
    g = torch.Generator().manual_seed(seed)
    B = batch_size * num_chunks // num_chunks_in_group
    probs = torch.tensor(num_shuffle_probs(num_chunks_in_group, max(shuffle_prob, 1e-6)), dtype=torch.float64)
    d = {
        "chunk_u": torch.rand(batch_size, num_chunks, generator=g),
        "num_shuffle": torch.multinomial(probs / probs.sum(), B, True, generator=g).to(torch.int32),
        "pick_u": torch.rand(B, num_chunks_in_group, generator=g),
        "order_u": torch.rand(B, num_chunks_in_group, generator=g),
    }
    return {k: v.to(device) for k, v in d.items()}


def process_example(features: Dict[str, torch.Tensor], data_cfg: dict, model_cfg: dict, is_training: bool = True,
                    draws: Optional[Dict[str, torch.Tensor]] = None, seed: int = 0) -> Dict[str, torch.Tensor]:
    """model/dataloader.py:210-272.  `features`: images [b, n, h, w, 3], input_ids [b, n, L], video_src_ids [b, n] (+ any of the
    other per-chunk keys).  Returns a new dict with `shuffled_idx_img` [B*g] int32 added and images flattened."""
    out = dict(features)
    ids = out["input_ids"]
    if ids.dim() != 3:
        raise ValueError(f"input_ids must be [batch, num_chunks, L], got {tuple(ids.shape)}")
    b, n, _ = ids.shape
    g = model_cfg.get("num_chunks_in_group", n)
    if (b * n) % g != 0:
        raise ValueError(f"batch*num_chunks = {b * n} is not divisible by num_chunks_in_group = {g}")
    B = b * n // g
    p = model_cfg.get("image_shuffle_prob", 0.5)  # :226 (merged data+model config; the key lives in `model:`)
    dev = ids.device
    if draws is None:
        draws = make_draws(b, n, g, p, seed, dev)

    if data_cfg.get("shuffle_chunks", False):  # :211-224
        vid = out["video_src_ids"].long()
        mapping = torch.argsort(draws["chunk_u"].to(dev), dim=-1, stable=True)
        new_chunkid = torch.gather(mapping, 1, vid)
        trg = new_chunkid * n + torch.arange(n, device=dev)[None]
        idx = torch.argsort(trg, dim=1, stable=True)
        for k in _PER_CHUNK_KEYS:
            if k in out:
                v = out[k]
                ix = idx.reshape(b, n, *([1] * (v.dim() - 2))).expand(b, n, *v.shape[2:])
                out[k] = torch.gather(v, 1, ix)

    base = torch.arange(g, dtype=torch.int32, device=dev)[None].expand(B, g)
    if p < 1e-6:  # :234-237
        shuffled = base
    else:  # :238-257
        num_shuffle = draws["num_shuffle"].to(dev).to(torch.int32)
        do_shuffle = torch.argsort(draws["pick_u"].to(dev), dim=1, stable=True).to(torch.int32) < num_shuffle[:, None]
        order = torch.argsort(draws["order_u"].to(dev), dim=1, stable=True).to(torch.int32)
        shuffled = torch.where(do_shuffle, SHUFFLE_OFFSET + order, base)
    out["shuffled_idx_img"] = shuffled.reshape(-1).contiguous()

    img = out["images"]
    if img.dim() != 5 or img.shape[-1] != 3:
        raise ValueError(f"images must be [batch, num_chunks, h, w, 3], got {tuple(img.shape)}")
    img = img.reshape(b * img.shape[1], *img.shape[2:])  # :260-261
    if is_training and model_cfg.get("transpose_input", False):  # :262-264
        img = img.permute(1, 2, 3, 0)
    out["images"] = img
    return out


def expected_out_of_place(num_chunks_in_group: int, shuffle_prob: float) -> float:
    """The figure the reference logs (:245-247)."""
    return math.fsum(i * q for i, q in enumerate(num_shuffle_probs(num_chunks_in_group, shuffle_prob)))


# ---------------------------------------------------------------------------------------------------------------------------
# per-example parser (model/dataloader.py:19-126)
# ---------------------------------------------------------------------------------------------------------------------------
START, NEXTCAPTION_START = 2, 5  # utils/encode/encoder.py
YOUTUBE_ID_LEN = 64              # encode_string(., 64), :66
AUGMENT_DELTA = 0.8 * 0.4        # lightweight_image_augment: max_{brightness,contrast}_delta = 0.8 * strength


def _scalar(example, key: str, default):
    """A FixedLenFeature((), dtype, default) of the chunk_k2f schema (:19-31)."""
    v = example.get(key)
    if v is None:
        return default
    if len(v) != 1:
        raise ValueError(f"Example feature {key!r} has {len(v)} values, expected 1")
    return v[0]


def frame_bytes(example, num_chunks: int) -> List[bytes]:
    """The encoded frames c00/image/encoded .. c{n-1}/image/encoded."""
    return [_scalar(example, f"c{i:02d}/image/encoded", b"") for i in range(num_chunks)]


def parse_text(example, num_chunks: int, chunk_text_len: int, do_clean: bool) -> Dict[str, np.ndarray]:
    """The text and metadata features of `_dataset_parser` (:65-69, :100-125) for one example and one do_clean draw:
    youtube_id [n, 64] int32, chunk_num [n] int32, mean_time [n] f32, input_ids [n, chunk_text_len] int32, is_eoc [n] bool,
    video_src_ids [n] int32."""
    n, L = num_chunks, chunk_text_len
    key = "tokenized_cleaned_asr" if do_clean else "tokenized_raw_asr"
    start = START if do_clean else NEXTCAPTION_START
    ids = np.zeros((n, L), dtype=np.int32)
    yid = np.zeros((n, YOUTUBE_ID_LEN), dtype=np.int32)
    for i in range(n):
        toks = np.concatenate([[start], np.asarray(example.get(f"c{i:02d}/{key}", []), dtype=np.int64)])
        toks = toks.astype(np.int32)[:L]  # tf.cast(int64 -> int32), then pad_to_fixed_size(truncate=True)
        ids[i, :len(toks)] = toks
        raw = np.frombuffer(_scalar(example, f"c{i:02d}/youtube_id", b""), dtype=np.uint8)[:YOUTUBE_ID_LEN]
        yid[i, :len(raw)] = raw
    is_eoc = np.array([_scalar(example, f"c{i:02d}/is_eoc", 1) for i in range(n - 1)] + [1], dtype=np.int64) != 0
    return {
        "youtube_id": yid,
        "chunk_num": np.array([_scalar(example, f"c{i:02d}/chunk_num", 1) for i in range(n)], dtype=np.int64).astype(np.int32),
        "mean_time": np.array([_scalar(example, f"c{i:02d}/mean_time", 1.0) for i in range(n)], dtype=np.float32),
        "input_ids": ids,
        "is_eoc": is_eoc,
        "video_src_ids": np.cumsum(np.concatenate([[0], is_eoc[:-1].astype(np.int32)])).astype(np.int32),
    }


def decode_jpeg(buf: bytes) -> np.ndarray:
    """tf.image.decode_jpeg(channels=3) with Pillow: uint8 [h, w, 3] RGB (grayscale replicated).  Pillow releases the GIL while
    it decodes, so a thread pool decodes in parallel."""
    from PIL import Image
    with Image.open(io.BytesIO(buf)) as im:
        return np.asarray(im.convert("RGB"))


def frame_draws(rng: np.random.Generator, n: int, data_cfg: dict) -> Dict[str, np.ndarray]:
    """The random draws of n frames' `_load_and_resize_img` (:72-89): the scale factor and the two crop offsets of
    resize_and_pad (utils/model_utils.py:877,896-897), the resize method (apply_with_random_selector, :912-915; TF1 ResizeMethod
    order 0 bilinear, 1 nearest, 2 bicubic, 3 area), and lightweight_image_augment's Bernoulli(augment_prob), transform
    (1 brightness, 2 contrast; 0 = not augmented) and per-channel factor U[1 - 0.32, 1 + 0.32)."""
    f32 = np.float32
    lo, hi = f32(data_cfg.get("random_scale_min", 0.95)), f32(data_cfg.get("random_scale_max", 1.05))
    scale = lo + rng.random(n, dtype=f32) * (hi - lo)
    u_y, u_x = rng.random(n, dtype=f32), rng.random(n, dtype=f32)
    method = rng.integers(0, 4, n).astype(np.int32)
    p = data_cfg.get("augment_prob", 0.0)
    augmented = rng.random(n) < p if p > 0.0 else np.zeros(n, dtype=bool)  # augmentation only when augment_prob > 0 (:85)
    transform = rng.integers(1, 3, n).astype(np.int32)
    lo_f, hi_f = f32(1.0 - AUGMENT_DELTA), f32(1.0 + AUGMENT_DELTA)
    factor = lo_f + rng.random((n, 3), dtype=f32) * (hi_f - lo_f)
    return {"scale": scale, "u_y": u_y, "u_x": u_x, "method": method, "augment": np.where(augmented, transform, 0).astype(np.int32),
            "factor": factor}


def plan_frames(src_h, src_w, out_size: Sequence[int], scale, u_y, u_x) -> Dict[str, np.ndarray]:
    """resize_and_pad(do_random_scale=True)'s size and offset arithmetic (utils/model_utils.py:869-899), in float32 like the
    graph: resized size (scaled_h, scaled_w) and crop origin (offset_y, offset_x) of every frame, int32."""
    f32 = np.float32
    Hd, Wd = out_size
    h, w = np.asarray(src_h).astype(f32), np.asarray(src_w).astype(f32)
    s = np.asarray(scale, dtype=f32)
    scaled_y = (s * f32(Hd)).astype(np.int32)
    scaled_x = (s * f32(Wd)).astype(np.int32)
    image_scale = np.minimum(scaled_x.astype(f32) / w, scaled_y.astype(f32) / h)
    image_scale = np.maximum(image_scale, f32(64.0) / np.minimum(h, w))  # no side below 64 pixels (:886-888)
    sh = (h * image_scale).astype(np.int32)
    sw = (w * image_scale).astype(np.int32)
    oy = (np.maximum(f32(0.0), (sh - Hd).astype(f32)) * np.asarray(u_y, dtype=f32)).astype(np.int32)
    ox = (np.maximum(f32(0.0), (sw - Wd).astype(f32)) * np.asarray(u_x, dtype=f32)).astype(np.int32)
    return {"scaled_h": sh, "scaled_w": sw, "offset_y": oy, "offset_x": ox}


# ---------------------------------------------------------------------------------------------------------------------------
# input_fn_builder (model/dataloader.py:129-278), training input
# ---------------------------------------------------------------------------------------------------------------------------
def train_files(data_cfg: dict) -> List[str]:
    """data.train_file: comma-separated globs, sorted (NeatConfig's expansion, utils/neat_config.py:72-97)."""
    if "train_file_expanded" in data_cfg:
        return list(data_cfg["train_file_expanded"])
    return [f for pat in str(data_cfg.get("train_file", "")).split(",") for f in sorted(glob.glob(pat))]


def shard_files(files: Sequence[str], rank: int, world: int) -> List[str]:
    """Multi-host rule (:163-167): every rank reads its own fixed subset, file i going to rank i % world."""
    if world > 1:
        if len(files) < world:
            raise ValueError(f"{len(files)} training files cannot be sharded over {world} ranks: need at least one per rank")
        return list(files[rank::world])
    return list(files)


class InputPipeline:
    """Iterator of training batches in the feature dict model_fn takes (images [b*n, H, W, 3] bf16, input_ids [b, n, L],
    video_src_ids, shuffled_idx_img, plus youtube_id, chunk_num, mean_time and is_eoc), on `device`.

    A background thread reads and shuffles records, parses them and hands the JPEGs to a pool of `num_threads` decoders; it
    packs a batch's frames into one pinned staging buffer, copies it to the device and runs K14 and `process_example` on a
    data stream of its own.  Up to two prepared batches wait in a queue, so batch k+1 is prepared while step k runs; the
    consumer's stream waits on the batch's event (no host synchronisation).  `close()` stops and joins the thread.
    `last_info` holds the records and draws behind the batch returned last (tests, debugging)."""

    def __init__(self, config, files: Sequence[str], batch_size: int, rank: int = 0, seed: int = 0, device=None, prefetch: int = 2):
        self.data_cfg, self.model_cfg = dict(config.data), dict(config.model)
        self.files = list(files)
        self.batch_size = batch_size
        self.num_chunks = self.data_cfg.get("num_chunks", self.model_cfg.get("num_chunks_in_group", 4))
        self.chunk_text_len = self.data_cfg.get("chunk_text_len", 32)
        self.out_size = tuple(self.model_cfg["image_size"])
        num_threads = self.data_cfg.get("num_threads", 64)
        self.cycle_length = min(num_threads, len(self.files))
        self.shuffle_buffer_size = self.data_cfg.get("shuffle_buffer_size", 256)
        self.device = torch.device(device if device is not None else torch.cuda.current_device())
        self.rng = np.random.default_rng([seed, rank])
        self.last_info = None
        self._queue = queue.Queue(maxsize=prefetch)
        self._stop = threading.Event()
        self._pool = ThreadPoolExecutor(max_workers=num_threads, thread_name_prefix="merlot-jpeg")
        self._stream = torch.cuda.Stream(self.device)
        self._thread = threading.Thread(target=self._run, name="merlot-input", daemon=True)
        self._thread.start()

    # -- record stream: list_files -> repeat -> parallel_interleave(cycle_length) -> shuffle (:153-184) --
    def _file_names(self):
        while True:
            yield from (self.files[i] for i in self.rng.permutation(len(self.files)))

    def _records(self):
        names = self._file_names()
        readers = collections.deque(read_records(next(names)) for _ in range(self.cycle_length))
        ended_in_a_row = 0
        while not self._stop.is_set():
            r = readers.popleft()
            try:
                rec = next(r)
            except StopIteration:
                ended_in_a_row += 1
                if ended_in_a_row > len(self.files) + self.cycle_length:
                    raise ValueError(f"no records in {self.files}")
                readers.append(read_records(next(names)))
                continue
            ended_in_a_row = 0
            readers.append(r)
            yield rec

    def _shuffled(self):
        buf, size = [], self.shuffle_buffer_size
        for rec in self._records():
            if len(buf) < size:
                buf.append(rec)
                continue
            i = int(self.rng.integers(size))
            buf[i], rec = rec, buf[i]
            yield rec
        yield from buf  # only reached when stopping

    # -- one batch --
    def _batch(self, records):
        b, n = self.batch_size, self.num_chunks
        Hd, Wd = self.out_size
        examples = [parse_example(r) for r in records]
        decodes = [self._pool.submit(decode_jpeg, jpg) for ex in examples for jpg in frame_bytes(ex, n)]
        do_clean = self.rng.random(b) < self.data_cfg.get("clean_asr_prob", 0.5)  # sample_bernoulli, one per example (:101-102)
        text = [parse_text(ex, n, self.chunk_text_len, bool(c)) for ex, c in zip(examples, do_clean)]
        draws = frame_draws(self.rng, b * n, self.data_cfg)
        process_seed = int(self.rng.integers(1 << 62))
        frames = [d.result() for d in decodes]
        sizes = np.array([f.size for f in frames], dtype=np.int64)
        offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]])
        staging = torch.empty(int(sizes.sum()), dtype=torch.uint8, pin_memory=True)
        host = staging.numpy()
        for f, o, s in zip(frames, offsets, sizes):
            host[o:o + s] = f.reshape(-1)
        hw = np.array([f.shape[:2] for f in frames], dtype=np.int64)
        plan = plan_frames(hw[:, 0], hw[:, 1], self.out_size, draws["scale"], draws["u_y"], draws["u_x"])
        plan.update(src_offset=offsets, src_h=hw[:, 0], src_w=hw[:, 1], method=draws["method"], augment=draws["augment"],
                    factor=draws["factor"])

        from . import ops
        dev = self.device
        src = staging.to(dev, non_blocking=True)
        images = ops.frames_prepare(src, plan, Hd, Wd)
        feats = {k: torch.from_numpy(np.stack([t[k] for t in text])).pin_memory().to(dev, non_blocking=True) for k in text[0]}
        feats["images"] = images.view(b, n, Hd, Wd, 3)
        g = self.model_cfg.get("num_chunks_in_group", n)
        pdraws = make_draws(b, n, g, self.model_cfg.get("image_shuffle_prob", 0.5), process_seed, dev)
        feats = process_example(feats, self.data_cfg, self.model_cfg, is_training=True, draws=pdraws)
        info = {"records": list(records), "do_clean": do_clean, "frame_draws": draws, "plan": plan,
                "process_draws": {k: v.cpu() for k, v in pdraws.items()}}
        return feats, info

    def _run(self):
        try:
            with torch.cuda.device(self.device), torch.cuda.stream(self._stream):
                recs = self._shuffled()
                while not self._stop.is_set():
                    records = [next(recs) for _ in range(self.batch_size)]  # batch(drop_remainder=True) of a repeated stream
                    feats, info = self._batch(records)
                    ev = torch.cuda.Event()
                    ev.record(self._stream)
                    if not self._put((feats, ev, info)):
                        return
        except BaseException as e:  # handed to the consumer, raised by __next__
            self._put(e)

    def _put(self, item) -> bool:
        while not self._stop.is_set():
            try:
                self._queue.put(item, timeout=0.1)
                return True
            except queue.Full:
                pass
        return False

    def __iter__(self):
        return self

    def __next__(self) -> Dict[str, torch.Tensor]:
        if self._stop.is_set():
            raise StopIteration
        item = self._queue.get()
        if isinstance(item, BaseException):
            raise item
        feats, ev, self.last_info = item
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ev)
        for t in feats.values():
            t.record_stream(cur)  # the data stream's allocations stay alive until the consumer's use of them is done
        return feats

    def close(self):
        self._stop.set()
        while self._thread.is_alive():
            try:
                self._queue.get(timeout=0.1)
            except queue.Empty:
                pass
        self._thread.join()
        self._pool.shutdown(wait=True, cancel_futures=True)
        self._stream.synchronize()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def input_fn_builder(config, is_training: bool = True, rank: int = 0, world: int = 1, seed: int = 0,
                     batch_size: Optional[int] = None, device=None) -> InputPipeline:
    """model/dataloader.py:129-278 for training: the files of data.train_file (sharded by rank when world > 1), interleaved
    over min(num_threads, files) readers, a shuffle buffer of shuffle_buffer_size records, the parser, batches of
    `batch_size` (default device.train_batch_size // world) with drop_remainder, and `process_example`.  Returns the
    running pipeline (an iterator of feature dicts; close() it)."""
    if not is_training:
        raise NotImplementedError("only the training input is provided (val_file / eval input is not)")
    if config.data.get("unbatch_size", 1) > 1:
        raise NotImplementedError("data.unbatch_size > 1 is not provided")
    files = train_files(config.data)
    if not files:
        raise ValueError(f"data.train_file {config.data.get('train_file')!r} matches no file")
    files = shard_files(files, rank, world)
    if batch_size is None:
        batch_size = max(1, config.device.get("train_batch_size", 8) // world)
    return InputPipeline(config, files, batch_size, rank=rank, seed=seed, device=device)
