"""Zero-shot story unshuffling (downstream/sort_story): story records in, per-story temporal probabilities and the paper's
three metrics out.  `python -m merlot_b200.sort_story <yaml> [--out logits_val.h5|.npz]` is the role of both reference
scripts, get_zero_shot_logits.py and score_permutations.py.

  * records    -- `parse_story` (dataloader.py:15-109: story_id, permutation_identity_encode, five sentences, five JPEGs),
                  `plan_frames_eval` (resize_and_pad's do_random_scale=False branch), `input_fn_builder` (files in sorted
                  order, interleaved, batch(drop_remainder=True)); the pixels go through K14 (bilinear, no augmentation).
  * forward    -- `zero_shot_predict`: get_zero_shot_logits.py:36-90 on MerlotModel, each story tiled `duplication_factor`
                  times in story-major order with a fixed shuffle per copy; the copies share one ViT pass (frame_copies)
                  and `temporal_probs` averages each story over its own copies (DESIGN.md 2 states why this differs from
                  the reference's tf.tile layout).
  * scoring    -- score_permutations.py:15-80: every assignment of images to sentences, best permutation per story, the
                  three means; plain NumPy, tested bit for bit against a loop restatement.
"""
from __future__ import annotations

import argparse
import itertools
import os
import re
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from .dataloader import (DEFAULT_NUM_THREADS, DevicePipeline, decode_jpeg, eval_decode_threads, interleave_records,
                         plan_frames_eval, stage_frames)
from .tfrecord import parse_example

NUM_CHUNKS = 5       # get_zero_shot_logits.py:26-28: five sentences and five frames per story
MAX_NUM_TOKENS = 32  # dataloader.py:75
START, PADDING = 2, 0  # utils/encode/encoder.py


def temporal_probs(model, duplication_factor: int = 1, scope_name: str = "lang_viz_temporal"):
    """get_zero_shot_logits.py:68-86 for one modality pair: [batch, n, n, 3] probabilities of (equal, before, after)."""
    import torch
    n, H = model.num_chunks_in_group, model.hidden_size
    h_lang = model.encoder_hidden_states["lang"].reshape(model.B, n, model.lang_chunk_length, H)[:, :, 0]
    h_viz = model.encoder_hidden_states["viz"].reshape(model.B, n, model.viz_chunk_length, H)[:, :, 0]
    xa, xb = (h_lang, h_viz) if scope_name == "lang_viz_temporal" else (h_viz, h_viz)
    logits = model.allpairs_temporal_logits(xa=xa, xb=xb, scope_name=scope_name)
    probs = torch.softmax(logits.float(), -1)[:, 1:]
    return probs.reshape(model.B // duplication_factor, duplication_factor, n, n, 3).mean(1)


def permutation_scores(probs: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """score_permutations.py:15-29,57-62 for all permutations at once.  probs [n, n, 3]; sentence i keeps position i, image j is
    assigned position perm[j]; a pair contributes log P(eq) if i == perm[j], log P(before) if i < perm[j], log P(after) otherwise.
    Returns (perms [n!, n] in itertools order, scores [n!])."""
    probs = np.asarray(probs, dtype=np.float64)
    n = probs.shape[0]
    if probs.shape != (n, n, 3):
        raise ValueError(f"probs must be [n, n, 3], got {probs.shape}")
    perms = np.array(list(itertools.permutations(range(n))), dtype=np.int64)  # [n!, n]
    i = np.arange(n)[None, :, None]                                            # sentence positions
    pj = perms[:, None, :]                                                     # image positions under each permutation
    cls = np.where(i == pj, 0, np.where(i < pj, 1, 2))                         # [n!, n, n]
    lp = np.log(probs)
    picked = np.take_along_axis(np.broadcast_to(lp[None], (len(perms), n, n, 3)), cls[..., None], axis=-1)[..., 0]
    return perms, picked.sum((1, 2))


def best_permutation(probs: np.ndarray) -> Tuple[Tuple[int, ...], float]:
    """The permutation the reference keeps (:64): highest score, first in itertools order among ties (stable sort)."""
    perms, scores = permutation_scores(probs)
    k = int(np.argmax(scores))
    return tuple(int(v) for v in perms[k]), float(scores[k])


def spearman_acc(story: Sequence[int]) -> float:  # :32-33 (scipy.stats.spearmanr against the identity; no ties in a permutation)
    s = np.asarray(story, dtype=np.float64)
    n = len(s)
    d = s - np.arange(n)
    return float(1.0 - 6.0 * np.sum(d * d) / (n * (n * n - 1)))


def absolute_distance(story: Sequence[int]) -> float:  # :35-36
    s = np.asarray(story, dtype=np.float64)
    return float(np.mean(np.abs(s - np.arange(len(s)))))


def pairwise_acc(story: Sequence[int]) -> float:  # :39-46
    n = len(story)
    correct = sum(1 for a in range(n) for b in range(a + 1, n) if story[a] < story[b])
    return correct / (n * (n - 1) // 2)


def evaluate(all_probs: Iterable[np.ndarray]) -> Dict[str, float]:
    """score_permutations.py:54-80: best permutation per story, then the three means the script prints."""
    stories: List[Tuple[int, ...]] = [best_permutation(p)[0] for p in all_probs]
    return {"spearman": float(np.mean([spearman_acc(s) for s in stories])),
            "absolute_distance": float(np.mean([absolute_distance(s) for s in stories])),
            "pairwise": float(np.mean([pairwise_acc(s) for s in stories])), "stories": stories}


def write_logits_h5(path: str, predictions: Iterable[Dict], include_images: bool = True) -> int:
    """The writer loop of get_zero_shot_logits.py:105-119: one HDF5 group per story id with `permutation_identity_encode`,
    optional uint8 `images` (255 * image), `sentences`, and `{lang_viz,viz_viz}_probs`; a story id seen twice is skipped like the
    reference's `except ValueError: continue`.  `predictions` yields per-story dicts (what estimator.predict yields there; here
    e.g. {'story_id': id, 'lang_viz_probs': temporal_probs(model)[i].cpu().numpy(), ...}).  Returns the number of groups written.
    Needs h5py (not part of this image: raises ImportError with that message instead of writing another format silently)."""
    try:
        import h5py
    except ImportError as e:  # pragma: no cover - depends on the environment
        raise ImportError("write_logits_h5 needs h5py (downstream/sort_story/get_zero_shot_logits.py:105 writes HDF5); "
                          "use write_logits_npz for an h5py-free container with the same keys") from e
    n = 0
    with h5py.File(path, "w") as h5:
        for x in predictions:
            key = str(x["story_id"])
            if key in h5:
                continue
            grp = h5.create_group(key)
            grp.create_dataset("permutation_identity_encode", data=np.asarray(x["permutation_identity_encode"]))
            if include_images and "images" in x:
                grp.create_dataset("images", data=(255 * np.asarray(x["images"], dtype=np.float32)).astype(np.uint8))
            grp.create_dataset("sentences", data=np.asarray(x["sentences"]))
            for modality_name in ("lang_viz", "viz_viz"):
                grp.create_dataset(f"{modality_name}_probs", data=np.asarray(x[f"{modality_name}_probs"]))
            n += 1
    return n


def write_logits_npz(path: str, predictions: Iterable[Dict], include_images: bool = False) -> int:
    """Same records as write_logits_h5 in a NumPy .npz (keys `<story_id>/<dataset>`), for environments without h5py;
    read_logits_npz gives back {story_id: {dataset: array}} -- the structure score_permutations.py walks (:77-87)."""
    out, seen = {}, set()
    for x in predictions:
        key = str(x["story_id"])
        if key in seen:
            continue
        seen.add(key)
        out[f"{key}/permutation_identity_encode"] = np.asarray(x["permutation_identity_encode"])
        if include_images and "images" in x:
            out[f"{key}/images"] = (255 * np.asarray(x["images"], dtype=np.float32)).astype(np.uint8)
        out[f"{key}/sentences"] = np.asarray(x["sentences"])
        for modality_name in ("lang_viz", "viz_viz"):
            out[f"{key}/{modality_name}_probs"] = np.asarray(x[f"{modality_name}_probs"])
    np.savez_compressed(path, **out)
    return len(seen)


def read_logits_npz(path: str) -> Dict[str, Dict[str, np.ndarray]]:
    res: Dict[str, Dict[str, np.ndarray]] = {}
    with np.load(path) as z:
        for k in z.files:
            sid, name = k.split("/", 1)
            res.setdefault(sid, {})[name] = z[k]
    return res


def fixed_shuffle_index(batch_size: int, num_chunks: int, seed: int = 1234) -> np.ndarray:
    """The evaluation-time frame order of get_zero_shot_logits.py:55-56: argsort of a FIXED uniform draw per story, + 64 (the
    'hard' index range of temporal_loss, model/modeling.py:635).  The reference draws with tf.random.stateless_uniform(seed=
    [123, 1234]); that generator cannot be reproduced without TensorFlow, so the order differs from the reference's but is
    equally fixed (stated in INTEGRATION.md)."""
    rng = np.random.RandomState(seed)
    return (np.argsort(rng.uniform(size=(batch_size, num_chunks)), 1).astype(np.int32) + 64)


# ---------------------------------------------------------------------------------------------------------------------------
# story records (downstream/sort_story/dataloader.py)
# ---------------------------------------------------------------------------------------------------------------------------
def _scalar_int(example, key: str, default: int = -1) -> int:
    v = example.get(key)
    if v is None or len(v) == 0:
        return default
    if len(v) != 1:
        raise ValueError(f"story feature {key!r} has {len(v)} values, expected 1")
    return int(v[0])


def parse_story(example, num_chunks: int = NUM_CHUNKS) -> Dict:
    """One parsed story record (dataloader.py:15-109) without its pixels: story_id and permutation_identity_encode (int64
    scalars, default -1), sentences [num_chunks, 32] int32 -- [START] + sentence/sentence_{i}, truncated to 32 and padded
    with PADDING (an absent sentence is [START] alone) -- and frames, the encoded image/image_{i}_encoded (b'' if absent)."""
    sents = np.full((num_chunks, MAX_NUM_TOKENS), PADDING, dtype=np.int32)
    for i in range(num_chunks):
        toks = np.concatenate([[START], np.asarray(example.get(f"sentence/sentence_{i}", []), dtype=np.int64)])
        toks = toks.astype(np.int32)[:MAX_NUM_TOKENS]  # tf.cast(int64 -> int32), then pad_to_fixed_size(truncate=True)
        sents[i, :len(toks)] = toks
    frames = []
    for i in range(num_chunks):
        v = example.get(f"image/image_{i}_encoded")
        frames.append(bytes(v[0]) if v else b"")
    return {"story_id": _scalar_int(example, "story_id"),
            "permutation_identity_encode": _scalar_int(example, "permutation_identity_encode"),
            "sentences": sents, "frames": frames}


def decode_frame(story: Dict, i: int) -> np.ndarray:
    """Frame i of a parsed story as uint8 [h, w, 3] RGB; a missing or undecodable image raises ValueError naming the story."""
    buf = story["frames"][i]
    if not buf:
        raise ValueError(f"story {story['story_id']}: image {i} is missing")
    try:
        return decode_jpeg(buf)
    except Exception as e:
        raise ValueError(f"story {story['story_id']}: image {i} cannot be decoded ({type(e).__name__}: {e})") from e


def eval_frame_plan(hw: np.ndarray, story_ids: Sequence[int], out_size: Sequence[int]) -> Dict[str, np.ndarray]:
    """The K14 plan of a batch's frames ([n, 2] heights and widths, story by story): plan_frames_eval, bilinear, no
    augmentation.  A frame whose resized side truncates to 0 raises (TensorFlow's resize fails there too), naming the story."""
    plan = plan_frames_eval(hw[:, 0], hw[:, 1], out_size)
    bad = np.flatnonzero((plan["scaled_h"] < 1) | (plan["scaled_w"] < 1))
    if len(bad):
        k = int(bad[0])
        raise ValueError(f"story {story_ids[k // NUM_CHUNKS]}: image {k % NUM_CHUNKS} of {hw[k, 0]}x{hw[k, 1]} pixels resizes to "
                         f"{plan['scaled_h'][k]}x{plan['scaled_w'][k]} for image_size {list(out_size)}")
    n = len(hw)
    plan.update(src_h=hw[:, 0], src_w=hw[:, 1], method=np.zeros(n, np.int32), augment=np.zeros(n, np.int32),
                factor=np.ones((n, 3), np.float32))
    return plan


def batch_records(records: Iterable, batch_size: int, tail: List):
    """batch(batch_size, drop_remainder=True): lists of batch_size records in order; a last partial batch goes to `tail`."""
    batch = []
    for r in records:
        batch.append(r)
        if len(batch) == batch_size:
            yield batch
            batch = []
    tail.extend(batch)


def eval_batches(files: Sequence[str], cycle_length: int, batch_size: int, tail: List, stop=None, rank: int = 0,
                 world: int = 1):
    """The evaluation record stream -- `files` in order, interleave_records over cycle_length readers, batch_records with
    drop_remainder -- as rank `rank` of `world` sees it: the global batches k with k % world == rank, in order.  The set of
    batches and their composition do not depend on `world`.  Every rank walks the whole stream to find the batch boundaries,
    but reads another rank's records by their headers only (read_records' skip path): their data is never checksummed,
    parsed or decoded here.  A last partial batch goes to `tail` (None in place of another rank's records), so len(tail) is
    the global count of dropped records on every rank."""
    if world == 1:
        yield from batch_records(interleave_records(iter(files), cycle_length, files, stop), batch_size, tail)
        return
    recs = interleave_records(iter(files), cycle_length, files, stop, keep=lambda i: (i // batch_size) % world == rank)
    for k, records in enumerate(batch_records(recs, batch_size, tail)):
        if k % world == rank:
            yield records


def val_files(config) -> List[str]:
    """data.val_file: comma-separated globs, each sorted (list_files(shuffle=False))."""
    if "val_file_expanded" in config.data:
        return list(config.data["val_file_expanded"])
    import glob
    return [f for pat in str(config.data.get("val_file", "")).split(",") if pat for f in sorted(glob.glob(pat))]


class StoryPipeline(DevicePipeline):
    """Iterator of evaluation batches {images [b*5, H, W, 3] bf16, sentences [b, 5, 32] int32 (both on `device`), story_id
    [b] and permutation_identity_encode [b] (int64 NumPy)} over the records of `files` in deterministic order: the files in
    the given order, interleaved over min(num_threads, files) readers, no shuffle, no repeat.  A last partial batch is not
    returned; after the iteration ends `dropped` is the number of records it held.  As rank `rank` of `world` evaluation
    processes it returns the batches k with k % world == rank (eval_batches); `dropped` stays the global count."""

    def __init__(self, config, files: Sequence[str], batch_size: int, device=None, prefetch: int = 2, rank: int = 0,
                 world: int = 1):
        self.files = list(files)
        self.batch_size = batch_size
        self.rank, self.world = rank, world
        self.out_size = tuple(config.model["image_size"])
        num_threads = config.data.get("num_threads", DEFAULT_NUM_THREADS)
        self.cycle_length = min(num_threads, len(self.files))
        self.dropped = None
        super().__init__(device, eval_decode_threads(config.data), prefetch)

    def _batch(self, records):
        from . import ops
        import torch
        stories = [parse_story(parse_example(r)) for r in records]
        decodes = [self._pool.submit(decode_frame, s, i) for s in stories for i in range(NUM_CHUNKS)]
        staging, offsets, hw = stage_frames([d.result() for d in decodes])
        ids = [s["story_id"] for s in stories]
        plan = eval_frame_plan(hw, ids, self.out_size)
        plan["src_offset"] = offsets
        images = ops.frames_prepare(staging.to(self.device, non_blocking=True), plan, *self.out_size)
        sents = torch.from_numpy(np.stack([s["sentences"] for s in stories])).pin_memory().to(self.device, non_blocking=True)
        feats = {"images": images, "sentences": sents, "story_id": np.array(ids, dtype=np.int64),
                 "permutation_identity_encode": np.array([s["permutation_identity_encode"] for s in stories], dtype=np.int64)}
        return feats, {"records": list(records), "plan": plan}

    def _produce(self):
        tail = []
        for records in eval_batches(self.files, self.cycle_length, self.batch_size, tail, self._stop, self.rank, self.world):
            yield self._batch(records)
        self.dropped = len(tail)


def input_fn_builder(config, batch_size: Optional[int] = None, device=None, rank: int = 0, world: int = 1) -> StoryPipeline:
    """dataloader.py:111-170 with is_training=False: the story records of data.val_file, batches of `batch_size` (default
    device.val_batch_size, 16 if unset) with drop_remainder; rank `rank` of `world` gets the batches k with
    k % world == rank.  Returns the running pipeline (an iterator; close() it)."""
    if config.model.get("num_chunks_in_group", NUM_CHUNKS) != NUM_CHUNKS:  # get_zero_shot_logits.py:28
        raise ValueError(f"zero-shot story unshuffling needs model.num_chunks_in_group == {NUM_CHUNKS}, "
                         f"got {config.model.get('num_chunks_in_group')}")
    files = val_files(config)
    if not files:
        raise ValueError(f"data.val_file {config.data.get('val_file')!r} matches no file")
    if batch_size is None:
        batch_size = config.device.get("val_batch_size", 16)
    return StoryPipeline(config, files, batch_size, device=device, rank=rank, world=world)


# ---------------------------------------------------------------------------------------------------------------------------
# zero-shot forward (get_zero_shot_logits.py:36-90)
# ---------------------------------------------------------------------------------------------------------------------------
def tiled_inputs(sentences, duplication_factor: int, seed: int = 1234):
    """The text inputs of `duplication_factor` copies of every story in story-major order -- row s*dup + d is copy d of story
    s -- and their fixed frame orders: (input_ids [b*dup, 5, 32], shuffled_idx_img [b*dup*5] int32 = fixed_shuffle_index
    of b*dup rows), on the device of `sentences`."""
    import torch
    b = sentences.shape[0]
    ids = sentences[:, :, :MAX_NUM_TOKENS].repeat_interleave(duplication_factor, 0).contiguous()
    shuf = torch.from_numpy(fixed_shuffle_index(b * duplication_factor, NUM_CHUNKS, seed).reshape(-1)).to(sentences.device)
    return ids, shuf


def zero_shot_predict(config, store, batch: Dict, duplication_factor: int = 2, seed: int = 1234) -> Dict:
    """Per-story lang_viz_probs and viz_viz_probs [b, 5, 5, 3] (fp32 CUDA tensors) of one StoryPipeline batch: MerlotModel in
    eval mode without masking on `duplication_factor` story-major copies of every story (tiled_inputs), the frames of a
    story passed through the ViT once (frame_copies), then `temporal_probs` per modality pair.  Also returns the batch's
    untiled sentences, story_id and permutation_identity_encode."""
    from .modeling import MerlotModel
    ids, shuf = tiled_inputs(batch["sentences"], duplication_factor, seed)
    model = MerlotModel(config.model, is_training=False, use_tpu=False, image=batch["images"], input_ids=ids, mask_input=False,
                        shuffled_idx_img=shuf, params=store, log_attention_probs=False, frame_copies=duplication_factor)
    out = {f"{name}_probs": temporal_probs(model, duplication_factor, f"{name}_temporal") for name in ("lang_viz", "viz_viz")}
    out.update(sentences=batch["sentences"], story_id=batch["story_id"],
               permutation_identity_encode=batch["permutation_identity_encode"])
    return out


def zero_shot_variables(store) -> List[str]:
    """The entries the zero-shot forward reads: everything but the language-only embeddings and encoder (share_params:
    False), the pretraining heads and the encoder layers beyond the joint encoder's depth."""
    joint = store.cfg["num_hidden_layers"]

    def read(name):
        if name.startswith(("langonly_embeddings/", "langonly_encoder/", "lm_head/", "contrastive/")):
            return False
        m = re.match(r"encoder/layer(\d+)/", name)
        return m is None or int(m.group(1)) < joint
    return [n for n in store.entries if read(n)]


def restore_for_zero_shot(config, prefix: str, device="cuda"):
    """A ParamStore without optimizer slots, restored by name from the checkpoint `prefix`.  Raises if a variable the
    zero-shot forward reads is not in the checkpoint (scoring with initial weights would be meaningless)."""
    from .params import ParamStore
    store = ParamStore(config.model, device=device, with_optimizer_state=False)
    missing = set(store.load_checkpoint(prefix))
    need = [n for n in zero_shot_variables(store) if n in missing]
    if need:
        raise ValueError(f"{prefix}: {len(need)} variables the zero-shot forward reads are not in the checkpoint: "
                         + ", ".join(need))
    return store


# ---------------------------------------------------------------------------------------------------------------------------
# files and driver (get_zero_shot_logits.py:92-119, score_permutations.py:50-80)
# ---------------------------------------------------------------------------------------------------------------------------
def read_logits_h5(path: str) -> Dict[str, Dict[str, np.ndarray]]:
    import h5py
    with h5py.File(path, "r") as h5:
        return {k: {n: np.array(v) for n, v in h5[k].items()} for k in h5.keys()}


def score_file(path: str) -> Dict:
    """score_permutations.py:50-80 on an existing logits file (.h5 or .npz): lang_viz_probs of every story in sorted integer
    story_id order, then `evaluate`."""
    groups = read_logits_h5(path) if path.endswith(".h5") else read_logits_npz(path)
    keys = sorted(int(k) for k in groups)
    return evaluate([groups[str(k)]["lang_viz_probs"] for k in keys])


def _story_rows(pred: Dict):
    probs = {k: pred[k].cpu().numpy() for k in ("lang_viz_probs", "viz_viz_probs")}
    sents = pred["sentences"].cpu().numpy()
    for i, sid in enumerate(pred["story_id"]):
        yield {"story_id": int(sid), "permutation_identity_encode": pred["permutation_identity_encode"][i],
               "sentences": sents[i], "lang_viz_probs": probs["lang_viz_probs"][i], "viz_viz_probs": probs["viz_viz_probs"][i]}


def gather_story_rows(config, prefix: str, group, seed: int = 1234) -> Tuple[List[List[Dict]], int]:
    """Every rank of `group` restores `prefix` (restore_for_zero_shot) and runs zero_shot_predict on its batches
    (input_fn_builder with the group's rank and world).  Returns, on every rank, the _story_rows of every batch in global
    batch order and the number of records dropped.  A failure on any rank raises RankFailure on every rank."""
    import torch

    def own():
        store = restore_for_zero_shot(config, prefix)
        rows = []
        with torch.no_grad(), input_fn_builder(config, rank=group.rank, world=group.world) as pipe:
            for batch in pipe:
                rows.append(list(_story_rows(zero_shot_predict(config, store, batch, seed=seed))))
            return rows, pipe.dropped
    from .eval_ranks import in_batch_order
    per_rank = group.run_and_gather(own)
    return in_batch_order([rows for rows, _ in per_rank]), per_rank[0][1]


def main(argv=None) -> Dict:
    """`python -m merlot_b200.sort_story <yaml> [--out logits_val.h5|.npz]`: the story records of $SORTSTORY_PATH (or
    data.val_file when it is unset), the latest checkpoint of device.output_dir restored by name, one group per story
    written to --out, then the number of stories scored and dropped and score_permutations.py's three metrics.  Returns
    the metrics.

    Under torchrun with WORLD_SIZE > 1 every rank scores its share of the batches (eval_batches) from the checkpoint rank 0
    chose, and rank 0 writes the stories in the order one process writes them, prints and scores; every rank returns the
    metrics."""
    import torch
    from .config import NeatConfig
    from .eval_ranks import eval_group
    from .tf_checkpoint import latest_checkpoint
    ap = argparse.ArgumentParser(description="Zero-shot story unshuffling: temporal probabilities of every story and scores")
    ap.add_argument("config_file")
    ap.add_argument("--out", default="logits_val.h5", help="output file: .h5 (needs h5py) or .npz")
    ap.add_argument("--seed", type=int, default=1234, help="seed of the fixed frame orders (fixed_shuffle_index)")
    args = ap.parse_args(argv)
    if args.out.endswith(".h5"):
        try:
            import h5py  # noqa: F401
        except ImportError as e:
            raise ImportError(f"--out {args.out} writes HDF5 and needs h5py; pass an .npz path instead") from e
        write = write_logits_h5
    elif args.out.endswith(".npz"):
        write = write_logits_npz
    else:
        raise ValueError(f"--out {args.out!r}: the extension must be .h5 or .npz")
    config = NeatConfig.from_yaml(args.config_file)
    if os.environ.get("SORTSTORY_PATH"):  # get_zero_shot_logits.py:24
        config.data["val_file"] = os.environ["SORTSTORY_PATH"]
        config.data.pop("val_file_expanded", None)
    files = val_files(config)
    if not files:
        raise ValueError(f"SORTSTORY_PATH / data.val_file {config.data.get('val_file')!r} matches no file")
    with eval_group() as group:
        # rank 0 picks the checkpoint, so a checkpoint written meanwhile cannot split the ranks
        prefix = group.broadcast(latest_checkpoint(str(config.device["output_dir"])) if group.rank == 0 else None)
        if not prefix:
            raise ValueError(f"device.output_dir {config.device['output_dir']!r} holds no checkpoint")
        if group.world == 1:
            store = restore_for_zero_shot(config, prefix)
            with input_fn_builder(config) as pipe:
                def rows():
                    with torch.no_grad():
                        for batch in pipe:
                            yield from _story_rows(zero_shot_predict(config, store, batch, seed=args.seed))
                n = write(args.out, rows())
                dropped = pipe.dropped
        else:
            batches, dropped = gather_story_rows(config, prefix, group, seed=args.seed)
            n = group.on_rank0(lambda: write(args.out, (row for rows in batches for row in rows)))

        def report():
            print(f"restored {prefix}; scored {n} stories, dropped {dropped} (the last partial batch of "
                  f"{config.device.get('val_batch_size', 16)}); wrote {args.out}", flush=True)
            res = score_file(args.out)
            print("Spearman:", res["spearman"], "Absolute Distance:", res["absolute_distance"], "Pairwise:", res["pairwise"],
                  sep="\n", flush=True)
            return res
        return group.broadcast(group.on_rank0(report))


if __name__ == "__main__":
    main()
