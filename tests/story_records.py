"""TEST INFRASTRUCTURE ONLY: sort_story records (downstream/sort_story/dataloader.py:15-31's keys) built from a seed with
tests/tfrecord_writer.py, and a NumPy restatement of their text parse and of the evaluation resize plan."""
import os
import sys

import numpy as np

from tests import tfrecord_writer as W

F = np.float32
# (h, w) of the frames: portrait, landscape, square, very wide and tall; every one resizes to >= 1 pixel at 32 x 48
SIZES = [(37, 53), (61, 29), (48, 48), (20, 90), (90, 20), (33, 47), (64, 96)]


def story(rng, story_id, max_sentence=40, sizes=SIZES, gray_frame=1, vocab=1000, pie=None, drop_sentence=None):
    """One story as plain values: five JPEG frames (frame `gray_frame` grayscale), five sentences of 0..max_sentence ids."""
    frames = [W.jpeg(rng, *sizes[(story_id + i) % len(sizes)], gray=(i == gray_frame)) for i in range(5)]
    sents = [rng.integers(7, vocab, int(rng.integers(0, max_sentence))).tolist() for _ in range(5)]
    if drop_sentence is not None:
        sents[drop_sentence] = None
    return {"story_id": story_id, "permutation_identity_encode": int(rng.integers(0, 120)) if pie is None else pie,
            "frames": frames, "sentences": sents}


def story_example(s, with_ids=True) -> bytes:
    feats = {}
    if with_ids:
        feats["story_id"] = ("int64", [s["story_id"]])
        feats["permutation_identity_encode"] = ("int64", [s["permutation_identity_encode"]])
    for i, ids in enumerate(s["sentences"]):
        if ids is not None:
            feats[f"sentence/sentence_{i}"] = ("int64", ids, i % 2 == 0)
    for i, jpg in enumerate(s["frames"]):
        if jpg is not None:
            feats[f"image/image_{i}_encoded"] = ("bytes", [jpg])
            feats[f"image/image_{i}_format"] = ("bytes", [b"jpeg"])
            feats[f"image/image_{i}_sha256"] = ("bytes", [b"0" * 64])
    return W.example(feats)


def write_stories(dirpath, counts, seed=0, **kw):
    """Files val-000.tfrecord, ... holding counts[k] stories each; story ids run 0, 1, ... file by file.  Returns the stories."""
    rng = np.random.default_rng(seed)
    out, sid = [], 0
    for k, n in enumerate(counts):
        recs = []
        for _ in range(n):
            s = story(rng, sid, **kw)
            out.append(s)
            recs.append(story_example(s))
            sid += 1
        W.write_records(dirpath / f"val-{k:03d}.tfrecord", recs)
    return out


def sentences_np(sents):
    """[START] + ids, int32, truncated to 32, padded with 0 (an absent sentence is [START])."""
    out = np.zeros((5, 32), np.int32)
    for i, ids in enumerate(sents):
        row = [2] + list(ids or [])
        row = np.asarray(row, np.int64).astype(np.int32)[:32]
        out[i, :len(row)] = row
    return out


def eval_plan(h, w, desired):
    """resize_and_pad's else-branch (utils/model_utils.py:900-907) for one frame, float32 scalars."""
    Hd, Wd = desired
    image_scale = min(F(Hd) / F(h), F(Wd) / F(w))
    return int(F(h) * image_scale), int(F(w) * image_scale), 0, 0


def five_segments_model():
    """merlot_5segments.yaml's model section: merlot.yaml sizes, 5 segments per story, 384x384 frames, the hybrid stem."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import bench
    return dict(bench.load_config().model, num_chunks_in_group=5, image_size=[384, 384], resnet_layers=[3, 4, 9],
                image_shuffle_prob=0.5, contrast_coef=0.5)
