"""TEST INFRASTRUCTURE ONLY: VCR records (the keys of downstream/vcr/dataloader_joint.py:37-71 and dataloader.py:40-65) built
from a seed with tests/tfrecord_writer.py, and a NumPy restatement of both reference parsers' ids, texts and labels
(dataloader_joint.py:132-193, dataloader.py:113-157).  The prompts and END are taken from tests/golden/vcr_prompts.json."""
import json
import os

import numpy as np

from tests import tfrecord_writer as W

MODES = ("answer", "rationale")
PADDING, START, END = 0, 2, 3  # utils/encode/encoder.py
# (h, w) of the images: portrait, landscape, square, very wide and tall, small (below the training plan's 64-pixel floor)
SIZES = [(37, 53), (61, 29), (48, 48), (20, 90), (90, 20), (120, 200), (30, 40)]


def golden():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vcr_prompts.json")) as f:
        return json.load(f)


def prompts():
    enc = golden()["encode"]
    return {"answer": [START] + enc[" answer question:"], "rationale": [START] + enc[" provide rationale:"]}


def question(rng, k, max_ctx=40, max_choice=30, vocab=50000, sizes=SIZES, draws=("segm",)):
    """One question as plain values: per mode an image for every draw of `draws`, a ctx, four choices, their (unused) tags
    and a label in [0, 4).  Set a value to None to leave its feature out of the record."""
    q = {"img_id": f"movie_{k}.jpg", "annot_id": f"val-{k}"}
    for j, mode in enumerate(MODES):
        for d in draws:
            q[f"{mode}/{d}/image"] = W.jpeg(rng, *sizes[(2 * k + j) % len(sizes)], gray=(k % 5 == 4))
        q[f"{mode}/ctx"] = rng.integers(7, vocab, int(rng.integers(0, max_ctx))).tolist()
        q[f"{mode}/ctx_tags"] = rng.integers(-1, 5, len(q[f"{mode}/ctx"])).tolist()
        for i in range(4):
            q[f"{mode}/choice_{i}"] = rng.integers(7, vocab, int(rng.integers(0, max_choice))).tolist()
            q[f"{mode}/choice_tags_{i}"] = rng.integers(-1, 5, len(q[f"{mode}/choice_{i}"])).tolist()
        q[f"label/{mode}_label"] = int(rng.integers(0, 4))
    return q


def vcr_example(q) -> bytes:
    feats = {}
    for key, v in q.items():
        if v is None:
            continue
        if key in ("img_id", "annot_id"):
            feats[key] = ("bytes", [v.encode()])
        elif key.endswith("/image"):
            feats[key + "/encoded"] = ("bytes", [v])
            feats[key + "/format"] = ("bytes", [b"jpeg"])
            feats[key + "/key/sha256"] = ("bytes", [b"0" * 64])
        elif key.startswith("label/"):
            feats[key] = ("int64", [v])
        else:
            feats[key] = ("int64", v, len(v) % 2 == 0)  # packed and unpacked lists
    return W.example(feats)


def write_questions(dirpath, counts, prefix="vcr", seed=0, **kw):
    """Files <prefix>-000.tfrecord, ... holding counts[f] questions each; question k of the run is `question(rng, k)`.
    Returns the questions in write order."""
    rng = np.random.default_rng(seed)
    out = []
    for f, n in enumerate(counts):
        qs = [question(rng, len(out) + i, **kw) for i in range(n)]
        out += qs
        W.write_records(dirpath / f"{prefix}-{f:03d}.tfrecord", [vcr_example(q) for q in qs])
    return out


def texts_np(q, mode, max_tokens):
    """[4, max_tokens] int32: prompt + ctx + choice_i + END, int64 -> int32, truncated, padded with 0."""
    out = np.zeros((4, max_tokens), np.int32)
    for i in range(4):
        row = prompts()[mode] + list(q.get(f"{mode}/ctx") or []) + list(q.get(f"{mode}/choice_{i}") or []) + [END]
        row = np.asarray(row, np.int64).astype(np.int32)[:max_tokens]
        out[i, :len(row)] = row
    return out


def label_np(q, mode):
    v = q.get(f"label/{mode}_label")
    return -1 if v is None else v


def joint_np(q):
    """dataloader_joint.py's lm_input [2, 4, 184] and lm_targets [2] of one question."""
    return np.stack([texts_np(q, m, 184) for m in MODES]), np.array([label_np(q, m) for m in MODES])


def eval_np(q, mode):
    """dataloader.py's lm_input [4, 134 (answer) or 184 (rationale)] and label of one question."""
    return texts_np(q, mode, 134 if mode == "answer" else 184), label_np(q, mode)
