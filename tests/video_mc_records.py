"""TEST INFRASTRUCTURE ONLY: multiple-choice video QA records (the schema of merlot_b200/video_mc_input.py, INTEGRATION.md)
built from a seed with tests/tfrecord_writer.py, and a NumPy restatement of the parser's texts, labels and frame mask."""
import numpy as np

from tests import tfrecord_writer as W

PADDING, START, END = 0, 2, 3  # utils/encode/encoder.py
SIZES = [(37, 53), (61, 29), (48, 48), (20, 90), (90, 20), (120, 200), (30, 40)]


def question(rng, k, num_frames, num_choices, max_question=30, max_choice=20, vocab=1000, sizes=SIZES, frames=None):
    """One question as plain values: 1..num_frames frames (`frames` fixes the count), a question, num_choices choices and
    a label in [0, num_choices).  Set a value to None to leave its feature out of the record."""
    n = int(rng.integers(1, num_frames + 1)) if frames is None else frames
    q = {"id": f"q-{k}",
         "frames": [W.jpeg(rng, *sizes[(3 * k + f) % len(sizes)], gray=(k % 5 == 4 and f == 0)) for f in range(n)],
         "question": rng.integers(7, vocab, int(rng.integers(0, max_question))).tolist(),
         "label": int(rng.integers(0, num_choices))}
    for i in range(num_choices):
        q[f"choice_{i}"] = rng.integers(7, vocab, int(rng.integers(0, max_choice))).tolist()
    return q


def example(q) -> bytes:
    feats = {}
    for key, v in q.items():
        if v is None:
            continue
        if key == "id":
            feats[key] = ("bytes", [v.encode()])
        elif key == "frames":
            feats["frames/encoded"] = ("bytes", list(v))
        elif key == "label":
            feats[key] = ("int64", [v])
        else:
            feats[key] = ("int64", v, len(v) % 2 == 0)  # packed and unpacked lists
    return W.example(feats)


def write_questions(dirpath, counts, num_frames, num_choices, prefix="mc", seed=0, **kw):
    """Files <prefix>-000.tfrecord, ... holding counts[f] questions each; question k of the run is `question(rng, k, ...)`.
    Returns the questions in write order."""
    rng = np.random.default_rng(seed)
    out = []
    for f, n in enumerate(counts):
        qs = [question(rng, len(out) + i, num_frames, num_choices, **kw) for i in range(n)]
        out += qs
        W.write_records(dirpath / f"{prefix}-{f:03d}.tfrecord", [example(q) for q in qs])
    return out


def texts_np(q, num_choices, max_len):
    """[num_choices, max_len] int32: START + question + choice_i + END, int64 -> int32, truncated, padded with 0."""
    out = np.zeros((num_choices, max_len), np.int32)
    for i in range(num_choices):
        row = [START] + list(q.get("question") or []) + list(q[f"choice_{i}"]) + [END]
        row = np.asarray(row, np.int64).astype(np.int32)[:max_len]
        out[i, :len(row)] = row
    return out


def label_np(q):
    return -1 if q.get("label") is None else q["label"]


def mask_np(q, num_frames):
    return np.array([f < len(q["frames"]) for f in range(num_frames)])
