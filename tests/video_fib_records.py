"""TEST INFRASTRUCTURE ONLY: fill-in-the-blank video QA records (the schema of merlot_b200/video_fib_input.py,
INTEGRATION.md) built from a seed with tests/tfrecord_writer.py, answer-token files, and a NumPy restatement of the
parser's text and blank position."""
import json

import numpy as np

from tests import tfrecord_writer as W
from tests import video_mc_records as MR

MASK = 1  # utils/encode/encoder.py


def question(rng, k, num_frames, num_answers, max_words=30, vocab=1000, sizes=MR.SIZES, frames=None, oov_every=0):
    """One question as plain values: 1..num_frames frames, a sentence of 1..max_words word ids in [7, vocab) with one of
    them replaced by MASK, and an answer in [0, num_answers), or -1 for every question k with k % oov_every ==
    oov_every - 1.  Set a value to None to leave its feature out."""
    n = int(rng.integers(1, num_frames + 1)) if frames is None else frames
    words = rng.integers(7, vocab, int(rng.integers(1, max_words + 1))).tolist()
    words[int(rng.integers(0, len(words)))] = MASK
    q = {"id": f"q-{k}",
         "frames": [W.jpeg(rng, *sizes[(3 * k + f) % len(sizes)], gray=(k % 5 == 4 and f == 0)) for f in range(n)],
         "question": words, "answer": int(rng.integers(0, num_answers))}
    if oov_every and k % oov_every == oov_every - 1:
        q["answer"] = -1
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
        elif key == "answer":
            feats[key] = ("int64", [v])
        else:
            feats[key] = ("int64", v, len(v) % 2 == 0)
    return W.example(feats)


def write_questions(dirpath, counts, num_frames, num_answers, prefix="fib", seed=0, **kw):
    """Files <prefix>-000.tfrecord, ... holding counts[f] questions each; returns the questions in write order."""
    rng = np.random.default_rng(seed)
    out = []
    for f, n in enumerate(counts):
        qs = [question(rng, len(out) + i, num_frames, num_answers, **kw) for i in range(n)]
        out += qs
        W.write_records(dirpath / f"{prefix}-{f:03d}.tfrecord", [example(q) for q in qs])
    return out


def answers(rng, num_answers, vocab=1000, max_tokens=1):
    """num_answers distinct answers of 1..max_tokens token ids in [7, vocab) each."""
    out, seen = [], set()
    while len(out) < num_answers:
        a = rng.integers(7, vocab, int(rng.integers(1, max_tokens + 1))).tolist()
        if tuple(a) not in seen:
            seen.add(tuple(a))
            out.append(a)
    return out


def write_answers(path, ans) -> str:
    with open(path, "w") as f:
        json.dump(ans, f)
    return str(path)


def text_np(q, max_len):
    """[max_len] int32: START + question + END, int64 -> int32, truncated, padded with 0."""
    row = np.asarray([MR.START] + list(q.get("question") or []) + [MR.END], np.int64).astype(np.int32)[:max_len]
    out = np.zeros(max_len, np.int32)
    out[:len(row)] = row
    return out


def blank_np(q):
    """The MASK's position in the text: 1 + its index in the question."""
    return 1 + list(q["question"]).index(MASK)
