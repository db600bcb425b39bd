"""CPU tests of frame <-> transcript retrieval's host half: the NumPy oracle of K17's contract on hand-made rows, the metrics
arithmetic (ties, even N), the feature row <-> (batch, video, chunk) mapping, the assignment of query chunks to ranks, the
command line's refusals (all before any GPU work), the results line and the predictions file."""
import json

import numpy as np
import pytest
import yaml

from merlot_b200 import _lib
from merlot_b200 import retrieval_validate as RV
from tests import retrieval_oracle as RO

NAN = np.nan


# ---- K17's contract, restated -----------------------------------------------------------------------------------------
def test_oracle_counts_ties_and_orders_top_k():
    s = np.array([[3, 5, 5, 1, 5, 2],
                  [0, 0, 0, 0, 0, 0],
                  [9, NAN, 7, NAN, 8, 9]], np.float32)
    g, t, idx, val = RO.rank_topk(s, np.array([1, 3, 5]), 4)
    assert g.tolist() == [0, 0, 0]
    assert t.tolist() == [2, 5, 1]                       # other entries equal to the positive
    assert idx.tolist() == [[1, 2, 4, 0], [0, 1, 2, 3], [0, 5, 4, 2]]  # score descending, index ascending
    assert val.tolist() == [[5, 5, 5, 3], [0, 0, 0, 0], [9, 9, 8, 7]]
    g, t, _, _ = RO.rank_topk(s, np.array([3, 0, 2]), 1)
    assert g.tolist() == [5, 0, 3] and t.tolist() == [0, 5, 0]  # NaN is never greater


def test_oracle_nan_positive_short_rows_and_bad_pos():
    s = np.array([[NAN, 1, 2], [NAN, NAN, 4], [1, 2, 3]], np.float32)
    g, t, idx, val = RO.rank_topk(s, np.array([0, 2, 3]), 3)
    assert g.tolist() == [-1, 0, -2] and t.tolist() == [0, 0, 0]
    assert idx[1].tolist() == [2, -1, -1] and val[1, 0] == 4 and np.isnan(val[1, 1:]).all()  # fewer non-NaN entries than k
    assert idx[0].tolist() == [2, 1, -1]


def test_rank_topk_is_bound_from_the_header():
    restype, argtypes = _lib._PROTOTYPES["merlot_rank_topk"]
    assert len(argtypes) == 11 and argtypes[3] is _lib.C.c_longlong


# ---- metrics ------------------------------------------------------------------------------------------------------------
def test_metrics_arithmetic_with_ties_and_even_count():
    greater = np.array([0, 0, 4, 9, 10, 99])  # ranks 1, 1, 5, 10, 11, 100
    ties = np.array([0, 3, 0, 1, 0, 0])
    m = RV.direction_metrics(greater, ties)
    assert m == {"r1": 2 / 6, "r5": 3 / 6, "r10": 4 / 6, "median_rank": 7.5, "mean_rank": 128 / 6, "tied": 2}
    m = RV.direction_metrics(greater[:5], ties[:5])
    assert m["median_rank"] == 5.0 and m["mean_rank"] == 28 / 5


def test_results_line_schema_and_file(tmp_path):
    per = {"lang_to_viz": (np.array([0, 1, 2, 3]), np.zeros(4, np.int32)),
           "viz_to_lang": (np.array([0, 0, 0, 12]), np.array([0, 1, 0, 0]))}
    res = RV.results_line(7, 4, per)
    assert list(res) == ["global_step", "segments", "lang_to_viz", "viz_to_lang"]
    for d in RV.DIRECTIONS:
        assert sorted(res[d]) == ["mean_rank", "median_rank", "r1", "r10", "r5", "tied"]
    assert res["viz_to_lang"]["tied"] == 1 and res["lang_to_viz"]["median_rank"] == 2.5
    path = RV.append_result(str(tmp_path), res)
    RV.append_result(str(tmp_path), res)
    assert path == str(tmp_path / "eval" / "retrieval.jsonl")
    assert [json.loads(x) for x in open(path).read().splitlines()] == [res, res]


def test_nan_positive_raises_naming_the_segment():
    g = {"lang_to_viz": np.zeros(40, np.int32), "viz_to_lang": np.zeros(40, np.int32)}
    RV.check_nan_positives(g, 2, 4)
    g["viz_to_lang"][[21, 30]] = -1
    with pytest.raises(ValueError, match=r"viz_to_lang.*segment 21 \(global batch 2, video 1, chunk 1\).*2 queries"):
        RV.check_nan_positives(g, 2, 4)


# ---- rows, chunks and ranks ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch_size,num_chunks", [(1, 1), (2, 4), (16, 16), (3, 5)])
def test_row_to_segment_mapping(batch_size, num_chunks):
    nb = 3
    rows = np.arange(nb * batch_size * num_chunks).reshape(nb, batch_size, num_chunks)  # the arenas' row order
    for k in range(nb):
        for v in range(batch_size):
            for c in range(num_chunks):
                assert RV.segment_of(rows[k, v, c], batch_size, num_chunks) == (k, v, c)


@pytest.mark.parametrize("n,chunk", [(1, 1), (7, 3), (32, 32), (33, 8), (16384, 1024), (163840, 1000)])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_query_chunks_cover_each_row_once_across_ranks(n, chunk, world):
    chunks = RV.query_chunks(n, chunk)
    assert chunks[0][0] == 0 and chunks[-1][1] == n
    assert all(a[1] == b[0] for a, b in zip(chunks, chunks[1:]))
    assert all(0 < e - s <= chunk for s, e in chunks)
    owners = [RV.chunk_owner(c, world) for c in range(len(chunks))]
    per_rank = [[c for c, r in enumerate(owners) if r == rank] for rank in range(world)]
    assert sorted(c for p in per_rank for c in p) == list(range(len(chunks)))
    assert max(map(len, per_rank)) - min(map(len, per_rank)) <= 1  # round-robin


# ---- command line -------------------------------------------------------------------------------------------------------
def _config(tmp_path, records=True, **over):
    if records:
        (tmp_path / "val-00.tfrecord").write_bytes(b"")
    d = {"data": {"val_file": str(tmp_path / "val-*.tfrecord"), "num_chunks": 4},
         "model": {"hidden_size": 128, "contrastive_size": 128, "num_chunks_in_group": 2},
         "optimizer": {}, "device": {"output_dir": str(tmp_path / "out"), "val_batch_size": 2}, "validate": {},
         "downstream": {}}
    for k, v in over.items():
        d[k].update(v)
    path = tmp_path / "cfg.yaml"
    path.write_text(yaml.safe_dump(d))
    return str(path)


@pytest.fixture
def no_gpu(monkeypatch):
    """Fails the test if the command line gets as far as the process group or the GPU."""
    import merlot_b200.eval_ranks as ER

    def touched(*a, **kw):
        raise AssertionError("the refusal came after the GPU was touched")
    monkeypatch.setattr(ER, "eval_group", touched)
    monkeypatch.setattr(RV, "Validator", touched)


@pytest.mark.parametrize("task", ["vcr", "video_mc", "video_qa", "video_fib"])
def test_refuses_finetuning_task(tmp_path, no_gpu, task):
    with pytest.raises(ValueError, match=f"downstream.task is '{task}'"):
        RV.main([_config(tmp_path, downstream={"task": task})])


def test_refuses_empty_val_file(tmp_path, no_gpu):
    with pytest.raises(ValueError, match="data.val_file"):
        RV.main([_config(tmp_path, records=False)])
    with pytest.raises(ValueError, match="data.val_file"):
        RV.main([_config(tmp_path, data={"val_file": ""})])


def test_refuses_less_than_one_batch(tmp_path, no_gpu):
    with pytest.raises(ValueError, match="less than one batch"):
        RV.main([_config(tmp_path, validate={"eval_samples": 1})])


@pytest.mark.parametrize("args,msg", [(["--chunk", "0"], "--chunk 0"), (["--chunk", "-3"], "--chunk -3"),
                                      (["--top-k", "0"], "--top-k 0"), (["--top-k", "33"], "--top-k 33"),
                                      (["--predictions", "p.npz"], "--predictions needs --checkpoint")])
def test_refuses_bad_options(tmp_path, no_gpu, args, msg):
    with pytest.raises(ValueError, match=msg):
        RV.main([_config(tmp_path)] + args)


def test_defaults():
    a = RV.parse_args(["c.yaml"])
    assert (a.chunk, a.top_k, a.seed, a.checkpoint, a.predictions) == (1024, 10, 0, None, None)


# ---- predictions file ------------------------------------------------------------------------------------------------------
def test_predictions_file(tmp_path):
    n, k = 12, 3
    rng = np.random.default_rng(0)
    pred = {d: (rng.integers(0, n, n).astype(np.int32), np.zeros(n, np.int32), rng.integers(0, n, (n, k)).astype(np.int32),
                rng.standard_normal((n, k)).astype(np.float32)) for d in RV.DIRECTIONS}
    path = RV.write_predictions(str(tmp_path / "sub" / "p.npz"), pred, batch_size=3, num_chunks=2)
    z = np.load(path)
    assert z["segment"].tolist() == list(range(n))
    assert [RV.segment_of(i, 3, 2) for i in range(n)] == list(zip(z["batch"].tolist(), z["video"].tolist(), z["chunk"].tolist()))
    for d in RV.DIRECTIONS:
        assert np.array_equal(z[f"{d}_rank"], 1 + pred[d][0].astype(np.int64))
        assert np.array_equal(z[f"{d}_topk_idx"], pred[d][2]) and np.array_equal(z[f"{d}_topk_score"], pred[d][3])
