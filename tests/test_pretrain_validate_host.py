"""CPU tests of pretraining validation's host half: the evaluation input's record order against a plain restatement of
sorted globs, an ordered interleave and drop_remainder; its batches and draws on 1, 2 and 3 ranks against the one-rank
sequence (other ranks' records never checksummed, parsed or decoded); its parser against tests/input_oracle.py; the
training pipeline's draws; the results line; and every host check of a bad record or configuration."""
import json
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import dataloader as D
from merlot_b200 import ops
from merlot_b200 import pretrain_validate as PV
from merlot_b200 import tfrecord as T
from merlot_b200.config import NeatConfig
from merlot_b200.tfrecord import parse_example
from tests import input_oracle as O
from tests import tfrecord_writer as W

N_CHUNKS, G, L, HW = 4, 2, 8, (32, 48)


def _write(tmp_path, counts, num_chunks=N_CHUNKS, seed=3, prefix="val"):
    """counts[i] pretraining records in <prefix>-i.tfrecord (written in reverse so that the glob's sort matters).  Returns
    {record bytes: its chunks}."""
    rng = np.random.default_rng(seed)
    by_record = {}
    for fi in reversed(range(len(counts))):
        recs = []
        for e in range(counts[fi]):
            chunks = W.video_chunks(rng, num_chunks, frame_hw=(8, 8), max_caption=12, video=f"f{fi}e{e}", vocab=1000)
            rec = W.chunks_example(chunks)
            by_record[rec] = chunks
            recs.append(rec)
        W.write_records(tmp_path / f"{prefix}-{fi:02d}.tfrecord", recs)
    return by_record


def _config(tmp_path, val_file=None, num_threads=2, **data):
    d = {"val_file": str(tmp_path / "val-*.tfrecord") if val_file is None else val_file, "num_chunks": N_CHUNKS,
         "chunk_text_len": L, "num_threads": num_threads, "random_scale_min": 1.0, "random_scale_max": 1.5, "augment_prob": 0.5,
         "clean_asr_prob": 0.5, "shuffle_chunks": True}
    d.update(data)
    return NeatConfig.from_dict({"data": d, "model": {"image_size": list(HW), "num_chunks_in_group": G, "image_shuffle_prob": 0.5},
                                 "optimizer": {}, "device": {"output_dir": str(tmp_path / "out"), "val_batch_size": 2}})


class _Counter:
    def __init__(self, fn, count=lambda *a: True):
        self.fn, self.count, self.calls = fn, count, 0
        self.lock = threading.Lock()

    def __call__(self, *a, **kw):
        if self.count(*a):
            with self.lock:
                self.calls += 1
        return self.fn(*a, **kw)


def _cpu_init(self, device, num_threads, prefetch):
    """DevicePipeline.__init__ without a device or a thread: the test drives _produce() itself."""
    self.device, self.last_info = torch.device("cpu"), None
    self._stop = threading.Event()
    self._pool = ThreadPoolExecutor(max_workers=num_threads)


def _cpu_stage(frames):
    return torch.empty(0, dtype=torch.uint8), np.zeros(len(frames), np.int64), np.array([f.shape[:2] for f in frames], np.int64)


@pytest.fixture
def cpu(monkeypatch):
    """The pipelines on the host: no thread, no pinned staging, K14 replaced by zeros.  Returns the parse/decode counters."""
    parse, decode = _Counter(D.parse_example), _Counter(D.decode_jpeg)
    monkeypatch.setattr(D.DevicePipeline, "__init__", _cpu_init)
    monkeypatch.setattr(D, "parse_example", parse)
    monkeypatch.setattr(D, "decode_jpeg", decode)
    monkeypatch.setattr(D, "stage_frames", _cpu_stage)
    monkeypatch.setattr(D, "_to_device", lambda a, device: torch.from_numpy(np.ascontiguousarray(a)))
    monkeypatch.setattr(ops, "frames_prepare", lambda src, plan, h, w: torch.zeros(len(plan["scaled_h"]), h, w, 3))
    return parse, decode


def _run(pipe):
    out = list(pipe._produce())
    pipe._pool.shutdown()
    return out


def _eval(config, rank=0, world=1, seed=7, batch_size=2):
    return D.input_fn_builder(config, is_training=False, rank=rank, world=world, seed=seed, batch_size=batch_size)


def _reference_order(tmp_path, counts, cycle, b):
    """The record order restated: sorted file names; parallel_interleave(cycle, block_length=1, sloppy=False) -- one record
    from each open file in turn, a file that ends replaced in its slot by the next file, that slot's turn yielding nothing;
    then batch(b, drop_remainder=True)."""
    names = sorted(str(p) for p in tmp_path.glob("val-*.tfrecord"))
    contents = [list(T.read_records(n)) for n in names]
    nxt, slots, order, i = cycle, [[*c] for c in contents[:cycle]], [], 0
    while slots:
        i %= len(slots)
        if slots[i]:
            order.append(slots[i].pop(0))
            i += 1
        elif nxt < len(contents):
            slots[i] = [*contents[nxt]]
            nxt += 1
            i += 1
        else:
            del slots[i]
    whole = len(order) // b * b
    return [order[k:k + b] for k in range(0, whole, b)], len(order) - whole


# ---- record order and ranks --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("counts,threads", [([5], 2), ([3, 4], 2), ([2, 1, 4, 3], 2), ([3, 2, 4], 8)])
def test_record_order_is_sorted_glob_ordered_interleave_drop_remainder(tmp_path, cpu, counts, threads):
    _write(tmp_path, counts)
    config = _config(tmp_path, num_threads=threads)
    pipe = _eval(config)
    got = [info["records"] for _, info in _run(pipe)]
    ref, dropped = _reference_order(tmp_path, counts, min(threads, len(counts)), 2)
    assert got == ref and pipe.dropped == dropped


@pytest.mark.parametrize("counts", [[7], [4, 5], [3, 1, 4, 2, 5]])
def test_rank_batches_and_draws_are_the_one_rank_sequence(tmp_path, cpu, monkeypatch, counts):
    _write(tmp_path, counts)
    config = _config(tmp_path)
    one = _run(_eval(config))
    total = sum(counts)
    assert len(one) == total // 2
    for world in (1, 2, 3):
        for rank in range(world):
            parse, decode = _Counter(D.parse_example), _Counter(D.decode_jpeg)
            data_crc = _Counter(T.crc32c, lambda buf: len(buf) != 8)  # a header's checksum covers its 8 length bytes
            monkeypatch.setattr(D, "parse_example", parse)
            monkeypatch.setattr(D, "decode_jpeg", decode)
            monkeypatch.setattr(T, "crc32c", data_crc)
            pipe = _eval(config, rank, world)
            mine = _run(pipe)
            ks = list(range(rank, len(one), world))
            assert [info["batch"] for _, info in mine] == ks and pipe.dropped == total % 2
            for (feats, info), k in zip(mine, ks):
                ref_feats, ref_info = one[k]
                assert info["records"] == ref_info["records"]
                np.testing.assert_array_equal(info["do_clean"], ref_info["do_clean"])
                for key, v in ref_info["frame_draws"].items():
                    np.testing.assert_array_equal(info["frame_draws"][key], v, err_msg=key)
                for key, v in ref_feats.items():
                    assert torch.equal(feats[key], v), key
            # only this rank's records are checksummed, parsed and decoded (the partial batch's owner reads it too)
            owned = sum(1 for i in range(total) if (i // 2) % world == rank)
            assert data_crc.calls == owned
            assert parse.calls == 2 * len(ks) and decode.calls == 2 * len(ks) * N_CHUNKS


def test_draws_depend_on_seed_and_batch_only(tmp_path, cpu):
    _write(tmp_path, [6])
    a = _run(_eval(_config(tmp_path), seed=7))
    b = _run(_eval(_config(tmp_path), seed=8))
    assert len(a) == 3
    for (_, ia), (_, ib), k in zip(a, b, range(3)):
        rng = np.random.default_rng([7, k])  # the documented key: (seed, k)
        np.testing.assert_array_equal(ia["do_clean"], rng.random(2) < 0.5)
        assert not np.array_equal(ia["frame_draws"]["scale"], ib["frame_draws"]["scale"])


# ---- parser -------------------------------------------------------------------------------------------------------------
def test_parser_matches_oracle_without_process_example(tmp_path, cpu):
    by_record = _write(tmp_path, [3, 3])
    config = _config(tmp_path, shuffle_chunks=True)
    batches = _run(_eval(config))
    assert len(batches) == 3
    for feats, info in batches:
        assert feats["images"].shape == (2 * N_CHUNKS, *HW, 3)  # flattened, not transposed
        assert feats["shuffled_idx_img"].dtype == torch.int32
        assert feats["shuffled_idx_img"].tolist() == list(range(G)) * (2 * N_CHUNKS // G)
        assert sorted(feats) == sorted(["images", "input_ids", "video_src_ids", "is_eoc", "youtube_id", "chunk_num", "mean_time",
                                        "shuffled_idx_img"])
        for e, rec in enumerate(info["records"]):
            ref = O.dataset_parser_text(by_record[rec], L, bool(info["do_clean"][e]))
            for key, v in ref.items():  # no chunk shuffle even with shuffle_chunks: True
                got = feats[key][e].numpy()
                assert got.dtype == v.dtype, key
                np.testing.assert_array_equal(got, v, err_msg=key)
        assert info["frame_draws"]["augment"].shape == (2 * N_CHUNKS,) and "process_draws" not in info


def test_training_draws_are_unchanged(tmp_path, cpu):
    """The training pipeline draws, from its (seed, rank) generator, what it drew before the evaluation input shared its
    parser: per batch the records of the shuffled stream, the clean coins, frame_draws, then the process_example seed."""
    _write(tmp_path, [3, 4], prefix="train")
    config = _config(tmp_path)
    config.data["train_file"] = str(tmp_path / "train-*.tfrecord")
    pipe = D.input_fn_builder(config, True, rank=1, seed=11, batch_size=2)
    produced = pipe._produce()
    got = [next(produced) for _ in range(4)]
    pipe._stop.set()
    pipe._pool.shutdown()
    files = sorted(str(p) for p in tmp_path.glob("train-*.tfrecord"))
    rng = np.random.default_rng([11, 1])
    recs = D.shuffled_records(files, rng, 2, 256, None)
    for feats, info in got:
        records = [next(recs) for _ in range(2)]
        do_clean = rng.random(2) < 0.5
        fd = D.frame_draws(rng, 2 * N_CHUNKS, config.data)
        pd = D.make_draws(2, N_CHUNKS, G, 0.5, int(rng.integers(1 << 62)))
        assert info["records"] == records
        np.testing.assert_array_equal(info["do_clean"], do_clean)
        for key, v in fd.items():
            np.testing.assert_array_equal(info["frame_draws"][key], v, err_msg=key)
        for key, v in pd.items():
            assert torch.equal(info["process_draws"][key], v), key
        assert feats["images"].shape == (2 * N_CHUNKS, *HW, 3)


# ---- host checks ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunks", [3, 5])
def test_record_with_other_chunk_count_raises_naming_it(tmp_path, cpu, chunks):
    _write(tmp_path, [4])
    rng = np.random.default_rng(0)
    W.write_records(tmp_path / "val-01.tfrecord",  # batch 2 of one reader: the odd record, then a good one
                    [W.chunks_example(W.video_chunks(rng, n, frame_hw=(8, 8), video=v, vocab=1000))
                     for n, v in ((chunks, "odd"), (N_CHUNKS, "good"))])
    with pytest.raises(ValueError, match=rf"record 0 of evaluation batch 2 \(c00/youtube_id 'odd[0-9a-f]+'\): {chunks} chunks"):
        _run(_eval(_config(tmp_path, num_threads=1)))


def test_video_src_ids_outside_range_raises_naming_the_record(tmp_path, cpu, monkeypatch):
    _write(tmp_path, [4])
    parse_text = D.parse_text

    def bad(ex, n, L, do_clean):
        out = parse_text(ex, n, L, do_clean)
        if bytes(ex["c00/youtube_id"][0]).startswith(b"f0e3"):
            out["video_src_ids"] = out["video_src_ids"] + n
        return out
    monkeypatch.setattr(D, "parse_text", bad)
    with pytest.raises(ValueError, match=r"record 1 of evaluation batch 1 \(c00/youtube_id 'f0e3.*video_src_ids .* outside \[0, 4\)"):
        _run(_eval(_config(tmp_path)))


def test_token_id_outside_vocabulary_raises_naming_the_record(tmp_path, cpu):
    _write(tmp_path, [4])
    config = _config(tmp_path)
    config.model["vocab_size"] = 7  # every caption token is >= 7
    with pytest.raises(ValueError, match=r"record 0 of evaluation batch 0 \(c00/youtube_id 'f0e0.*token id \d+ outside the "
                                         r"vocabulary \[0, 7\)"):
        _run(_eval(config))


def test_batch_not_divisible_into_groups_raises(tmp_path, cpu):
    _write(tmp_path, [4])
    config = _config(tmp_path, num_chunks=3)
    with pytest.raises(ValueError, match="is not divisible by model.num_chunks_in_group 2"):
        _eval(config, batch_size=1)


def test_image_index_beyond_position_embeddings_raises(tmp_path, cpu):
    _write(tmp_path, [4])
    config = _config(tmp_path)
    config.model["max_vision_pos_embeddings"] = 1
    with pytest.raises(ValueError, match="exceeds max_vision_pos_embeddings 1"):
        _eval(config)


@pytest.mark.parametrize("val_file", ["", "nothing-*.tfrecord"])
def test_empty_or_unmatched_val_file_raises(tmp_path, val_file):
    config = _config(tmp_path, val_file=str(tmp_path / val_file) if val_file else "")
    with pytest.raises(ValueError, match="data.val_file"):
        D.input_fn_builder(config, is_training=False)
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump({"data": dict(config.data), "model": dict(config.model), "optimizer": {},
                                    "device": dict(config.device)}))
    with pytest.raises(ValueError, match="data.val_file"):  # before any device is touched
        PV.main([str(path)])


# ---- results line ---------------------------------------------------------------------------------------------------------
def test_eval_samples_truncates_and_less_than_a_batch_raises(tmp_path):
    config = _config(tmp_path)
    assert PV.eval_batch_count(config) is None  # absent: every whole batch
    for samples, n in ((2, 1), (5, 2), (6, 3)):
        config.validate = {"eval_samples": samples}
        assert PV.eval_batch_count(config) == n
    config.validate = {"eval_samples": 1}
    with pytest.raises(ValueError, match="less than one batch"):
        PV.eval_batch_count(config)


def test_results_line_holds_per_batch_means(tmp_path):
    keys = ["attn/encoder/lang2lang", "contr/loss_all", "lang/acc", "lang/loss", "temporal/loss"]
    rng = np.random.default_rng(0)
    vecs = [torch.from_numpy(rng.random(len(keys) + 1).astype(np.float32)) for _ in range(5)]
    res = PV.reduce_batches(keys, vecs, 16, 40)
    mean = torch.stack(vecs).mean(0)
    assert res == dict({"global_step": 40, "loss": float(mean[0]), "videos": 80}, **{k: float(mean[i + 1]) for i, k in enumerate(keys)})
    np.testing.assert_allclose([res[k] for k in ["loss"] + keys], np.mean(np.stack([v.numpy() for v in vecs]), 0), rtol=1e-6)
    path = PV.append_result(str(tmp_path), res)
    PV.append_result(str(tmp_path), dict(res, global_step=50))
    lines = [json.loads(x) for x in open(path).read().splitlines()]
    assert [x["global_step"] for x in lines] == [40, 50] and lines[0] == res
    assert "learning_rate" not in lines[0]
    with pytest.raises(ValueError, match="no whole batch of 16 videos"):
        PV.reduce_batches(keys, [], 16, 40)

