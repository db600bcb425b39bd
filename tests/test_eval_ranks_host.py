"""CPU tests of the evaluation programs on several ranks (merlot_b200/eval_ranks.py, sort_story.eval_batches): the ranks'
batches against the one-rank batch sequence, the header-only skip path (no data checksum, parse or decode of another rank's
record; which corruption each rank reports), and, in world-2 gloo processes, checkpoint following under an injected clock
and a failure on one rank raising on both."""
import os
import socket
import struct
import threading
import traceback
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from merlot_b200 import sort_story as S
from merlot_b200 import tfrecord as T
from merlot_b200 import vcr_input as VI
from merlot_b200.dataloader import DevicePipeline, eval_decode_threads
from merlot_b200.eval_ranks import in_batch_order
from merlot_b200.tfrecord import RecordFormatError
from tests import story_records as SR
from tests import tfrecord_writer as W
from tests import vcr_records as VR

B = 3  # records per batch


def _write(tmp_path, kind, counts):
    if kind == "story":
        SR.write_stories(tmp_path, counts, max_sentence=3, sizes=[(8, 8)])
        return sorted(str(p) for p in tmp_path.glob("val-*.tfrecord"))
    VR.write_questions(tmp_path, counts, prefix="val", max_ctx=2, max_choice=2, sizes=[(8, 8)])
    return sorted(str(p) for p in tmp_path.glob("val-*.tfrecord"))


def _rank_batches(files, cycle, rank, world, b=B):
    tail = []
    return list(S.eval_batches(files, cycle, b, tail, rank=rank, world=world)), len(tail)


# files fewer than, as many as and more than the two interleave readers; every case ends in a partial batch
@pytest.mark.parametrize("counts", [[7], [4, 5], [3, 1, 4, 2, 5]])
@pytest.mark.parametrize("kind", ["story", "vcr"])
def test_rank_batches_are_the_one_rank_sequence(tmp_path, kind, counts):
    files = _write(tmp_path, kind, counts)
    cycle = min(2, len(files))
    one, dropped = _rank_batches(files, cycle, 0, 1)
    assert dropped == sum(counts) % B and len(one) == sum(counts) // B
    for world in (1, 2, 3):
        per_rank = [_rank_batches(files, cycle, r, world) for r in range(world)]
        assert [d for _, d in per_rank] == [dropped] * world  # the global count, known on every rank
        for r, (batches, _) in enumerate(per_rank):
            assert all(len(x) == B and None not in x for x in batches)
            assert len(batches) == len(range(r, len(one), world))
        assert in_batch_order([b for b, _ in per_rank]) == one


class _Counter:
    def __init__(self, fn, count=lambda *a: True):
        self.fn, self.count, self.calls = fn, count, 0
        self.lock = threading.Lock()

    def __call__(self, *a, **kw):
        if self.count(*a):
            with self.lock:
                self.calls += 1
        return self.fn(*a, **kw)


@pytest.mark.parametrize("world", [2, 3])
def test_other_ranks_data_is_never_checksummed(tmp_path, monkeypatch, world):
    files = _write(tmp_path, "story", [4, 5, 3])
    n = 12
    for rank in range(world):
        data_crc = _Counter(T.crc32c, lambda buf: len(buf) != 8)  # a header's checksum covers its 8 length bytes
        monkeypatch.setattr(T, "crc32c", data_crc)
        batches, dropped = _rank_batches(files, 2, rank, world, b=5)
        assert dropped == 2
        owned = sum(1 for i in range(n) if (i // 5) % world == rank)  # the owner of the partial batch reads it too
        assert data_crc.calls == owned and sum(map(len, batches)) == owned - (2 if (n // 5) % world == rank else 0)
        monkeypatch.undo()


class _CpuPipeline:
    """DevicePipeline.__init__ without a device or a thread: the test drives _produce() itself."""

    def __init__(self, device, num_threads, prefetch):
        self.device, self.num_threads, self.last_info = torch.device("cpu"), num_threads, None
        self._stop = threading.Event()
        self._pool = ThreadPoolExecutor(max_workers=num_threads)


def _cpu_stage(frames):
    offsets = np.zeros(len(frames), np.int64)
    return torch.empty(0, dtype=torch.uint8), offsets, np.array([f.shape[:2] for f in frames], dtype=np.int64)


@pytest.mark.parametrize("rank", [0, 1])
def test_vcr_pipeline_parses_and_decodes_its_batches_only(tmp_path, monkeypatch, rank):
    from merlot_b200 import ops
    from merlot_b200.config import NeatConfig
    _write(tmp_path, "vcr", [5, 4])
    config = NeatConfig.from_dict({"data": {"val_file": str(tmp_path / "val-*.tfrecord"), "num_threads": 2},
                                   "model": {"image_size": [16, 16]}, "optimizer": {}, "device": {"output_dir": str(tmp_path)},
                                   "downstream": {"task": "vcr", "mode": "answer"}})
    parse, decode = _Counter(VI.parse_example), _Counter(VI.decode_image)
    monkeypatch.setattr(DevicePipeline, "__init__", _CpuPipeline.__init__)
    monkeypatch.setattr(VI, "parse_example", parse)
    monkeypatch.setattr(VI, "decode_image", decode)
    monkeypatch.setattr(VI, "stage_frames", _cpu_stage)
    monkeypatch.setattr(VI, "_to_device", lambda a, device: torch.from_numpy(np.ascontiguousarray(a)))
    monkeypatch.setattr(ops, "frames_prepare", lambda src, plan, h, w: torch.zeros(len(plan["scaled_h"]), h, w, 3))
    pipe = VI.input_fn_builder(config, is_training=False, batch_size=2, rank=rank, world=2)
    seen = [feats["annot_id"] for feats, _ in pipe._produce()]
    pipe._pool.shutdown()
    order = ["val-0", "val-5", "val-1", "val-6", "val-2", "val-7", "val-3", "val-8", "val-4"]  # two files interleaved
    assert seen == [order[2 * k:2 * k + 2] for k in range(rank, 4, 2)] and pipe.dropped == 1
    assert parse.calls == decode.calls == 4  # two batches of two: nothing of the other rank's, nor of the dropped record


def _record_offsets(path):
    """(offset, length) of every record of a TFRecord file."""
    out, pos, raw = [], 0, open(path, "rb").read()
    while pos < len(raw):
        (length,) = struct.unpack("<Q", raw[pos:pos + 8])
        out.append((pos, length))
        pos += 12 + length + 4
    return out


def _corrupt(path, at):
    raw = bytearray(open(path, "rb").read())
    raw[at] ^= 0x40
    open(path, "wb").write(bytes(raw))


def _outcome(files, rank, world, b=2):
    try:
        _rank_batches(files, 1, rank, world, b=b)
        return "ok"
    except RecordFormatError as e:
        return str(e).split(": ", 1)[1]


def test_corrupt_data_is_reported_by_its_owner_only(tmp_path):
    files = _write(tmp_path, "story", [8])
    off, length = _record_offsets(files[0])[2]  # record 2: batch 1 of 2-record batches, rank 1's of 2
    _corrupt(files[0], off + 12 + length // 2)
    assert [_outcome(files, r, 2) for r in range(2)] == ["ok", "record data checksum mismatch"]
    assert [_outcome(files, r, 3) for r in range(3)] == ["ok", "record data checksum mismatch", "ok"]
    assert _outcome(files, 0, 1) == "record data checksum mismatch"


def test_corrupt_length_or_truncation_is_reported_by_every_rank(tmp_path):
    files = _write(tmp_path, "story", [8])
    off, _ = _record_offsets(files[0])[2]
    _corrupt(files[0], off + 1)
    assert [_outcome(files, r, 2) for r in range(2)] == ["record length checksum mismatch"] * 2
    files = _write(tmp_path, "story", [7])  # the last record, rank 1's of 2 (batch 3), loses its last bytes
    raw = open(files[0], "rb").read()
    open(files[0], "wb").write(raw[:-3])
    assert [_outcome(files, r, 2) for r in range(2)] == ["truncated record"] * 2


def test_decode_threads_split_over_local_ranks(monkeypatch):
    monkeypatch.delenv("LOCAL_WORLD_SIZE", raising=False)
    assert eval_decode_threads({}) == 64
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "8")
    assert eval_decode_threads({}) == 8 and eval_decode_threads({"num_threads": 5}) == 5
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "128")
    assert eval_decode_threads({}) == 1


# ---- world-2 gloo processes -----------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _follow(group, out, num_train_steps, timeout, poll, events):
    from merlot_b200 import vcr_validate as VV
    from tests.test_vcr_input_host import _Clock
    clk = _Clock(events if group.rank == 0 else [])
    seen = []
    for p in group.shared_prefixes(lambda sl: VV.follow_checkpoints(out, num_train_steps, timeout, poll, clk, sl), clk.sleep):
        seen.append(VV.checkpoint_step(p))
        if seen[-1] == 4:
            clk.t += 1000  # an evaluation longer than the timeout does not count against it
    return seen, clk.t


def _scenarios(rank, world, port, tmp, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    from pathlib import Path
    from merlot_b200.eval_ranks import RankFailure, eval_group
    from tests.test_vcr_input_host import _save
    res = {"rank": rank}
    try:
        with eval_group() as group:
            assert (group.rank, group.world, group.dist.get_backend()) == (rank, world, "gloo")
            final, lapse = Path(tmp) / "final", Path(tmp) / "lapse"
            if rank == 0:  # only rank 0 looks at the directory
                _save(final, 2)
                _save(final, 4)
            res["final"] = _follow(group, str(final), 10, 100, 10,
                                   [(1030, lambda: _save(final, 6)), (1030, lambda: _save(final, 8)),
                                    (1090, lambda: _save(final, 10)), (1095, lambda: _save(final, 12))])
            res["timeout"] = _follow(group, str(lapse), 100, 50, 7, [(20, lambda: _save(lapse, 3))])
            # a failure on rank 1 raises on both ranks; the ranks then go on together
            for name, fn in (("run", lambda: group.run_and_gather(lambda: [rank] if rank == 0 else
                                                                   VI.check_labels([{"annot_id": "val-3", "labels": [7]}],
                                                                                   ("answer",)))),
                             ("write", lambda: group.on_rank0(lambda: open(os.path.join(tmp, "no", "such"), "w")))):
                try:
                    fn()
                    res[name] = None
                except RankFailure as e:
                    res[name] = str(e)
            res["gather"] = in_batch_order(group.run_and_gather(lambda: [f"batch {k}" for k in range(rank, 5, world)]))
    except Exception:
        res["error"] = traceback.format_exc()
    q.put(res)


def test_two_gloo_ranks_follow_checkpoints_and_fail_together(tmp_path):
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_scenarios, args=(r, world, port, str(tmp_path), q)) for r in range(world)]
    try:
        for p in ps:
            p.start()
        res = sorted((q.get(timeout=180) for _ in range(world)), key=lambda r: r["rank"])
    finally:
        for p in ps:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    for r in res:
        assert "error" not in r, r["error"]
    # the same prefixes, oldest first, on both ranks, ending after num_train_steps; rank 0's clock as on one process
    assert res[0]["final"] == ([2, 4, 6, 8, 10], 1090) and res[1]["final"][0] == [2, 4, 6, 8, 10]
    assert res[0]["timeout"][0] == res[1]["timeout"][0] == [3] and 21 + 50 <= res[0]["timeout"][1] < 21 + 50 + 7
    for r in res:
        assert r["run"] == ("rank 1: ValueError: VCR record annot_id='val-3': label/answer_label is 7, outside [0, 4) "
                            "(an unlabelled record can only be scored without a loss)")
        assert r["write"].startswith("rank 0: FileNotFoundError:")
        assert r["gather"] == [f"batch {k}" for k in range(5)]
