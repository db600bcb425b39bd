"""GPU tests of the evaluation programs on two ranks (pytest -m gpu): `vcr_validate` and `sort_story` run as two processes
-- on one GPU with gloo for the collectives, or on two GPUs with NCCL -- against the one-process run on the same records
and checkpoints.  The model is the tiny patch-embed one: each batch runs the same kernels on the same rows on either side,
and that model's evaluation forward is bit-reproducible (tests/test_gpu_vcr_input.py compares two runs' log_prob bit for
bit), so the files must match bit for bit.  (The hybrid stem is not used: its GroupNorm atomics are not bit-reproducible.)"""
import json
import os
import socket
import traceback

import numpy as np
import pytest
import torch

from merlot_b200 import sort_story as S
from merlot_b200 import vcr_validate as VV
from tests import story_records as SR
from tests import vcr_records as R
from tests.test_gpu_sort_story import _cfg as _story_cfg
from tests.test_gpu_sort_story import _save_checkpoint
from tests.test_gpu_sort_story import _write_config as _story_config
from tests.test_gpu_vcr_input import _config as _vcr_config

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _vcr_rank(path, checkpoint, predictions):
    clock = iter(range(10 ** 6))
    followed = VV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
    single = VV.main([path, "--checkpoint", checkpoint, "--predictions", predictions])
    return followed, single


def _story_rank(path, out):
    return S.main([path, "--out", out])


def _rank_main(rank, world, port, target, args, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    try:
        from merlot_b200.eval_ranks import backend
        out = {"vcr": _vcr_rank, "story": _story_rank}[target](*args)
        q.put({"rank": rank, "out": out, "backend": backend(), "device": torch.cuda.current_device()})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


def _run_ranks(world, target, *args):
    """`target` in `world` spawned processes as torchrun would start them; every process is joined before returning."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_rank_main, args=(r, world, port, target, args, q)) for r in range(world)]
    try:
        for p in ps:
            p.start()
        res = sorted((q.get(timeout=900) for _ in range(world)), key=lambda r: r["rank"])
    finally:
        for p in ps:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in res:
        assert "error" not in r, r["error"]
    two_gpus = torch.cuda.device_count() >= world
    for r in res:
        assert r["backend"] == ("nccl" if two_gpus else "gloo") and r["device"] == (r["rank"] if two_gpus else 0)
    return [r["out"] for r in res]


def _results(out_dir):
    path = out_dir / "eval" / "results.jsonl"
    lines = [json.loads(x) for x in path.read_text().splitlines()]
    path.unlink()
    return lines


@pytest.mark.parametrize("mode", ["answer", "rationale"])
def test_vcr_validation_on_two_ranks_matches_one_process(tmp_path, tiny_cfg, mode):
    from merlot_b200 import train
    R.write_questions(tmp_path, [3, 3], prefix="train", seed=4)
    R.write_questions(tmp_path, [5, 3, 4], prefix="val", seed=5)  # three files, two interleave readers
    # eval_samples 7 in batches of 2: global batches 0 and 2 on rank 0, batch 1 on rank 1, 5 records never evaluated
    path, _ = _vcr_config(tmp_path, tiny_cfg, mode=mode, val_batch_size=2)
    train.main([path])
    out = tmp_path / "out"
    ckpt = str(out / "model.ckpt-4")
    clock = iter(range(10 ** 6))
    one = VV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
    one += VV.main([path, "--checkpoint", ckpt, "--predictions", str(tmp_path / "one.npz")])
    one_lines = _results(out)
    assert [r["global_step"] for r in one] == [2, 4, 4] and all(r["questions"] == 6 for r in one)
    ranks = _run_ranks(2, "vcr", path, ckpt, str(tmp_path / "two.npz"))
    two_lines = _results(out)
    # rank 0 alone appended its lines, equal to the last bit; every rank returns the one-process results
    assert two_lines == one_lines
    for followed, single in ranks:
        assert followed + single == one
    with np.load(tmp_path / "one.npz") as a, np.load(tmp_path / "two.npz") as b:
        assert sorted(a.files) == sorted(b.files) == ["annot_id", "img_id", "label", "log_prob", "prediction"]
        assert list(a["annot_id"]) == ["val-0", "val-5", "val-1", "val-6", "val-2", "val-7"]
        for k in a.files:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_story_scores_on_two_ranks_match_one_process(tmp_path, tiny_cfg, monkeypatch):
    cfg = _story_cfg(tiny_cfg)
    SR.write_stories(tmp_path, [4, 3, 4], seed=9)  # 11 stories: 5 batches of 2 (3 on rank 0, 2 on rank 1), 1 dropped
    path, _ = _story_config(tmp_path, cfg, 2)
    _save_checkpoint(cfg, str(tmp_path / "out"))
    monkeypatch.delenv("SORTSTORY_PATH", raising=False)
    one = S.main([str(path), "--out", str(tmp_path / "one.npz")])
    ranks = _run_ranks(2, "story", str(path), str(tmp_path / "two.npz"))
    assert ranks[0] == ranks[1] == one  # Spearman, distance, pairwise and the best permutations, on every rank
    a, b = S.read_logits_npz(str(tmp_path / "one.npz")), S.read_logits_npz(str(tmp_path / "two.npz"))
    assert len(a) == 10 and sorted(a) == sorted(b)
    for sid in a:
        assert sorted(a[sid]) == sorted(b[sid])
        for k in a[sid]:
            np.testing.assert_array_equal(a[sid][k], b[sid][k], err_msg=f"story {sid} {k}")
