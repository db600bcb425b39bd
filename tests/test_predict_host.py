"""Host tests of model_fn's PREDICT mode (no GPU): train.predictions() against a NumPy restatement of
model/modeling.py:774-784, the batch files and their reader, and the argument and configuration errors
`python -m merlot_b200.predict` raises before any device work."""
import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import predict
from merlot_b200.train import predictions


def _restated(features, bsz):
    """modeling.py:774-784 in NumPy: every key in sorted order; a scalar tiled to [bsz], a leading axis other than bsz
    reshaped to [bsz, -1]; then bf16 -> f32 (and, for the host files, every float as f32 and every integer as int32)."""
    out = {}
    for k in sorted(features):
        a = np.asarray(features[k])
        if a.ndim == 0:
            a = np.tile(a[None], [bsz])
        elif a.shape[0] != bsz:
            a = np.reshape(a, [bsz, -1])
        out[k] = a.astype(np.float32) if a.dtype.kind == "f" else a.astype(np.int32)
    return out


def test_predictions_follow_the_reference_reshapes():
    bsz, B, layers, S, L = 2, 8, 3, 20, 12
    g = torch.Generator().manual_seed(0)
    feats = {
        "self_attn_probs": torch.rand(bsz, B // bsz, S, S, generator=g),
        "lang_attn_probs": torch.rand(bsz, layers, L, L, generator=g),
        "masked_ids": torch.randint(0, 1000, (B, 16), generator=g, dtype=torch.int32),
        "input_ids": torch.randint(0, 1000, (bsz, 4, 8), generator=g, dtype=torch.int64),
        "shuffled_idx_img": torch.arange(16, dtype=torch.int32),
        "is_eoc": torch.rand(bsz, 4, generator=g) > 0.5,
        "mean_time": torch.rand(bsz, 4, generator=g).bfloat16(),
        "lang/loss": torch.tensor(1.25),
        "attn/encoder/viz2viz": torch.tensor(0.5, dtype=torch.float64),
        "contr/loss_all": torch.tensor(2.0).bfloat16(),
    }
    got = predictions(feats, bsz)
    ref = _restated({k: (v.float() if v.dtype == torch.bfloat16 else v).numpy() for k, v in feats.items()}, bsz)
    assert list(got) == sorted(feats)
    for k in ref:
        assert got[k].shape == ref[k].shape and got[k].dtype == ref[k].dtype, (k, got[k].shape, ref[k].shape)
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    assert got["masked_ids"].shape == (bsz, B // bsz * 16) and got["lang/loss"].tolist() == [1.25, 1.25]
    assert got["input_ids"].shape == (bsz, 4, 8) and got["shuffled_idx_img"].shape == (bsz, 8)


def test_batch_files_and_reader(tmp_path):
    bsz = 3
    batches = [{"b": np.full((bsz, 2), k, np.int32), "a": np.arange(bsz, dtype=np.float32) + 10 * k} for k in range(3)]
    for k in (2, 0, 1):  # written in any order, read in global order
        predict.write_batch(str(tmp_path), k, batches[k])
    videos = list(predict.read_predictions(str(tmp_path)))
    assert len(videos) == 9
    for i, v in enumerate(videos):
        k, j = divmod(i, bsz)
        assert sorted(v) == ["a", "b"] and float(v["a"]) == 10 * k + j and v["b"].tolist() == [k, k]
    again = tmp_path / "again"
    again.mkdir()
    predict.write_batch(str(again), 0, {"b": batches[0]["b"], "a": batches[0]["a"]})  # same bytes for any dict order
    assert (again / "batch-000000.npz").read_bytes() == (tmp_path / "batch-000000.npz").read_bytes()
    (tmp_path / "batch-000001.npz").unlink()
    with pytest.raises(ValueError, match="not batches"):
        list(predict.read_predictions(str(tmp_path)))


def _config(tmp_path, **over):
    cfg = {"data": {"val_file": str(tmp_path / "val-*.tfrecord"), "num_chunks": 4},
           "model": {"num_chunks_in_group": 2},
           "optimizer": {"num_train_steps": 4}, "device": {"output_dir": str(tmp_path / "run"), "val_batch_size": 2},
           "validate": {}}
    for k, v in over.items():
        cfg[k].update(v)
    path = tmp_path / "cfg.yaml"
    path.write_text(yaml.safe_dump(cfg))
    return str(path)


def test_program_errors_before_device_work(tmp_path, monkeypatch):
    from merlot_b200 import eval_ranks
    monkeypatch.setattr(eval_ranks, "eval_group", lambda: (_ for _ in ()).throw(AssertionError("device work started")))
    out = str(tmp_path / "pred")
    with pytest.raises(ValueError, match="val_file"):  # no held-out records
        predict.main([_config(tmp_path), "--out", out])
    (tmp_path / "val-00.tfrecord").write_bytes(b"")
    with pytest.raises(ValueError, match="holds no checkpoint"):  # Estimator.predict's default: the latest checkpoint
        predict.main([_config(tmp_path), "--out", out])
    with pytest.raises(ValueError, match="no .*index"):
        predict.main([_config(tmp_path), "--out", out, "--checkpoint", str(tmp_path / "model.ckpt-9")])
    with pytest.raises(ValueError, match="less than one batch"):
        predict.main([_config(tmp_path, validate={"eval_samples": 1}), "--out", out])
    with pytest.raises(ValueError, match="vcr"):
        predict.main([_vcr(tmp_path), "--out", out])
    (tmp_path / "model.ckpt-9.index").write_bytes(b"")
    (tmp_path / "pred").mkdir()
    (tmp_path / "pred" / "batch-000000.npz").write_bytes(b"")
    with pytest.raises(ValueError, match="already holds"):
        predict.main([_config(tmp_path), "--out", out, "--checkpoint", str(tmp_path / "model.ckpt-9")])
    with pytest.raises(SystemExit):  # --out is required
        predict.main([_config(tmp_path)])


def _vcr(tmp_path):
    path = _config(tmp_path)
    cfg = yaml.safe_load(open(path))
    cfg["downstream"] = {"task": "vcr"}
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    return path
