"""GPU tests of the VCR input and validator (pytest -m gpu): the training and evaluation pipelines' batches against
tests/input_oracle.py and the NumPy restatement of the parsers (tests/vcr_records.py), a train step fed by the pipeline
against the same step fed the same tensors built directly, and the validator over two checkpoints written by the trainer
against a per-question loop of cls_head_val + cls_loss, with and without chunks, labelled and unlabelled."""
import io
import json
import threading

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import vcr_input as VI
from merlot_b200 import vcr_validate as VV
from merlot_b200.config import NeatConfig
from tests import input_oracle as IO
from tests import story_records as SR
from tests import vcr_records as R
from tests.test_gpu_sort_story import _check_bilinear

pytestmark = pytest.mark.gpu
DEV = "cuda"
OUT = (48, 64)
OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=4, num_warmup_steps=0, weight_decay_rate=0.01,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"], {"weight_decay_rate": 0}]])


def _u8(jpg):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(jpg)).convert("RGB"))


def _config(tmp_path, tiny_cfg, mode="answer", val="val-*.tfrecord", **device):
    model = dict(tiny_cfg, num_texts=4, num_chunks_in_group=1, image_size=list(OUT), vocab_size=50370,
                 max_position_embeddings=256, hidden_dropout_prob=0.1, transpose_input=True)
    d = {"data": {"train_file": str(tmp_path / "train-*.tfrecord"), "val_file": str(tmp_path / val), "draw": "segm",
                  "num_threads": 2, "shuffle_buffer_size": 4},
         "model": model, "optimizer": dict(OCFG),
         "device": dict({"use_tpu": False, "output_dir": str(tmp_path / "out"), "train_batch_size": 2, "val_batch_size": 3,
                         "iterations_per_loop": 2}, **device),
         "downstream": {"task": "vcr", "mode": mode}, "validate": {"eval_samples": 7, "eval_timeout": 0}}
    path = tmp_path / f"vcr_{mode}_{val[:3]}.yaml"
    path.write_text(yaml.safe_dump(d))
    return str(path), NeatConfig.from_dict(d)


def test_train_pipeline_batch_matches_oracle(tmp_path, tiny_cfg):
    qs = {q["annot_id"]: q for q in R.write_questions(tmp_path, [3, 2], prefix="train", seed=1)}
    _, config = _config(tmp_path, tiny_cfg)
    with VI.input_fn_builder(config, is_training=True, seed=4, batch_size=2) as pipe:
        for _ in range(3):
            batch = next(pipe)
            info = pipe.last_info
            torch.cuda.synchronize()
            assert batch["images"].shape == (4, *OUT, 3) and batch["images"].dtype == torch.bfloat16
            assert batch["lm_input"].shape == (16, 184) and batch["lm_targets"].shape == (4,)
            imgs = batch["images"].float().cpu().numpy()
            plan = info["plan"]
            for k, aid in enumerate(info["annot_id"]):
                q = qs[aid]
                lm, labels = R.joint_np(q)
                np.testing.assert_array_equal(batch["lm_input"][8 * k:8 * k + 8].cpu().numpy(), lm.reshape(8, 184))
                np.testing.assert_array_equal(batch["lm_targets"][2 * k:2 * k + 2].cpu().numpy(), labels)
                for j, mode in enumerate(R.MODES):  # [q answer, q rationale] per question
                    f = 2 * k + j
                    ref, want = IO.load_and_resize_img(_u8(q[f"{mode}/segm/image"]), OUT, plan["scale"][f], plan["u_y"][f],
                                                       plan["u_x"][f], 0, 0, np.ones(3, np.float32))
                    assert tuple(int(plan[n][f]) for n in ("scaled_h", "scaled_w", "offset_y", "offset_x")) == want
                    assert 0.9 <= plan["scale"][f] < 1.1
                    _check_bilinear(imgs[f], ref, f"{aid} {mode}")
    assert not [t.name for t in threading.enumerate() if t.name.startswith("merlot-")]


@pytest.mark.parametrize("mode", ["answer", "rationale"])
def test_eval_pipeline_batch_matches_oracle(tmp_path, tiny_cfg, mode):
    written = R.write_questions(tmp_path, [4, 3], prefix="val", seed=2)
    qs = {q["annot_id"]: q for q in written}
    _, config = _config(tmp_path, tiny_cfg, mode=mode)
    L = VI.EVAL_MAX_NUM_TOKENS[mode]
    seen = []
    with VI.input_fn_builder(config, is_training=False) as pipe:
        for batch in pipe:
            torch.cuda.synchronize()
            assert batch["images"].shape == (3, *OUT, 3) and batch["lm_input"].shape == (3, 4, L)
            imgs = batch["images"].float().cpu().numpy()
            for k, aid in enumerate(batch["annot_id"]):
                q = qs[aid]
                lm, label = R.eval_np(q, mode)
                assert batch["img_id"][k] == q["img_id"] and int(batch["lm_targets"][k]) == label
                np.testing.assert_array_equal(batch["lm_input"][k].cpu().numpy(), lm)
                u8 = _u8(q[f"{mode}/segm/image"])
                sh, sw, oy, ox = SR.eval_plan(u8.shape[0], u8.shape[1], OUT)
                ref = IO.bf16_round(IO.resize_and_pad(u8.astype(np.float32) * IO.INV255, OUT, sh, sw, oy, ox, 0))
                _check_bilinear(imgs[k], ref, f"{aid} {mode}")
            seen += batch["annot_id"]
        assert pipe.dropped == 1
    assert seen == ["val-0", "val-4", "val-1", "val-5", "val-2", "val-6"]  # sorted files interleaved, no shuffle


def test_missing_label_raises_from_pipeline_unless_unlabelled(tmp_path, tiny_cfg):
    rng = np.random.default_rng(0)
    q = R.question(rng, 0)
    q["annot_id"], q["label/answer_label"] = "val-unlabelled", None
    from tests import tfrecord_writer as W
    W.write_records(tmp_path / "val-000.tfrecord", [R.vcr_example(q)])
    _, config = _config(tmp_path, tiny_cfg, val_batch_size=1)
    with VI.input_fn_builder(config, is_training=False) as pipe:
        with pytest.raises(ValueError, match="annot_id='val-unlabelled': label/answer_label is -1"):
            next(pipe)
    with VI.input_fn_builder(config, is_training=False, labelled=False) as pipe:
        assert int(next(pipe)["lm_targets"][0]) == -1


def test_train_step_from_pipeline_equals_direct_tensors(tmp_path, tiny_cfg):
    from merlot_b200.vcr import vcr_model_fn_builder
    qs = {q["annot_id"]: q for q in R.write_questions(tmp_path, [3, 3], prefix="train", seed=3)}
    _, config = _config(tmp_path, tiny_cfg)
    with VI.input_fn_builder(config, is_training=True, seed=0, batch_size=2) as pipe:
        feats = next(pipe)
        ids = pipe.last_info["annot_id"]
    direct = {"images": feats["images"].clone(),
              "lm_input": torch.from_numpy(np.concatenate([R.joint_np(qs[a])[0].reshape(8, 184) for a in ids])).to(DEV),
              "lm_targets": torch.from_numpy(np.concatenate([R.joint_np(qs[a])[1] for a in ids]).astype(np.int32)).to(DEV)}
    assert all(torch.equal(feats[k], direct[k]) for k in direct)
    runs = []
    for f in (feats, direct, direct):
        fn = vcr_model_fn_builder(config, seed=5)
        spec = fn(f)
        loss = float(spec.metrics["loss"])
        spec.train_op()
        torch.cuda.synchronize()
        runs.append((loss, fn.store.p.clone()))
    assert runs[0][0] == runs[1][0]
    if torch.equal(runs[1][1], runs[2][1]):
        assert torch.equal(runs[0][1], runs[1][1])
    else:  # the towers' weight gradients accumulate with fp32 atomics: two direct runs already differ in the last bits
        assert (runs[0][1] - runs[1][1]).norm() <= 2 * (runs[1][1] - runs[2][1]).norm() + 1e-7 * runs[1][1].norm()


def _per_question_loop(config, prefix, mode):
    """(avg, loss, logits [n, 4]) of the first eval_samples // val_batch_size batches, one question per forward."""
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import ParamStore
    from merlot_b200.vcr import cls_head_val, cls_loss, head_from_store
    store = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer, task="vcr")
    store.restore_checkpoint(prefix)
    b = config.device["val_batch_size"]
    n = config.validate["eval_samples"] // b * b
    accs, losses, logits = [], [], []
    with torch.no_grad(), VI.input_fn_builder(config, is_training=False, batch_size=1) as pipe:
        for _, q in zip(range(n), pipe):
            m = MerlotModel(config.model, is_training=False, use_tpu=False, image=q["images"], input_ids=q["lm_input"].reshape(4, -1),
                            mask_input=False, params=store, log_attention_probs=False)
            lg = cls_head_val(m, head_from_store(store, mode), mode)
            loss, acc = cls_loss(lg, q["lm_targets"])
            accs.append(float(acc))
            losses.append(float(loss))
            logits.append(lg.float().cpu().numpy()[0])
    per_batch = np.array(losses).reshape(-1, b).mean(1)
    return float(np.mean(accs)), float(per_batch.mean()), np.stack(logits)


@pytest.mark.parametrize("mode", ["answer", "rationale"])
def test_validator_over_trainer_checkpoints(tmp_path, tiny_cfg, mode, capsys):
    from merlot_b200 import train
    R.write_questions(tmp_path, [3, 3], prefix="train", seed=4)
    val = R.write_questions(tmp_path, [5, 3], prefix="val", seed=5)
    path, config = _config(tmp_path, tiny_cfg, mode=mode)
    train.main([path])
    assert "training on synthetic batches" not in capsys.readouterr().out
    out = tmp_path / "out"
    ckpts = [str(out / "model.ckpt-2"), str(out / "model.ckpt-4")]
    clock = iter(range(10 ** 6))
    res = VV.main([path], clock=lambda: next(clock), sleep=lambda s: None)
    lines = [json.loads(x) for x in (out / "eval" / "results.jsonl").read_text().splitlines()]
    assert [r["global_step"] for r in res] == [x["global_step"] for x in lines] == [2, 4]
    chunked = VV.main([path, "--chunk", "2", "--poll-interval", "0"], clock=lambda: next(clock), sleep=lambda s: None)
    for prefix, r, c in zip(ckpts, res, chunked):
        avg, loss, _ = _per_question_loop(config, prefix, mode)
        for got in (r, c):
            # the CE kernel's accuracy is an fp32 mean with a small denominator guard: equal to about 1e-5
            assert got["questions"] == 6 and got["avg"] == pytest.approx(avg, abs=1e-5)
            assert got["loss"] == pytest.approx(loss, rel=2e-3), (prefix, got["loss"], loss)
        assert c["loss"] == pytest.approx(r["loss"], rel=2e-3)
    # predictions of one checkpoint, then the same questions without their labels
    VV.main([path, "--checkpoint", ckpts[1], "--predictions", str(tmp_path / "p.npz")])
    _, _, logits = _per_question_loop(config, ckpts[1], mode)
    with np.load(tmp_path / "p.npz") as z:
        order = ["val-0", "val-5", "val-1", "val-6", "val-2", "val-7"]
        assert list(z["annot_id"]) == order and list(z["img_id"]) == [f"movie_{a[4:]}.jpg" for a in order]
        by_id = {q["annot_id"]: q for q in val}
        assert list(z["label"]) == [by_id[a][f"label/{mode}_label"] for a in order]
        np.testing.assert_allclose(z["log_prob"], VV.log_softmax(logits), atol=2e-2)
        assert (z["prediction"] == z["log_prob"].argmax(-1)).all()
        labelled = {k: z[k] for k in z.files}
    for q in val:
        for m in R.MODES:
            q[f"label/{m}_label"] = None
    from tests import tfrecord_writer as W
    W.write_records(tmp_path / "unl-000.tfrecord", [R.vcr_example(q) for q in val[:5]])
    W.write_records(tmp_path / "unl-001.tfrecord", [R.vcr_example(q) for q in val[5:]])
    upath, _ = _config(tmp_path, tiny_cfg, mode=mode, val="unl-*.tfrecord")
    (res_u,) = VV.main([upath, "--checkpoint", ckpts[1], "--predictions", str(tmp_path / "u.npz"), "--unlabelled"])
    assert res_u["avg"] is None and res_u["loss"] is None
    with np.load(tmp_path / "u.npz") as z:
        assert (z["label"] == -1).all()
        np.testing.assert_array_equal(z["log_prob"], labelled["log_prob"])
        np.testing.assert_array_equal(z["annot_id"], labelled["annot_id"])
    assert len((out / "eval" / "results.jsonl").read_text().splitlines()) == 5  # 2 + 2 followed, 1 single; none unlabelled
