"""Multiple-choice video QA on the GPU (pytest -m gpu): the mc_cls head and the video_mc step (merlot_b200/video_mc.py)
against the fp32 oracle restatement (tests/video_mc_oracle.py over tests/multi_image_oracle.py) on bf16-rounded weights,
with the oracle drawing the very dropout masks the kernels draw; the equivalences with VCR's head, masked frame slots and
gradient accumulation; the input pipeline against the NumPy restatement; the validator over saved checkpoints, on one and
two ranks; and a forward at a realistic size.  Bars as tests/test_gpu_vcr_train.py: losses 1e-3 relative, activations
1e-2 and gradients 4e-2 relative-Frobenius."""
import io
import json
import os
import socket
import tempfile
import traceback

import numpy as np
import pytest
import torch
import yaml

from oracle import merlot_oracle as O
from tests import multi_image_oracle as MIO
from tests import video_mc_oracle as MO
from tests import video_mc_records as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=0, weight_decay_rate=0.01,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"], {"weight_decay_rate": 0}]])


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def mc_cfg(tiny_cfg, F=3, C=5, **kw):
    return dict(dict(tiny_cfg, num_imgs=F, num_texts=C, num_chunks_in_group=1, hidden_dropout_prob=0.1), **kw)


def build(cfg, seed=1, tower_scale=3.0, encoder_scale=5.0, device=DEV):
    """Oracle-initialised video_mc variables, GEMM operands rounded to bf16, in a ParamStore(task="video_mc"); the two
    scalings of tests/test_gpu_vcr_train.py.build keep the candidates' first tokens and the logits apart."""
    from merlot_b200.params import ParamStore
    params = MO.init_params(cfg, seed=seed, perturb=0.05)
    for k in params:
        if k.startswith(MO.TOWER) and k.endswith("kernel"):
            params[k] = params[k] * tower_scale
        elif k.startswith("encoder/layer") and k.endswith("kernel"):
            params[k] = params[k] * encoder_scale
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    store = ParamStore(cfg, device=device, optimizer_cfg=OCFG, task="video_mc")
    store.load_tf_dict(params)
    return params, store


def batch(cfg, b, L=16, hw=(64, 96), seed=0, counts=None):
    """b questions: images [b*F] (zeros in empty slots), img_mask [b, F] (question i holds counts[i] frames), ids [b*C, L],
    targets [b]."""
    F, C = cfg["num_imgs"], cfg["num_texts"]
    g = torch.Generator().manual_seed(seed)
    counts = counts or [F - i % F for i in range(b)]
    mask = torch.arange(F)[None] < torch.tensor(counts)[:, None]
    image = torch.rand(b * F, *hw, 3, generator=g).bfloat16().float() * mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, cfg["vocab_size"], (b * C, L), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(L // 2, L + 1, (b * C,), generator=g)
    ids = (ids * (torch.arange(L)[None] < lens[:, None])).int()
    target = torch.randint(0, C, (b,), generator=g).int()
    return image, mask, ids, target


def neat(cfg, **opt):
    from merlot_b200.config import NeatConfig
    return NeatConfig.from_dict({"data": {}, "model": dict(cfg, image_size=[64, 96]), "optimizer": dict(OCFG, **opt),
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_video_mc"},
                                 "downstream": {"task": "video_mc"}})


def feats_of(image, mask, ids, target):
    return {"images": image.to(DEV).bfloat16(), "img_mask": mask.to(DEV), "lm_input": ids.to(DEV), "lm_targets": target.to(DEV)}


@pytest.mark.parametrize("stem", ["patch", "hybrid"])
def test_training_step_against_oracle(tiny_cfg, monkeypatch, stem):
    """C = 5, F = 3, 3 questions holding 3, 2 and 1 frames, hidden dropout 0.1 under the kernels' own masks: logits, loss,
    accuracy, every parameter gradient and one AdamW step against the oracle.  With the hybrid stem the oracle's
    lite_resnet50 is a leaf holding the GPU's stem output (tests/test_gpu_vcr_train.py's rule)."""
    from merlot_b200 import video_mc as VM
    cfg = mc_cfg(tiny_cfg, resnet_layers=[1, 2, 1] if stem == "hybrid" else [])
    params, store = build(cfg)
    image, mask, ids, target = batch(cfg, 3, seed=3)
    seed = 2 ** 32 + 7
    fn = VM.video_mc_model_fn_builder(neat(cfg), store=store, seed=seed)
    spec = fn(feats_of(image, mask, ids, target), None, "train")
    m = spec.model
    if stem == "hybrid":
        rc = m._stem.tape[-1][1]["y"]
        N, hs, ws = image.shape[0], 64 // 16, 96 // 16
        leaf_rc = rc.float().cpu().reshape(N, hs, ws, rc.shape[1]).clone().requires_grad_(True)
        monkeypatch.setattr(O, "lite_resnet50", lambda x, p, scope, layers, width=64, rnd=O._ident: leaf_rc)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    hook = MO.dropout_hook(seed, 0.1)
    om = MIO.MultiImageOracle(cfg, leaf, image, ids, img_mask=mask, log_attention_probs=False, dropout=hook)
    assert rel(m.encoder_hidden_states["lang"], om.encoder_hidden_states["lang"]) < 1e-2
    ref_logits = MO.mc_head_train(om, leaf, 5, dropout=hook)
    ref_loss, _ = MO.mc_loss(ref_logits, target)
    logits = m._mc["logits"][:, :5]
    assert tuple(logits.shape) == (3, 5) and rel(logits, ref_logits) < 1e-2
    assert abs(float(spec.metrics["loss"]) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    # the CE kernel's accuracy is an fp32 mean with a small denominator guard: equal to about 1e-5
    assert float(spec.metrics["accuracy"]) == pytest.approx(float((logits.argmax(-1).cpu() == target.long()).float().mean()),
                                                            abs=1e-5)
    no_drop = MO.mc_head_train(om, {k: v.detach() for k, v in leaf.items()}, 5, dropout=MO.dropout_hook(seed + 1, 0.1))
    assert rel(logits, no_drop) > 1e-2  # negative control: another seed's tower masks
    store.g.zero_()
    d_hidden = VM.mc_head_backward(m, store)
    m.backward(d_hidden_state=d_hidden)
    ref_loss.backward()
    grads = store.to_tf_dict("g")
    assert set(grads) == set(leaf)
    worst = {k: rel(grads[k], v.grad) for k, v in leaf.items()
             if "resnet50lite" not in k and v.grad is not None and float(v.grad.norm()) >= 1e-7}
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    for k in ("mc_cls/classifier_mlp1/kernel", "mc_cls/classifier_mlp0/kernel", "mc_cls/classifier_mlp0/bias",
              "vision_backbone/img_idx_pe", "encoder/layer00/query_layer/kernel"):
        assert k in worst, k
    if stem == "hybrid":
        vals = sorted(worst.values())
        assert len(worst) > 40 and max(vals) < 6e-2 and vals[len(vals) // 2] < 2.5e-2, top
        assert rel(m.d_rc, leaf_rc.grad.reshape(N * hs * ws, -1)) < 4e-2
    else:
        assert len(worst) > 40 and max(worst.values()) < 4e-2, top
    assert float(grads["mc_cls/classifier_mlp1/bias"].abs().max()) < 1e-6  # softmax is shift invariant
    p_before = {k: v.clone() for k, v in store.to_tf_dict("p").items()}
    adam = O.AdamOracle(p_before, OCFG)
    adam.apply_gradients(p_before, grads)
    fn.optimizer.apply_gradients()
    after = store.to_tf_dict("p")
    for k in after:
        assert (after[k] - p_before[k]).abs().max().item() < 2e-6, k
    assert float(store.P("mc_cls/classifier_mlp1/kernel")[:, 1:].abs().max()) == 0.0
    assert float(store.g.abs().max()) == 0.0 and store.global_step == 1


def test_train_op_runs_and_eval_follows_the_trained_tower(tiny_cfg):
    """Two train_op steps through model_fn, then the eval and predict modes on the updated weights against the oracle; the
    predict mode runs no CE kernel."""
    from merlot_b200 import ops
    from merlot_b200 import video_mc as VM
    cfg = mc_cfg(tiny_cfg)
    _, store = build(cfg)
    fn = VM.video_mc_model_fn_builder(neat(cfg), store=store, seed=3)
    before = store.P("mc_cls/classifier_mlp0/kernel").clone()
    for s in range(2):
        spec = fn(feats_of(*batch(cfg, 2, seed=10 + s)))
        spec.train_op()
    assert store.global_step == 2 and not torch.equal(before, store.P("mc_cls/classifier_mlp0/kernel"))
    image, mask, ids, target = batch(cfg, 2, seed=20, counts=[2, 3])
    f = feats_of(image, mask, ids.reshape(2, 5, -1), target)
    spec = fn(f, None, "eval")
    assert spec.train_op is None
    trained = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v)
               for k, v in store.to_tf_dict("p").items()}
    om = MIO.MultiImageOracle(cfg, trained, image, ids, img_mask=mask, log_attention_probs=False)
    ref = MO.mc_head_train(om, trained, 5)
    assert tuple(spec.metrics["logits"].shape) == (2, 5) and rel(spec.metrics["logits"], ref) < 1e-2
    ref_loss, _ = MO.mc_loss(ref, target)
    assert abs(float(spec.metrics["loss"]) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    assert torch.equal(spec.metrics["predictions"].cpu(), spec.metrics["logits"].argmax(-1).cpu())
    calls = []
    real = ops.softmax_ce_fwd
    ops.softmax_ce_fwd = lambda *a, **k: (calls.append(1), real(*a, **k))[1]
    try:
        pred = fn({k: v for k, v in f.items() if k != "lm_targets"}, None, "predict")
    finally:
        ops.softmax_ce_fwd = real
    assert calls == [] and "loss" not in pred.metrics
    assert torch.equal(pred.metrics["logits"], spec.metrics["logits"])


class _Stand:
    """A model as the heads read it: the joint hidden state, its pieces and the store's buffers."""

    def __init__(self, model, hidden, num_texts):
        self.encoder_info = {"hidden_state": hidden}
        self.encoder_pieces, self._bufs, self.store, self.num_texts = model.encoder_pieces, model._bufs, model.store, num_texts


def test_four_choices_one_frame_is_vcr_answer_head(tiny_cfg):
    """C = 4, F = 1, all-true img_mask, dropout off: the hidden state is bitwise that of img_mask=None (VCR's input), and the
    mc_cls head with the answer tower's weights computes, bit for bit, VCR's answer logits: the same kernels in the same
    order on the same rows (both heads read the answer images' sequences, [b*4, Sj, H])."""
    from merlot_b200 import vcr
    from merlot_b200 import video_mc as VM
    from merlot_b200.modeling import MerlotModel
    from tests.test_gpu_vcr_train import batch as vcr_batch
    from tests.test_gpu_vcr_train import build as vcr_build
    cfg = dict(tiny_cfg, num_texts=4, num_chunks_in_group=1, hidden_dropout_prob=0.0)
    vparams, vstore = vcr_build(cfg, tower_scale=10.0)
    mparams = {k: v for k, v in vparams.items() if k.split("/")[0] not in ("answer_cls", "rationale_cls")}
    mparams.update({k.replace("answer_cls/", "mc_cls/"): v for k, v in vparams.items() if k.startswith("answer_cls/")})
    from merlot_b200.params import ParamStore
    mstore = ParamStore(dict(cfg, num_imgs=1), device=DEV, optimizer_cfg=OCFG, task="video_mc")
    mstore.load_tf_dict(mparams)
    image, ids, target = vcr_batch(cfg, 2)  # 4 images (answer, rationale, answer, rationale), 16 texts
    mv = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), params=vstore)
    mm = MerlotModel(dict(cfg, num_imgs=1), is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV),
                     img_mask=torch.ones(4, 1, dtype=torch.bool, device=DEV), params=mstore)
    assert torch.equal(mv.encoder_info["hidden_state"], mm.encoder_info["hidden_state"])
    vcr_logits = vcr.cls_head(mv, vstore)  # [4, 4]: rows 0 and 2 from answer_cls on images 0 and 2
    y = mm.encoder_info["hidden_state"]
    answer_rows = y.reshape(2, 2, 4, *y.shape[1:])[:, 0].reshape(8, *y.shape[1:]).contiguous()
    mc_logits = VM.mc_head(_Stand(mm, answer_rows, 4), mstore)
    assert torch.equal(mc_logits, vcr_logits[0::2])


def test_masked_slot_pixels_do_not_change_the_logits(tiny_cfg):
    """Eval mode: zeros or random pixels in the empty frame slots give bitwise the same logits (no valid token attends to a
    masked frame's tokens)."""
    from merlot_b200 import video_mc as VM
    cfg = mc_cfg(tiny_cfg)
    _, store = build(cfg)
    fn = VM.video_mc_model_fn_builder(neat(cfg), store=store)
    image, mask, ids, target = batch(cfg, 3, seed=5, counts=[1, 2, 3])
    noisy = image.clone()
    empty = ~mask.reshape(-1)
    noisy[empty] = torch.rand(noisy[empty].shape, generator=torch.Generator().manual_seed(8)).bfloat16().float()
    outs = [fn(feats_of(im, mask, ids, target), None, "eval").metrics["logits"].clone() for im in (image, noisy)]
    assert torch.equal(outs[0], outs[1])
    other = mask.clone()
    other[0, 1] = True  # a slot that counts changes them
    assert not torch.equal(fn(feats_of(noisy, other, ids, target), None, "eval").metrics["logits"], outs[0])


def test_accumulation_matches_the_whole_batch(tiny_cfg):
    """A = 2 micro-batches of 2 questions against one batch of 4, dropout off: the same loss and the same gradient handed to
    AdamW (the mean over micro-batches of the per-micro-batch means)."""
    from merlot_b200 import video_mc as VM
    from tests.test_gpu_accumulation import capture_applied_gradient
    cfg = mc_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    micro = [feats_of(*batch(cfg, 2, seed=30 + j)) for j in range(2)]
    whole = {k: torch.cat([f[k] for f in micro], 0) for k in micro[0]}
    grads, losses = [], []
    for feats in (micro, whole):
        _, store = build(cfg)
        fn = VM.video_mc_model_fn_builder(neat(cfg), store=store)
        seen = capture_applied_gradient(fn, store)
        spec = fn(feats)
        spec.train_op()
        torch.cuda.synchronize()
        assert store.global_step == 1
        grads.append(torch.cat([v.reshape(-1) for v in seen.values()]))
        losses.append(float(spec.metrics["loss"]))
    print(f"video_mc A=2 x 2 vs 1 x 4: loss {losses[0]:.6f} vs {losses[1]:.6f}, gradient {rel(grads[0], grads[1]):.2e}")
    assert abs(losses[0] - losses[1]) <= 1e-4 * abs(losses[1])
    assert rel(grads[0], grads[1]) <= 1e-3


# ------------------------------------------------------------------------------------------------------------
# input pipeline and validator
# ------------------------------------------------------------------------------------------------------------
OUT = (48, 64)


def _u8(jpg):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(jpg)).convert("RGB"))


def _config(tmp_path, tiny_cfg, val="val-*.tfrecord", F=3, C=5, **device):
    model = dict(tiny_cfg, num_imgs=F, num_texts=C, num_chunks_in_group=1, image_size=list(OUT), vocab_size=1000,
                 max_position_embeddings=64, hidden_dropout_prob=0.1, transpose_input=True)
    d = {"data": {"train_file": str(tmp_path / "train-*.tfrecord"), "val_file": str(tmp_path / val), "num_threads": 2,
                  "shuffle_buffer_size": 4},
         "model": model, "optimizer": dict(OCFG, num_train_steps=4),
         "device": dict({"use_tpu": False, "output_dir": str(tmp_path / "out"), "train_batch_size": 2, "val_batch_size": 3,
                         "iterations_per_loop": 2}, **device),
         "downstream": {"task": "video_mc", "max_text_len": 40}, "validate": {"eval_samples": 7, "eval_timeout": 0}}
    path = tmp_path / f"mc_{val[:3]}.yaml"
    path.write_text(yaml.safe_dump(d))
    from merlot_b200.config import NeatConfig
    return str(path), NeatConfig.from_dict(d)


def _check_batch(batch, qs, plan, F, C, draws=None):
    from tests import input_oracle as IO
    from tests.test_gpu_sort_story import _check_bilinear
    b = len(batch["id"])
    assert batch["images"].shape == (b * F, *OUT, 3) and batch["images"].dtype == torch.bfloat16
    assert batch["lm_input"].shape == (b * C, 40) and batch["img_mask"].shape == (b, F)
    imgs = batch["images"].float().cpu().numpy()
    for i, rid in enumerate(batch["id"]):
        q = qs[rid]
        np.testing.assert_array_equal(batch["lm_input"][i * C:(i + 1) * C].cpu().numpy(), R.texts_np(q, C, 40))
        np.testing.assert_array_equal(batch["img_mask"][i].cpu().numpy(), R.mask_np(q, F))
        assert int(batch["lm_targets"][i]) == R.label_np(q)
        for f in range(F):
            s = i * F + f
            if f >= len(q["frames"]):
                assert float(np.abs(imgs[s]).max()) == 0.0, (rid, f)  # an empty slot is all zeros
                continue
            u8 = _u8(q["frames"][f])
            if draws is None:
                from tests import story_records as SR
                sh, sw, oy, ox = SR.eval_plan(u8.shape[0], u8.shape[1], OUT)
                ref = IO.bf16_round(IO.resize_and_pad(u8.astype(np.float32) * IO.INV255, OUT, sh, sw, oy, ox, 0))
            else:  # one draw per question, every frame of it
                assert plan["scale"][s] == draws["scale"][i] and plan["u_y"][s] == draws["u_y"][i]
                ref, want = IO.load_and_resize_img(u8, OUT, draws["scale"][i], draws["u_y"][i], draws["u_x"][i], 0, 0,
                                                   np.ones(3, np.float32))
                assert tuple(int(plan[n][s]) for n in ("scaled_h", "scaled_w", "offset_y", "offset_x")) == want
            _check_bilinear(imgs[s], ref, f"{rid} frame {f}")


def test_pipelines_match_the_restatement(tmp_path, tiny_cfg):
    from merlot_b200 import video_mc_input as MI
    train_qs = {q["id"]: q for q in R.write_questions(tmp_path, [3, 2], 3, 5, prefix="train", seed=1)}
    val = R.write_questions(tmp_path, [4, 3], 3, 5, prefix="val", seed=2)
    _, config = _config(tmp_path, tiny_cfg)
    with MI.input_fn_builder(config, is_training=True, seed=4, batch_size=2) as pipe:
        for _ in range(3):
            b = next(pipe)
            torch.cuda.synchronize()
            _check_batch(b, train_qs, pipe.last_info["plan"], 3, 5, pipe.last_info["draws"])
    seen = []
    with MI.input_fn_builder(config, is_training=False) as pipe:
        for b in pipe:
            torch.cuda.synchronize()
            _check_batch(b, {q["id"]: q for q in val}, None, 3, 5)
            seen += b["id"]
        assert pipe.dropped == 1
    assert seen == ["q-0", "q-4", "q-1", "q-5", "q-2", "q-6"]  # sorted files interleaved, no shuffle


def _in_memory(config, store, labelled=True):
    """{accuracy, loss, questions, logits} of the first eval_samples // val_batch_size batches, evaluated in this process on
    `store` as it is, one batch per forward."""
    from merlot_b200 import video_mc_input as MI
    from merlot_b200.video_mc import video_mc_model_fn_builder
    fn = video_mc_model_fn_builder(config, store=store)
    b = config.device["val_batch_size"]
    n = config.validate["eval_samples"] // b
    acc, losses, logits, ids = [], [], [], []
    with torch.no_grad(), MI.input_fn_builder(config, is_training=False, labelled=labelled) as pipe:
        for _, batch in zip(range(n), pipe):
            spec = fn({k: batch[k] for k in ("images", "img_mask", "lm_input", "lm_targets")}, None,
                      "eval" if labelled else "predict")
            if labelled:
                acc.append(float(spec.metrics["accuracy"]))
                losses.append(float(spec.metrics["loss"]))
            logits.append(spec.metrics["logits"].float().cpu().numpy())
            ids += batch["id"]
    return {"accuracy": float(np.mean(acc)) if acc else None, "loss": float(np.mean(losses)) if losses else None,
            "questions": n * b, "logits": np.concatenate(logits), "id": ids}


def test_save_resume_and_validate(tmp_path, tiny_cfg, capsys):
    """The trainer on records writes checkpoints 2 and 4; the validator follows them and its results lines equal the
    in-memory evaluation of each restored checkpoint; --chunk gives the same means; --predictions holds id, log_prob,
    prediction and label; --unlabelled runs no CE and writes no line.  Restoring a checkpoint gives back its parameters,
    moments and step bit for bit, and a resumed trainer continues from it."""
    from merlot_b200 import ops, train
    from merlot_b200 import vcr_validate as VV
    from merlot_b200 import video_mc_validate as MV
    from merlot_b200.params import ParamStore
    R.write_questions(tmp_path, [3, 3], 3, 5, prefix="train", seed=4)
    val = R.write_questions(tmp_path, [5, 3], 3, 5, prefix="val", seed=5)
    path, config = _config(tmp_path, tiny_cfg)
    train.main([path])
    assert "training on synthetic batches" not in capsys.readouterr().out
    out = tmp_path / "out"
    ckpts = [str(out / "model.ckpt-2"), str(out / "model.ckpt-4")]
    clock = iter(range(10 ** 6))
    res = MV.main([path], clock=lambda: next(clock), sleep=lambda s: None)
    lines = [json.loads(x) for x in (out / "eval" / "results.jsonl").read_text().splitlines()]
    assert [r["global_step"] for r in res] == [x["global_step"] for x in lines] == [2, 4]
    assert all(set(x) == {"global_step", "accuracy", "loss", "questions"} for x in lines)
    chunked = MV.main([path, "--chunk", "2", "--poll-interval", "0"], clock=lambda: next(clock), sleep=lambda s: None)
    for prefix, r, c in zip(ckpts, res, chunked):
        store = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer, task="video_mc")
        store.restore_checkpoint(prefix)
        mem = _in_memory(config, store)
        assert r["questions"] == mem["questions"] == 6
        assert r["accuracy"] == pytest.approx(mem["accuracy"], abs=1e-6) and r["loss"] == pytest.approx(mem["loss"], rel=1e-6)
        assert c["accuracy"] == pytest.approx(r["accuracy"], abs=1e-5) and c["loss"] == pytest.approx(r["loss"], rel=2e-3)
    # restore is exact, and a resumed run continues from the latest checkpoint
    a = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer, task="video_mc")
    a.restore_checkpoint(ckpts[1])
    a.save_checkpoint(str(tmp_path / "again"))
    b = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer, task="video_mc")
    b.restore_checkpoint(str(tmp_path / "again"))
    assert b.global_step == 4 and torch.equal(a.p, b.p) and torch.equal(a.m, b.m) and torch.equal(a.v, b.v)
    assert float(b.m[b.entries["mc_cls/classifier_mlp0/kernel"].offset:].abs().max()) > 0  # the tower's moments are saved
    resumed = dict(yaml.safe_load(open(path)), optimizer=dict(OCFG, num_train_steps=5))
    rpath = tmp_path / "resume.yaml"
    rpath.write_text(yaml.safe_dump(resumed))
    train.main([str(rpath)])
    assert "restored" in capsys.readouterr().out and (out / "model.ckpt-5.index").exists()
    # predictions of one checkpoint, labelled then unlabelled
    MV.main([path, "--checkpoint", ckpts[1], "--predictions", str(tmp_path / "p.npz")])
    store = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer, task="video_mc")
    store.restore_checkpoint(ckpts[1])
    mem = _in_memory(config, store)
    by_id = {q["id"]: q for q in val}
    with np.load(tmp_path / "p.npz") as z:
        assert sorted(z.files) == ["id", "label", "log_prob", "prediction"]
        assert list(z["id"]) == mem["id"] == ["q-0", "q-5", "q-1", "q-6", "q-2", "q-7"]
        assert list(z["label"]) == [by_id[i]["label"] for i in mem["id"]] and z["log_prob"].shape == (6, 5)
        np.testing.assert_allclose(z["log_prob"], VV.log_softmax(mem["logits"]), atol=1e-6)
        assert (z["prediction"] == z["log_prob"].argmax(-1)).all()
        labelled = {k: z[k] for k in z.files}
    for q in val:
        q["label"] = None
    from tests import tfrecord_writer as W
    W.write_records(tmp_path / "unl-000.tfrecord", [R.example(q) for q in val[:5]])
    W.write_records(tmp_path / "unl-001.tfrecord", [R.example(q) for q in val[5:]])
    upath, _ = _config(tmp_path, tiny_cfg, val="unl-*.tfrecord")
    calls = []
    real = ops.softmax_ce_fwd
    ops.softmax_ce_fwd = lambda *a, **k: (calls.append(1), real(*a, **k))[1]
    try:
        (res_u,) = MV.main([upath, "--checkpoint", ckpts[1], "--predictions", str(tmp_path / "u.npz"), "--unlabelled"])
    finally:
        ops.softmax_ce_fwd = real
    assert calls == [] and res_u["accuracy"] is None and res_u["loss"] is None
    with np.load(tmp_path / "u.npz") as z:
        assert (z["label"] == -1).all()
        np.testing.assert_array_equal(z["log_prob"], labelled["log_prob"])
        np.testing.assert_array_equal(z["id"], labelled["id"])
    assert len((out / "eval" / "results.jsonl").read_text().splitlines()) == 5  # 2 + 2 followed, 1 single; none unlabelled


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, path, checkpoint, predictions, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    try:
        from merlot_b200 import video_mc_validate as MV
        clock = iter(range(10 ** 6))
        followed = MV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
        single = MV.main([path, "--checkpoint", checkpoint, "--predictions", predictions])
        q.put({"rank": rank, "out": (followed, single)})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


def test_validation_on_two_ranks_matches_one_process(tmp_path, tiny_cfg):
    """Two processes (two GPUs with NCCL, or one GPU with gloo) write the same results lines and predictions file as one,
    bit for bit, and return the same results (the tiny patch-embed model's evaluation forward is bit-reproducible)."""
    import torch.multiprocessing as mp
    from merlot_b200 import train
    from merlot_b200 import video_mc_validate as MV
    R.write_questions(tmp_path, [3, 3], 3, 5, prefix="train", seed=4)
    R.write_questions(tmp_path, [5, 3, 4], 3, 5, prefix="val", seed=5)  # three files, two interleave readers
    path, _ = _config(tmp_path, tiny_cfg, val_batch_size=2)  # eval_samples 7: batches 0, 2 on rank 0, batch 1 on rank 1
    train.main([path])
    out = tmp_path / "out"
    ckpt = str(out / "model.ckpt-4")
    results = out / "eval" / "results.jsonl"
    clock = iter(range(10 ** 6))
    one = MV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
    one += MV.main([path, "--checkpoint", ckpt, "--predictions", str(tmp_path / "one.npz")])
    one_lines = results.read_text()
    results.unlink()
    assert [r["global_step"] for r in one] == [2, 4, 4] and all(r["questions"] == 6 for r in one)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_rank_main, args=(r, 2, port, path, ckpt, str(tmp_path / "two.npz"), q)) for r in range(2)]
    try:
        for p in ps:
            p.start()
        res = sorted((q.get(timeout=900) for _ in range(2)), key=lambda r: r["rank"])
    finally:
        for p in ps:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in res:
        assert "error" not in r, r["error"]
        followed, single = r["out"]
        assert followed + single == one
    assert results.read_text() == one_lines
    with np.load(tmp_path / "one.npz") as a, np.load(tmp_path / "two.npz") as b:
        assert sorted(a.files) == sorted(b.files) == ["id", "label", "log_prob", "prediction"]
        for k in a.files:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


# ------------------------------------------------------------------------------------------------------------
# a realistic size
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", ["patch", "hybrid"])
def test_realistic_size_forward_against_oracle(stem, monkeypatch):
    """8 questions x 5 candidates x 6 frames of 192 x 352 (67 viz tokens per frame), texts of 128 tokens: B = 40,
    Sj = 6 * 67 + 128 = 530; merlot.yaml widths (ViT-B, 12 joint layers), questions holding 1 to 6 frames.  The eval
    forward's hidden states and logits against the oracle on the same bf16-rounded weights (bars of
    tests/test_gpu_fullsize.py: 1.5e-2 after 12 + 12 bf16 layers).  With the hybrid stem the oracle's lite_resnet50 returns
    the GPU's stem output (tests/test_gpu_vcr_train.py's rule; the stem has its own tests): its 16 GroupNorm layers in bf16
    put about 13 % into the viz tokens at this size and 1.3 % into the language rows.  The errors go to a JSON report
    ($MERLOT_VIDEO_MC_REPORT, else a fresh directory under the temporary directory; its path is printed)."""
    import sys
    from merlot_b200 import video_mc as VM
    from merlot_b200.params import ParamStore
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import bench
    base = bench.load_config().model
    cfg = dict(base, hidden_dropout_prob=0.0, num_imgs=6, num_texts=5, num_chunks_in_group=1,
               resnet_layers=[3, 4, 9] if stem == "hybrid" else [])
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    params = MO.init_params(cfg, seed=1, perturb=0.05)
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    store = ParamStore(cfg, device=DEV, task="video_mc")
    store.load_tf_dict(params)
    g = torch.Generator().manual_seed(21)
    counts = [6, 5, 4, 3, 2, 1, 6, 6]
    mask = torch.arange(6)[None] < torch.tensor(counts)[:, None]
    image = torch.rand(48, 192, 352, 3, generator=g).bfloat16().float() * mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, 50357, (40, 128), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(48, 129, (40,), generator=g)
    ids = (ids * (torch.arange(128)[None] < lens[:, None])).int()
    from merlot_b200.modeling import MerlotModel
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                    params=store, log_attention_probs=False, save_for_backward=stem == "hybrid")
    logits = VM.mc_head(m, store)
    torch.cuda.synchronize()
    assert (m.viz_chunk_length, m._dims["Pz"], m._dims["Sj"], m.B) == (67, 402, 530, 40)
    if stem == "hybrid":
        rc = m._stem.tape[-1][1]["y"].float().cpu().reshape(48, 12, 22, -1)
        monkeypatch.setattr(O, "lite_resnet50", lambda x, p, scope, layers, width=64, rnd=O._ident: rc)
    om = MIO.MultiImageOracle(cfg, params, image, ids, img_mask=mask, log_attention_probs=False)
    ref = MO.mc_head_train(om, params, 5)
    rep = {"dims": dict(questions=8, choices=5, frames=6, B=40, N=48, vcl=67, Pz=402, Sj=530, L=128), "stem": stem}
    rep["hidden_lang_rel"] = rel(m.encoder_hidden_states["lang"], om.encoder_hidden_states["lang"])
    v = om.is_valid
    rep["hidden_valid_tokens_rel"] = rel(m.encoder_info["hidden_state"].cpu()[v], om.encoder_info["hidden_state"][v])
    rep["logits_rel"] = rel(logits, ref)
    rep["logits_max_abs"] = float((logits.float().cpu() - ref).abs().max())
    path = os.environ.get("MERLOT_VIDEO_MC_REPORT") or os.path.join(tempfile.mkdtemp(prefix="merlot_video_mc_"), "parity.json")
    data = json.load(open(path)) if os.path.exists(path) else {}
    data[stem] = rep
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)
    print(f"video_mc parity report ({stem}): {path}: {rep}")
    assert rep["hidden_lang_rel"] < 1.5e-2 and rep["hidden_valid_tokens_rel"] < 1.5e-2, rep
    assert rep["logits_rel"] < 1e-2, rep
