"""Open-ended video QA on the GPU (pytest -m gpu): the qa_cls head and the video_qa step (merlot_b200/video_qa.py) against
an fp32 autograd restatement on bf16-rounded weights, with the oracle drawing the very dropout masks the kernels draw; the
padding columns of the output layer, the equality of the tower's hidden layer with video_mc's, out-of-vocabulary rows and
gradient accumulation; the input pipeline against the NumPy restatement; the validator over saved checkpoints, on one and
two ranks; and a forward at a realistic size.  Bars as tests/test_gpu_video_mc.py: losses 1e-3 relative, activations 1e-2
and gradients 4e-2 relative-Frobenius.

The records helpers (`question`, `example`, `write_questions`, `text_np`) are shared with tests/test_video_qa_host.py."""
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

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O
from tests import tfrecord_writer as W
from tests import video_mc_oracle as MO
from tests import video_mc_records as MR

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOWER = "qa_cls"
OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=0, weight_decay_rate=0.01,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"], {"weight_decay_rate": 0}]])


# ------------------------------------------------------------------------------------------------------------
# records (the schema of merlot_b200/video_qa_input.py)
# ------------------------------------------------------------------------------------------------------------
def question(rng, k, num_frames, num_answers, max_question=30, vocab=1000, sizes=MR.SIZES, frames=None, oov_every=0):
    """One question as plain values: 1..num_frames frames, question tokens and an answer in [0, num_answers), or -1 for
    every question k with k % oov_every == oov_every - 1.  Set a value to None to leave its feature out."""
    n = int(rng.integers(1, num_frames + 1)) if frames is None else frames
    q = {"id": f"q-{k}",
         "frames": [W.jpeg(rng, *sizes[(3 * k + f) % len(sizes)], gray=(k % 5 == 4 and f == 0)) for f in range(n)],
         "question": rng.integers(7, vocab, int(rng.integers(0, max_question))).tolist(),
         "answer": int(rng.integers(0, num_answers))}
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


def write_questions(dirpath, counts, num_frames, num_answers, prefix="qa", seed=0, **kw):
    """Files <prefix>-000.tfrecord, ... holding counts[f] questions each; returns the questions in write order."""
    rng = np.random.default_rng(seed)
    out = []
    for f, n in enumerate(counts):
        qs = [question(rng, len(out) + i, num_frames, num_answers, **kw) for i in range(n)]
        out += qs
        W.write_records(dirpath / f"{prefix}-{f:03d}.tfrecord", [example(q) for q in qs])
    return out


def text_np(q, max_len):
    """[max_len] int32: START + question + END, int64 -> int32, truncated, padded with 0."""
    row = np.asarray([MR.START] + list(q.get("question") or []) + [MR.END], np.int64).astype(np.int32)[:max_len]
    out = np.zeros(max_len, np.int32)
    out[:len(row)] = row
    return out


# ------------------------------------------------------------------------------------------------------------
# the head restated
# ------------------------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def qa_cfg(tiny_cfg, F=3, **kw):
    return dict(dict(tiny_cfg, num_imgs=F, num_texts=1, num_chunks_in_group=1, hidden_dropout_prob=0.1), **kw)


def init_params(cfg, A, seed=1, tower_scale=3.0, encoder_scale=5.0):
    """The VCR graph's model variables of tests/video_mc_oracle.py and a qa_cls tower: classifier_mlp0 the mc_cls tower's,
    classifier_mlp1 [H/2, A] and its bias drawn from `seed`; GEMM operands rounded to bf16."""
    p = MO.init_params(cfg, seed=seed, perturb=0.05)
    g = torch.Generator().manual_seed(seed + 100)
    H2 = cfg["hidden_size"] // 2
    out = {k: v for k, v in p.items() if not k.startswith(MO.TOWER + "/")}
    out[f"{TOWER}/classifier_mlp0/kernel"] = p[f"{MO.TOWER}/classifier_mlp0/kernel"] * tower_scale
    out[f"{TOWER}/classifier_mlp0/bias"] = p[f"{MO.TOWER}/classifier_mlp0/bias"]
    out[f"{TOWER}/classifier_mlp1/kernel"] = torch.randn(H2, A, generator=g) * 0.02 * tower_scale
    out[f"{TOWER}/classifier_mlp1/bias"] = torch.randn(A, generator=g) * 0.1
    for k in out:
        if k.startswith("encoder/layer") and k.endswith("kernel"):
            out[k] = out[k] * encoder_scale
    return {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in out.items()}


def build(cfg, A, seed=1, device=DEV, **kw):
    from merlot_b200.params import ParamStore
    params = init_params(cfg, A, seed=seed, **kw)
    store = ParamStore(cfg, device=device, optimizer_cfg=OCFG, task="video_qa", num_answers=A)
    store.load_tf_dict(params)
    return params, store


def qa_hook(seed, p):
    """MO.dropout_hook(seed, p) that also serves the qa tower's keys ("qa", "input" | "hidden")."""
    from merlot_b200 import modeling as M
    base = MO.dropout_hook(seed, p)

    def hook(key, x):
        if key[0] != "qa":
            return base(key, x)
        if p == 0.0:
            return x
        site = {"input": M._SITE_QA_IN, "hidden": M._SITE_QA_HID}[key[1]]
        keep = torch.from_numpy(DM.counter_dropout_keep(int(seed), site, x.shape[0], x.shape[1], float(p)))
        return x * (keep.to(x.dtype) * float(DM.dropout_scale(p)))

    return hook


def head_oracle(first, p, dropout=None):
    """The tower on the first language rows [b, H] -> fp32 logits [b, A]."""
    x = first if dropout is None else dropout(("qa", "input"), first)
    h = O.dense(x, p, f"{TOWER}/classifier_mlp0", O.gelu)
    if dropout is not None:
        h = dropout(("qa", "hidden"), h)
    return O.dense(h, p, f"{TOWER}/classifier_mlp1")


def ce_in_vocab(logits, target):
    """Mean softmax cross entropy over the rows whose target is >= 0, in the dtype of the logits."""
    keep = target >= 0
    return torch.nn.functional.cross_entropy(logits[keep], target[keep].long())


def batch(cfg, b, A, L=16, hw=(64, 96), seed=0, counts=None, oov=()):
    """b questions: images [b*F] (zeros in empty slots), img_mask [b, F], ids [b, L], targets [b] (-1 at rows `oov`)."""
    F = cfg["num_imgs"]
    g = torch.Generator().manual_seed(seed)
    counts = counts or [F - i % F for i in range(b)]
    mask = torch.arange(F)[None] < torch.tensor(counts)[:, None]
    image = torch.rand(b * F, *hw, 3, generator=g).bfloat16().float() * mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, cfg["vocab_size"], (b, L), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(L // 2, L + 1, (b,), generator=g)
    ids = (ids * (torch.arange(L)[None] < lens[:, None])).int()
    target = torch.randint(0, A, (b,), generator=g).int()
    target[list(oov)] = -1
    return image, mask, ids, target


def neat(cfg, A, **opt):
    from merlot_b200.config import NeatConfig
    return NeatConfig.from_dict({"data": {}, "model": dict(cfg, image_size=[64, 96]), "optimizer": dict(OCFG, **opt),
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_video_qa"},
                                 "downstream": {"task": "video_qa", "num_answers": A}})


def feats_of(image, mask, ids, target):
    return {"images": image.to(DEV).bfloat16(), "img_mask": mask.to(DEV), "lm_input": ids.to(DEV), "lm_targets": target.to(DEV)}


def _first_rows(m):
    """Row P*F of every sequence of the GPU model's joint hidden state, fp32 on the host, as an autograd leaf."""
    P = m.encoder_pieces[1]["start"]
    return m.encoder_info["hidden_state"][:, P, :].float().cpu().clone().requires_grad_(True), P


def _tower_grads_match(store, leaf, A):
    grads = store.to_tf_dict("g")
    for k in ("classifier_mlp0/kernel", "classifier_mlp0/bias", "classifier_mlp1/kernel", "classifier_mlp1/bias"):
        name = f"{TOWER}/{k}"
        assert grads[name].shape == leaf[name].shape
        assert rel(grads[name], leaf[name].grad) < 4e-2, (name, rel(grads[name], leaf[name].grad))
    assert float(store.G(f"{TOWER}/classifier_mlp1/kernel")[:, A:].abs().max()) == 0.0
    assert float(store.G(f"{TOWER}/classifier_mlp1/bias")[A:].abs().max()) == 0.0


@pytest.mark.parametrize("A", [13, 1500])
@pytest.mark.parametrize("stem", ["patch", "hybrid"])
def test_training_step_against_oracle(tiny_cfg, monkeypatch, stem, A):
    """F = 3, 3 questions holding 3, 2 and 1 frames, hidden dropout 0.1 under the kernels' own masks: the joint encoder's
    language rows against the multi-image oracle, then the head (logits, loss, accuracy, every tower gradient and
    d_hidden_state) against the restated head on the GPU's first rows; then model.backward and one AdamW step keep the
    padding columns zero.  A = 13 pads the output layer to 16 columns; A = 1500 (padded to 1504) crosses K1's tile widths.
    With the hybrid stem the oracle's lite_resnet50 is a leaf holding the GPU's stem output."""
    from merlot_b200 import video_qa as VQ
    from tests import multi_image_oracle as MIO
    cfg = qa_cfg(tiny_cfg, resnet_layers=[1, 2, 1] if stem == "hybrid" else [])
    params, store = build(cfg, A)
    image, mask, ids, target = batch(cfg, 3, A, seed=3)
    seed = 2 ** 32 + 7
    fn = VQ.video_qa_model_fn_builder(neat(cfg, A), store=store, seed=seed)
    spec = fn(feats_of(image, mask, ids, target), None, "train")
    m = spec.model
    if stem == "hybrid":
        rc = m._stem.tape[-1][1]["y"].float().cpu().reshape(image.shape[0], 4, 6, -1)
        monkeypatch.setattr(O, "lite_resnet50", lambda x, p, scope, layers, width=64, rnd=O._ident: rc)
    hook = qa_hook(seed, 0.1)
    with torch.no_grad():
        om = MIO.MultiImageOracle(cfg, params, image, ids, img_mask=mask, log_attention_probs=False, dropout=hook)
    assert rel(m.encoder_hidden_states["lang"], om.encoder_hidden_states["lang"]) < 1e-2
    first, P = _first_rows(m)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items() if k.startswith(TOWER + "/")}
    ref = head_oracle(first, leaf, dropout=hook)
    ref_loss = ce_in_vocab(ref, target)
    logits = m._qa["logits"][:, :A]
    assert tuple(logits.shape) == (3, A) and rel(logits, ref) < 1e-2
    assert abs(float(spec.metrics["loss"]) - ref_loss.item()) <= 1e-3 * abs(ref_loss.item())
    want_acc = float((logits.argmax(-1).cpu() == target.long()).float().mean())
    assert float(spec.metrics["accuracy"]) == pytest.approx(want_acc, abs=1e-6)
    assert rel(logits, head_oracle(first.detach(), leaf, dropout=qa_hook(seed + 1, 0.1))) > 1e-2  # another seed's masks
    store.g.zero_()
    d_hidden = VQ.qa_head_backward(m, store)
    ref_loss.backward()
    _tower_grads_match(store, leaf, A)
    B, Sj, H = m.encoder_info["hidden_state"].shape
    dh = d_hidden.float().cpu().reshape(B, Sj, H)
    assert rel(dh[:, P], first.grad) < 4e-2
    others = torch.ones(Sj, dtype=torch.bool)
    others[P] = False
    assert float(dh[:, others].abs().max()) == 0.0
    m.backward(d_hidden_state=d_hidden)
    fn.optimizer.apply_gradients()
    assert float(store.P(f"{TOWER}/classifier_mlp1/kernel")[:, A:].abs().max()) == 0.0
    assert store.global_step == 1


def test_padding_columns_stay_zero_through_train_ops(tiny_cfg):
    """A = 13 (16 stored columns): after four train_op() steps with weight decay the padding columns of the kernel and the
    bias, of their bf16 copies and of the first Adam moment are exactly zero while the real columns have moved.  (The
    second moment of a zero gradient is AdamW's g*g + 1e-30 floor, not zero, and moves nothing.)"""
    from merlot_b200 import video_qa as VQ
    cfg = qa_cfg(tiny_cfg)
    _, store = build(cfg, 13)
    fn = VQ.video_qa_model_fn_builder(neat(cfg, 13), store=store, seed=5)
    before = store.P(f"{TOWER}/classifier_mlp1/kernel").clone()
    for s in range(4):
        fn(feats_of(*batch(cfg, 3, 13, seed=40 + s))).train_op()
    torch.cuda.synchronize()
    assert store.global_step == 4
    for name in (f"{TOWER}/classifier_mlp1/kernel", f"{TOWER}/classifier_mlp1/bias"):
        e = store.entries[name]
        for buf in (store.p, store.m, store.pb):
            t = buf[e.offset:e.offset + e.numel].view(e.shape)
            assert float(t[..., 13:].float().abs().max()) == 0.0, name
    after = store.P(f"{TOWER}/classifier_mlp1/kernel")
    assert not torch.equal(after[:, :13], before[:, :13])


class _Stand:
    """A model as the heads read it: the joint hidden state, its pieces, the store's buffers and the text count."""

    def __init__(self, model, num_texts):
        self.encoder_info = {"hidden_state": model.encoder_info["hidden_state"]}
        self.encoder_pieces, self._bufs, self.store, self.num_texts = model.encoder_pieces, model._bufs, model.store, num_texts


def test_tower_hidden_layer_is_video_mc_tower_bit_for_bit(tiny_cfg):
    """The same classifier_mlp0 weights on the same hidden state, dropout off: the qa tower's input rows and hidden layer
    equal mc_head's bit for bit (both read row P*F of every sequence through the shared tower kernels)."""
    from merlot_b200 import video_mc as VM
    from merlot_b200 import video_qa as VQ
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import ParamStore
    cfg = qa_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    params, qstore = build(cfg, 13)
    mparams = {k: v for k, v in params.items() if not k.startswith(TOWER + "/")}
    mparams.update({k.replace(TOWER, MO.TOWER): v for k, v in params.items() if "classifier_mlp0" in k})
    mparams[f"{MO.TOWER}/classifier_mlp1/kernel"] = torch.zeros(cfg["hidden_size"] // 2, 1)
    mparams[f"{MO.TOWER}/classifier_mlp1/bias"] = torch.zeros(1)
    mstore = ParamStore(dict(cfg, num_texts=4), device=DEV, optimizer_cfg=OCFG, task="video_mc")
    mstore.load_tf_dict(mparams)
    image, mask, ids, _ = batch(cfg, 8, 13, seed=6)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                    params=qstore)
    VQ.qa_head(m, qstore)
    stand = _Stand(m, 4)
    VM.mc_head(stand, mstore)  # 8 sequences read as 2 questions of 4 candidates: the same 8 rows
    assert torch.equal(m._qa["x"], stand._mc["x"]) and torch.equal(m._qa["h"], stand._mc["h"])
    assert torch.equal(m._qa["gp"], stand._mc["gp"]) and float(m._qa["h"].float().abs().max()) > 0


def test_oov_rows_in_an_eval_batch(tiny_cfg):
    """Labels [a, -1, b, -1]: eval mode's loss is the mean CE over the two in-vocabulary rows, its accuracy counts the OOV
    rows wrong (over all four), and its counts are loss_sum / in_vocab 2 / correct; the head backward on the same batch
    gives the OOV rows a zero gradient and the tower the gradient of the in-vocabulary mean."""
    from merlot_b200 import video_qa as VQ
    A = 13
    cfg = qa_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    params, store = build(cfg, A)
    fn = VQ.video_qa_model_fn_builder(neat(cfg, A), store=store)
    image, mask, ids, target = batch(cfg, 4, A, seed=7, oov=(1, 3))
    spec = fn(feats_of(image, mask, ids, target), None, "eval")
    lg = spec.metrics["logits"].double().cpu()
    assert tuple(lg.shape) == (4, A)
    ref = ce_in_vocab(lg, target)
    assert float(spec.metrics["loss"]) == pytest.approx(float(ref), rel=1e-5)
    per = torch.nn.functional.cross_entropy(lg, target.clamp(min=0).long(), reduction="none")
    assert float(spec.metrics["loss_sum"]) == pytest.approx(float(per[[0, 2]].sum()), rel=1e-5)
    assert float(spec.metrics["in_vocab"]) == 2.0
    right = (lg.argmax(-1) == target.long()) & (target >= 0)
    assert float(spec.metrics["correct"]) == float(right.sum())
    assert float(spec.metrics["accuracy"]) == pytest.approx(float(right.sum()) / 4, abs=1e-7)
    m = spec.model
    first, P = _first_rows(m)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items() if k.startswith(TOWER + "/")}
    ce_in_vocab(head_oracle(first, leaf), target).backward()
    store.g.zero_()
    d_hidden = VQ.qa_head_backward(m, store)
    _tower_grads_match(store, leaf, A)
    B, Sj, H = m.encoder_info["hidden_state"].shape
    dh = d_hidden.float().cpu().reshape(B, Sj, H)
    assert float(dh[[1, 3]].abs().max()) == 0.0 and float(dh[[0, 2], P].abs().max()) > 0
    assert rel(dh[:, P], first.grad) < 4e-2


def test_accumulation_matches_the_whole_batch(tiny_cfg):
    """A = 2 micro-batches of 2 questions against one batch of 4, dropout off: the same loss and the same gradient handed
    to AdamW."""
    from merlot_b200 import video_qa as VQ
    from tests.test_gpu_accumulation import capture_applied_gradient
    cfg = qa_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    micro = [feats_of(*batch(cfg, 2, 13, seed=30 + j)) for j in range(2)]
    whole = {k: torch.cat([f[k] for f in micro], 0) for k in micro[0]}
    grads, losses = [], []
    for feats in (micro, whole):
        _, store = build(cfg, 13)
        fn = VQ.video_qa_model_fn_builder(neat(cfg, 13), store=store)
        seen = capture_applied_gradient(fn, store)
        spec = fn(feats)
        spec.train_op()
        torch.cuda.synchronize()
        assert store.global_step == 1
        grads.append(torch.cat([v.reshape(-1) for v in seen.values()]))
        losses.append(float(spec.metrics["loss"]))
    print(f"video_qa A=2 x 2 vs 1 x 4: loss {losses[0]:.6f} vs {losses[1]:.6f}, gradient {rel(grads[0], grads[1]):.2e}")
    assert abs(losses[0] - losses[1]) <= 1e-4 * abs(losses[1])
    assert rel(grads[0], grads[1]) <= 1e-3


# ------------------------------------------------------------------------------------------------------------
# input pipeline and validator
# ------------------------------------------------------------------------------------------------------------
OUT = (48, 64)
A_SMALL = 11


def _u8(jpg):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(jpg)).convert("RGB"))


def _config(tmp_path, tiny_cfg, val="val-*.tfrecord", F=3, **device):
    model = dict(tiny_cfg, num_imgs=F, num_texts=1, num_chunks_in_group=1, image_size=list(OUT), vocab_size=1000,
                 max_position_embeddings=64, hidden_dropout_prob=0.1, transpose_input=True)
    d = {"data": {"train_file": str(tmp_path / "train-*.tfrecord"), "val_file": str(tmp_path / val), "num_threads": 2,
                  "shuffle_buffer_size": 4},
         "model": model, "optimizer": dict(OCFG, num_train_steps=4),
         "device": dict({"use_tpu": False, "output_dir": str(tmp_path / "out"), "train_batch_size": 2, "val_batch_size": 3,
                         "iterations_per_loop": 2}, **device),
         "downstream": {"task": "video_qa", "max_text_len": 40, "num_answers": A_SMALL},
         "validate": {"eval_samples": 7, "eval_timeout": 0}}
    path = tmp_path / f"qa_{val[:3]}.yaml"
    path.write_text(yaml.safe_dump(d))
    from merlot_b200.config import NeatConfig
    return str(path), NeatConfig.from_dict(d)


def _check_batch(batch, qs, plan, F, draws=None):
    from tests import input_oracle as IO
    from tests import story_records as SR
    from tests.test_gpu_sort_story import _check_bilinear
    b = len(batch["id"])
    assert batch["images"].shape == (b * F, *OUT, 3) and batch["images"].dtype == torch.bfloat16
    assert batch["lm_input"].shape == (b, 40) and batch["img_mask"].shape == (b, F) and batch["lm_targets"].shape == (b,)
    imgs = batch["images"].float().cpu().numpy()
    for i, rid in enumerate(batch["id"]):
        q = qs[rid]
        np.testing.assert_array_equal(batch["lm_input"][i].cpu().numpy(), text_np(q, 40))
        np.testing.assert_array_equal(batch["img_mask"][i].cpu().numpy(), [f < len(q["frames"]) for f in range(F)])
        assert int(batch["lm_targets"][i]) == (-1 if q.get("answer") is None else q["answer"])
        for f in range(F):
            s = i * F + f
            if f >= len(q["frames"]):
                assert float(np.abs(imgs[s]).max()) == 0.0, (rid, f)
                continue
            u8 = _u8(q["frames"][f])
            if draws is None:
                sh, sw, oy, ox = SR.eval_plan(u8.shape[0], u8.shape[1], OUT)
                ref = IO.bf16_round(IO.resize_and_pad(u8.astype(np.float32) * IO.INV255, OUT, sh, sw, oy, ox, 0))
            else:
                assert plan["scale"][s] == draws["scale"][i] and plan["u_y"][s] == draws["u_y"][i]
                ref, want = IO.load_and_resize_img(u8, OUT, draws["scale"][i], draws["u_y"][i], draws["u_x"][i], 0, 0,
                                                   np.ones(3, np.float32))
                assert tuple(int(plan[n][s]) for n in ("scaled_h", "scaled_w", "offset_y", "offset_x")) == want
            _check_bilinear(imgs[s], ref, f"{rid} frame {f}")


def test_pipelines_match_the_restatement(tmp_path, tiny_cfg):
    """Training batches hold no OOV question and count the ones they skip; evaluation batches keep them (label -1); every
    field and pixel matches the restatement."""
    from merlot_b200 import video_qa_input as QI
    train_qs = {q["id"]: q for q in write_questions(tmp_path, [4, 3], 3, A_SMALL, prefix="train", seed=1, oov_every=3)}
    val = write_questions(tmp_path, [4, 3], 3, A_SMALL, prefix="val", seed=2, oov_every=3)
    _, config = _config(tmp_path, tiny_cfg)
    with QI.input_fn_builder(config, is_training=True, seed=4, batch_size=2) as pipe:
        for _ in range(4):
            b = next(pipe)
            torch.cuda.synchronize()
            assert (b["lm_targets"] >= 0).all()
            _check_batch(b, train_qs, pipe.last_info["plan"], 3, pipe.last_info["draws"])
        assert pipe.skipped > 0
    seen = []
    with QI.input_fn_builder(config, is_training=False) as pipe:
        for b in pipe:
            torch.cuda.synchronize()
            _check_batch(b, {q["id"]: q for q in val}, None, 3)
            seen += b["id"]
        assert pipe.dropped == 1
    assert seen == ["q-0", "q-4", "q-1", "q-5", "q-2", "q-6"]
    assert sorted(q["id"] for q in val if q["answer"] == -1) == ["q-2", "q-5"]  # evaluated, not skipped


def _in_memory(config, store, labelled=True):
    """{accuracy, loss, questions, oov, logits, id} of the first eval_samples // val_batch_size batches, evaluated in this
    process on `store` as it is, one batch per forward, reduced on the host in float64."""
    from merlot_b200 import video_qa_input as QI
    from merlot_b200.video_qa import video_qa_model_fn_builder
    fn = video_qa_model_fn_builder(config, store=store)
    b = config.device["val_batch_size"]
    n = config.validate["eval_samples"] // b
    sums = {"loss_sum": 0.0, "in_vocab": 0.0, "correct": 0.0}
    logits, ids = [], []
    with torch.no_grad(), QI.input_fn_builder(config, is_training=False, labelled=labelled) as pipe:
        for _, batch in zip(range(n), pipe):
            spec = fn({k: batch[k] for k in ("images", "img_mask", "lm_input", "lm_targets")}, None,
                      "eval" if labelled else "predict")
            if labelled:
                for k in sums:
                    sums[k] += float(spec.metrics[k])
            logits.append(spec.metrics["logits"].float().cpu().numpy())
            ids += batch["id"]
    return {"accuracy": sums["correct"] / (n * b), "loss": sums["loss_sum"] / sums["in_vocab"], "questions": n * b,
            "oov": n * b - int(sums["in_vocab"]), "logits": np.concatenate(logits), "id": ids}


def test_save_resume_and_validate(tmp_path, tiny_cfg, capsys):
    """The trainer on records (with OOV questions, which it skips) writes checkpoints 2 and 4; the validator follows them
    and its results lines equal the in-memory evaluation of each restored checkpoint; --chunk gives the same numbers;
    --predictions holds id, label, prediction and the top-5 answers with their log-probabilities; --unlabelled runs no CE
    and writes no line.  A restored checkpoint saves back bit for bit, with the tower's [H/2, A] and [A] shapes."""
    from merlot_b200 import ops, train
    from merlot_b200 import vcr_validate as VV
    from merlot_b200 import video_qa_validate as QV
    from merlot_b200.params import ParamStore
    from merlot_b200.tf_checkpoint import load_checkpoint
    write_questions(tmp_path, [3, 3], 3, A_SMALL, prefix="train", seed=4, oov_every=4)
    val = write_questions(tmp_path, [5, 3], 3, A_SMALL, prefix="val", seed=5, oov_every=3)
    path, config = _config(tmp_path, tiny_cfg)
    train.main([path])
    assert "training on synthetic batches" not in capsys.readouterr().out
    out = tmp_path / "out"
    ckpts = [str(out / "model.ckpt-2"), str(out / "model.ckpt-4")]
    saved = load_checkpoint(ckpts[1])
    assert tuple(saved[f"{TOWER}/classifier_mlp1/kernel"].shape) == (64, A_SMALL)
    assert tuple(saved[f"{TOWER}/classifier_mlp1/bias"].shape) == (A_SMALL,)
    clock = iter(range(10 ** 6))
    res = QV.main([path], clock=lambda: next(clock), sleep=lambda s: None)
    lines = [json.loads(x) for x in (out / "eval" / "results.jsonl").read_text().splitlines()]
    assert [r["global_step"] for r in res] == [x["global_step"] for x in lines] == [2, 4]
    assert all(set(x) == {"global_step", "accuracy", "loss", "questions", "oov"} for x in lines)
    chunked = QV.main([path, "--chunk", "2", "--poll-interval", "0"], clock=lambda: next(clock), sleep=lambda s: None)

    def store_at(prefix):
        st = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer, task="video_qa", num_answers=A_SMALL)
        st.restore_checkpoint(prefix)
        return st
    for prefix, r, c in zip(ckpts, res, chunked):
        mem = _in_memory(config, store_at(prefix))
        assert r["questions"] == mem["questions"] == 6 and r["oov"] == mem["oov"] == 2
        assert r["accuracy"] == pytest.approx(mem["accuracy"], abs=1e-9) and r["loss"] == pytest.approx(mem["loss"], rel=1e-6)
        assert c["oov"] == r["oov"] and c["accuracy"] == pytest.approx(r["accuracy"], abs=1e-9)
        assert c["loss"] == pytest.approx(r["loss"], rel=2e-3)
    a = store_at(ckpts[1])
    a.save_checkpoint(str(tmp_path / "again"))
    b = store_at(str(tmp_path / "again"))
    assert b.global_step == 4 and torch.equal(a.p, b.p) and torch.equal(a.m, b.m) and torch.equal(a.v, b.v)
    resumed = dict(yaml.safe_load(open(path)), optimizer=dict(OCFG, num_train_steps=5))
    rpath = tmp_path / "resume.yaml"
    rpath.write_text(yaml.safe_dump(resumed))
    train.main([str(rpath)])
    assert "restored" in capsys.readouterr().out and (out / "model.ckpt-5.index").exists()
    QV.main([path, "--checkpoint", ckpts[1], "--predictions", str(tmp_path / "p.npz")])
    mem = _in_memory(config, store_at(ckpts[1]))
    by_id = {q["id"]: q for q in val}
    with np.load(tmp_path / "p.npz") as z:
        assert sorted(z.files) == ["id", "label", "prediction", "top_k", "top_k_log_prob"]
        assert list(z["id"]) == mem["id"] == ["q-0", "q-5", "q-1", "q-6", "q-2", "q-7"]
        assert list(z["label"]) == [by_id[i]["answer"] for i in mem["id"]] and -1 in list(z["label"])
        lp = VV.log_softmax(mem["logits"])
        assert z["top_k"].shape == z["top_k_log_prob"].shape == (6, 5)
        np.testing.assert_array_equal(z["top_k"], np.argsort(-lp, axis=1, kind="stable")[:, :5])
        np.testing.assert_allclose(z["top_k_log_prob"], np.take_along_axis(lp, z["top_k"], 1), atol=1e-6)
        assert (z["prediction"] == lp.argmax(-1)).all() and (np.diff(z["top_k_log_prob"], axis=1) <= 0).all()
        labelled = {k: z[k] for k in z.files}
    for q in val:
        q["answer"] = None
    W.write_records(tmp_path / "unl-000.tfrecord", [example(q) for q in val[:5]])
    W.write_records(tmp_path / "unl-001.tfrecord", [example(q) for q in val[5:]])
    upath, _ = _config(tmp_path, tiny_cfg, val="unl-*.tfrecord")
    calls = []
    real = ops.softmax_ce_fwd
    ops.softmax_ce_fwd = lambda *a, **k: (calls.append(1), real(*a, **k))[1]
    try:
        (res_u,) = QV.main([upath, "--checkpoint", ckpts[1], "--predictions", str(tmp_path / "u.npz"), "--unlabelled"])
    finally:
        ops.softmax_ce_fwd = real
    assert calls == [] and res_u["accuracy"] is None and res_u["loss"] is None
    with np.load(tmp_path / "u.npz") as z:
        assert (z["label"] == -1).all()
        for k in ("top_k", "top_k_log_prob", "prediction", "id"):
            np.testing.assert_array_equal(z[k], labelled[k])
    assert len((out / "eval" / "results.jsonl").read_text().splitlines()) == 5


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
        from merlot_b200 import video_qa_validate as QV
        clock = iter(range(10 ** 6))
        followed = QV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
        single = QV.main([path, "--checkpoint", checkpoint, "--predictions", predictions])
        q.put({"rank": rank, "out": (followed, single)})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="two-rank validation needs two GPUs")
def test_validation_on_two_ranks_matches_one_process(tmp_path, tiny_cfg):
    """Two processes on two GPUs write the same results lines and predictions file as one, bit for bit."""
    import torch.multiprocessing as mp
    from merlot_b200 import train
    from merlot_b200 import video_qa_validate as QV
    write_questions(tmp_path, [3, 3], 3, A_SMALL, prefix="train", seed=4)
    write_questions(tmp_path, [5, 3, 4], 3, A_SMALL, prefix="val", seed=5, oov_every=3)
    path, _ = _config(tmp_path, tiny_cfg, val_batch_size=2)
    train.main([path])
    out = tmp_path / "out"
    ckpt = str(out / "model.ckpt-4")
    results = out / "eval" / "results.jsonl"
    clock = iter(range(10 ** 6))
    one = QV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
    one += QV.main([path, "--checkpoint", ckpt, "--predictions", str(tmp_path / "one.npz")])
    one_lines = results.read_text()
    results.unlink()
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
        for k in a.files:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


# ------------------------------------------------------------------------------------------------------------
# a realistic size
# ------------------------------------------------------------------------------------------------------------
def test_realistic_size_forward_against_oracle():
    """8 questions x 6 frames of 192 x 352 (67 viz tokens per frame), 64-token texts, A = 1500 answers: Sj = 6 * 67 + 64
    = 466; merlot.yaml widths (ViT-B, 12 joint layers), questions holding 1 to 6 frames.  The eval forward's language rows
    and logits against the oracle on the same bf16-rounded weights (tests/test_gpu_fullsize.py's 1.5e-2 for the hidden
    states after 12 + 12 bf16 layers, 1e-2 for the logits)."""
    import sys
    from merlot_b200 import video_qa as VQ
    from merlot_b200.modeling import MerlotModel
    from tests import multi_image_oracle as MIO
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import bench
    base = bench.load_config().model
    cfg = dict(base, hidden_dropout_prob=0.0, num_imgs=6, num_texts=1, num_chunks_in_group=1, resnet_layers=[])
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    params, store = build(cfg, 1500, tower_scale=1.0, encoder_scale=1.0)
    g = torch.Generator().manual_seed(21)
    counts = [6, 5, 4, 3, 2, 1, 6, 6]
    mask = torch.arange(6)[None] < torch.tensor(counts)[:, None]
    image = torch.rand(48, 192, 352, 3, generator=g).bfloat16().float() * mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, 50357, (8, 64), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(24, 65, (8,), generator=g)
    ids = (ids * (torch.arange(64)[None] < lens[:, None])).int()
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                    params=store, log_attention_probs=False, save_for_backward=False)
    logits = VQ.qa_head(m, store)
    torch.cuda.synchronize()
    assert (m.viz_chunk_length, m._dims["Sj"], m.B) == (67, 466, 8) and tuple(logits.shape) == (8, 1500)
    with torch.no_grad():
        om = MIO.MultiImageOracle(cfg, params, image, ids, img_mask=mask, log_attention_probs=False)
        ref = head_oracle(om.encoder_hidden_states["lang"][:, 0, :], params)
    rep = {"hidden_lang_rel": rel(m.encoder_hidden_states["lang"], om.encoder_hidden_states["lang"]),
           "logits_rel": rel(logits, ref), "logits_max_abs": float((logits.float().cpu() - ref).abs().max())}
    path = os.environ.get("MERLOT_VIDEO_QA_REPORT") or os.path.join(tempfile.mkdtemp(prefix="merlot_video_qa_"), "parity.json")
    with open(path, "w") as f:
        json.dump(rep, f, indent=1, sort_keys=True)
    print(f"video_qa parity report: {path}: {rep}")
    assert rep["hidden_lang_rel"] < 1.5e-2 and rep["logits_rel"] < 1e-2, rep
