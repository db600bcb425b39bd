"""Fill-in-the-blank video QA on the GPU (pytest -m gpu): the video_fib head and step (merlot_b200/video_fib.py) against an
fp32 autograd restatement on bf16-rounded weights -- the oracle's lm_head (oracle/merlot_oracle.py: projection, gelu,
LayerNorm) followed by a dense layer over the A answers, on the multi-image oracle's joint encoder with the kernels' own
dropout masks; the zero-shot identity with MerlotModel.lm_head; the answer layer derived from a pretraining checkpoint and
restored, not re-derived, from a video_fib one; padding columns, out-of-vocabulary rows, gradient accumulation and
clipping; the input pipeline against the NumPy restatement; the validator over saved checkpoints, zero-shot, on one and
two ranks; and a forward at a realistic size.  Bars as tests/test_gpu_video_qa.py: losses 1e-3 relative, activations 1e-2
and gradients 4e-2 relative-Frobenius."""
import json
import os
import tempfile
import traceback

import numpy as np
import pytest
import torch
import yaml

from oracle import merlot_oracle as O
from tests import video_fib_records as FR
from tests import video_mc_oracle as MO

pytestmark = pytest.mark.gpu
DEV = "cuda"
ANS = "fib_cls/answers"
HEAD = ("lm_head/projection/kernel", "lm_head/projection/bias", "lm_head/LayerNorm/gamma", "lm_head/LayerNorm/beta",
        f"{ANS}/kernel", f"{ANS}/bias")
OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=0, weight_decay_rate=0.01,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"], {"weight_decay_rate": 0}]])


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def fib_cfg(tiny_cfg, F=3, **kw):
    return dict(dict(tiny_cfg, num_imgs=F, num_texts=1, num_chunks_in_group=1, hidden_dropout_prob=0.1), **kw)


def init_params(cfg, A, seed=1, encoder_scale=5.0):
    """The VCR graph's model variables of tests/video_mc_oracle.py, lm_head/projection and LayerNorm drawn from `seed`, and
    fib_cls/answers [H, A] drawn too; GEMM operands rounded to bf16."""
    p = MO.init_params(cfg, seed=seed, perturb=0.05)
    g = torch.Generator().manual_seed(seed + 100)
    H = cfg["hidden_size"]
    out = {k: v for k, v in p.items() if not k.startswith(MO.TOWER + "/")}
    out["lm_head/projection/kernel"] = torch.randn(H, H, generator=g) * 0.1
    out["lm_head/projection/bias"] = torch.randn(H, generator=g) * 0.1
    out["lm_head/LayerNorm/gamma"] = 1.0 + torch.randn(H, generator=g) * 0.1
    out["lm_head/LayerNorm/beta"] = torch.randn(H, generator=g) * 0.1
    out[f"{ANS}/kernel"] = torch.randn(H, A, generator=g) * 0.1
    out[f"{ANS}/bias"] = torch.randn(A, generator=g) * 0.1
    for k in out:
        if k.startswith("encoder/layer") and k.endswith("kernel"):
            out[k] = out[k] * encoder_scale
    return {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in out.items()}


def build(cfg, A, seed=1, **kw):
    from merlot_b200.params import ParamStore
    params = init_params(cfg, A, seed=seed, **kw)
    store = ParamStore(cfg, device=DEV, optimizer_cfg=OCFG, task="video_fib", num_answers=A)
    store.load_tf_dict(params)
    return params, store


def head_oracle(rows, p):
    """lm_head's projection (oracle/merlot_oracle.py MerlotOracle.lm_head) then the answer layer: fp32 logits [b, A]."""
    h = O.layer_norm(O.dense(rows, p, "lm_head/projection", O.gelu), p, "lm_head/LayerNorm")
    return O.dense(h, p, ANS)


def ce_in_vocab(logits, target):
    keep = target >= 0
    return torch.nn.functional.cross_entropy(logits[keep], target[keep].long())


def batch(cfg, b, A, L=16, hw=(64, 96), seed=0, counts=None, oov=()):
    """b questions: images [b*F] (zeros in empty slots), img_mask [b, F], ids [b, L] with one MASK among the words,
    blank positions [b], targets [b] (-1 at rows `oov`)."""
    F = cfg["num_imgs"]
    g = torch.Generator().manual_seed(seed)
    counts = counts or [F - i % F for i in range(b)]
    mask = torch.arange(F)[None] < torch.tensor(counts)[:, None]
    image = torch.rand(b * F, *hw, 3, generator=g).bfloat16().float() * mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, cfg["vocab_size"], (b, L), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(L // 2, L + 1, (b,), generator=g)
    ids = (ids * (torch.arange(L)[None] < lens[:, None])).int()
    blank = 1 + (torch.rand(b, generator=g) * (lens - 1)).long()
    ids[torch.arange(b), blank] = FR.MASK
    target = torch.randint(0, A, (b,), generator=g).int()
    target[list(oov)] = -1
    return image, mask, ids, blank.int(), target


def answers_file(A, max_tokens=1, seed=0, vocab=1000):
    path = os.path.join(tempfile.mkdtemp(prefix="merlot_fib_answers_"), "answers.json")
    ans = FR.answers(np.random.default_rng(seed), A, vocab=vocab, max_tokens=max_tokens)
    return FR.write_answers(path, ans), ans


def neat(cfg, A, answers=None, **opt):
    from merlot_b200.config import NeatConfig
    path = answers or answers_file(A)[0]
    return NeatConfig.from_dict({"data": {}, "model": dict(cfg, image_size=[64, 96]), "optimizer": dict(OCFG, **opt),
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_video_fib"},
                                 "downstream": {"task": "video_fib", "answer_tokens": path}})


def feats_of(image, mask, ids, blank, target, with_blank=True):
    f = {"images": image.to(DEV).bfloat16(), "img_mask": mask.to(DEV), "lm_input": ids.to(DEV), "lm_targets": target.to(DEV)}
    if with_blank:
        f["blank_pos"] = blank.to(DEV)
    return f


def _blank_rows(m, blank):
    """The GPU model's joint hidden state at the blank rows, fp32 on the host, as an autograd leaf; and P * F."""
    P = m.encoder_pieces[1]["start"]
    hs = m.encoder_info["hidden_state"]
    rows = hs[torch.arange(hs.shape[0], device=hs.device), P + blank.long().to(hs.device)]
    return rows.float().cpu().clone().requires_grad_(True), P


@pytest.mark.parametrize("A,derived", [(13, False), (1500, True)])
@pytest.mark.parametrize("stem", ["patch", "hybrid"])
def test_training_step_against_oracle(tiny_cfg, monkeypatch, stem, A, derived):
    """F = 3, 3 questions holding 3, 2 and 1 frames, hidden dropout 0.1 under the kernels' own masks: logits, loss,
    accuracy, every lm_head and fib_cls gradient and every encoder gradient against the oracle; d_hidden_state is non-zero
    at the blank rows only.  A = 13 pads the answer layer to 16 columns; A = 1500 (1504 stored) uses an answer layer
    derived from 1..4-token answers and a random output bias.  With the hybrid stem the oracle's lite_resnet50 is a leaf
    holding the GPU's stem output."""
    from merlot_b200 import video_fib as VF
    from merlot_b200.params import derive_fib_answers
    from tests import multi_image_oracle as MIO
    cfg = fib_cfg(tiny_cfg, resnet_layers=[1, 2, 1] if stem == "hybrid" else [])
    params, store = build(cfg, A)
    path, ans = answers_file(A, max_tokens=4 if derived else 1, seed=A)
    if derived:
        derive_fib_answers(store, ans, torch.randn(cfg["vocab_size"], generator=torch.Generator().manual_seed(9)))
        d = store.to_tf_dict()
        params[f"{ANS}/kernel"], params[f"{ANS}/bias"] = d[f"{ANS}/kernel"].bfloat16().float(), d[f"{ANS}/bias"]
    image, mask, ids, blank, target = batch(cfg, 3, A, seed=3)
    seed = 2 ** 32 + 7
    fn = VF.video_fib_model_fn_builder(neat(cfg, A, path), store=store, seed=seed)
    spec = fn(feats_of(image, mask, ids, blank, target), None, "train")
    m = spec.model
    if stem == "hybrid":
        rc = m._stem.tape[-1][1]["y"]
        N, hs, ws = image.shape[0], 64 // 16, 96 // 16
        leaf_rc = rc.float().cpu().reshape(N, hs, ws, rc.shape[1]).clone().requires_grad_(True)
        monkeypatch.setattr(O, "lite_resnet50", lambda x, p, scope, layers, width=64, rnd=O._ident: leaf_rc)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    om = MIO.MultiImageOracle(cfg, leaf, image, ids, img_mask=mask, log_attention_probs=False,
                              dropout=MO.dropout_hook(seed, 0.1))
    assert rel(m.encoder_hidden_states["lang"], om.encoder_hidden_states["lang"]) < 1e-2
    # the head alone, on the GPU's blank rows
    rows, P = _blank_rows(m, blank)
    head_leaf = {k: v.detach().clone().requires_grad_(True) for k, v in params.items() if k in HEAD}
    ref = head_oracle(rows, head_leaf)
    ref_loss = ce_in_vocab(ref, target)
    logits = m._fib["logits"][:, :A]
    assert tuple(logits.shape) == (3, A) and rel(logits, ref) < 1e-2
    assert abs(float(spec.metrics["loss"]) - ref_loss.item()) <= 1e-3 * abs(ref_loss.item())
    want_acc = float((logits.argmax(-1).cpu() == target.long()).float().mean())
    assert float(spec.metrics["accuracy"]) == pytest.approx(want_acc, abs=1e-5)
    store.g.zero_()
    d_hidden = VF.fib_head_backward(m, store)
    ref_loss.backward()
    grads = store.to_tf_dict("g")
    for k in HEAD:
        assert grads[k].shape == head_leaf[k].shape and rel(grads[k], head_leaf[k].grad) < 4e-2, (k, rel(grads[k], head_leaf[k].grad))
    assert store.G(f"{ANS}/kernel")[:, A:].count_nonzero() == 0 and store.G(f"{ANS}/bias")[A:].count_nonzero() == 0
    B, Sj, H = m.encoder_info["hidden_state"].shape
    dh = d_hidden.float().cpu().reshape(B, Sj, H)
    at = torch.zeros(B, Sj, dtype=torch.bool)
    at[torch.arange(B), P + blank.long()] = True
    assert rel(dh[at], rows.grad) < 4e-2 and float(dh[~at].abs().max()) == 0.0
    # the whole graph: every parameter gradient against the oracle's
    m.backward(d_hidden_state=d_hidden)
    lang = om.encoder_hidden_states["lang"]
    full_loss = ce_in_vocab(head_oracle(lang[torch.arange(B), blank.long()], leaf), target)
    full_loss.backward()
    grads = store.to_tf_dict("g")
    assert set(grads) == set(leaf)
    worst = {k: rel(grads[k], v.grad) for k, v in leaf.items()
             if "resnet50lite" not in k and v.grad is not None and float(v.grad.norm()) >= 1e-7}
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    for k in HEAD + ("vision_backbone/img_idx_pe", "encoder/layer00/query_layer/kernel", "word_embeddings/word_embeddings"):
        assert k in worst, k
    if stem == "hybrid":
        vals = sorted(worst.values())
        assert len(worst) > 40 and max(vals) < 6e-2 and vals[len(vals) // 2] < 2.5e-2, top
        assert rel(m.d_rc, leaf_rc.grad.reshape(N * hs * ws, -1)) < 4e-2
    else:
        assert len(worst) > 40 and max(worst.values()) < 4e-2, top
    fn.optimizer.apply_gradients()
    assert float(store.P(f"{ANS}/kernel")[:, A:].abs().sum()) == 0.0 and store.global_step == 1


@pytest.mark.parametrize("do_bias", [False, True])
def test_zero_shot_identity_with_the_mlm_head(tiny_cfg, do_bias):
    """Freshly derived weights, one-token answers: the FiB logits equal the answer tokens' columns of
    MerlotModel.lm_head (modeling.py) at the blank rows, plus the output bias at those tokens with do_bias.  The two
    products read the same bf16 operands but K1 may choose another tile width or split-K at N = A8 than at N = vocab, so
    the bar is 1e-5 of the largest logit; on an H100 80GB HBM3 at 700 W the measured largest difference is 0 with and
    without the bias: the same bits."""
    from merlot_b200 import video_fib as VF
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import derive_fib_answers
    A = 40
    cfg = fib_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    _, store = build(cfg, A, encoder_scale=1.0)
    _, ans = answers_file(A, seed=2)
    bias = torch.randn(cfg["vocab_size"], generator=torch.Generator().manual_seed(5)) if do_bias else None
    derive_fib_answers(store, ans, bias)
    image, mask, ids, blank, _ = batch(cfg, 6, A, seed=11)
    m = MerlotModel(dict(cfg, do_bias=False), is_training=False, use_tpu=False, image=image.to(DEV).bfloat16(),
                    input_ids=ids.to(DEV), img_mask=mask.to(DEV), mask_input=False, params=store)
    fib = VF.fib_head(m, store, blank.to(DEV)).clone()
    P = m.encoder_pieces[1]["start"]
    hs = m.encoder_info["hidden_state"]
    rows = hs[torch.arange(6, device=DEV), P + blank.long().to(DEV)].contiguous()
    mlm = m.lm_head(rows)[:, [t[0] for t in ans]].float().cpu()
    if bias is not None:
        mlm = mlm + bias[[t[0] for t in ans]][None]
    diff = ((fib.cpu() - mlm).abs().max() / mlm.abs().max()).item()
    print(f"zero-shot identity (do_bias {do_bias}): largest difference {diff:.3e} of the largest logit")
    assert diff <= 1e-5


def _pretraining_checkpoint(cfg, path, seed=7):
    """A pretraining store (init_reference(seed), a random lm_head/output_bias) saved as checkpoint `path`."""
    from merlot_b200.params import ParamStore
    pre = ParamStore(dict(cfg, num_imgs=1), device=DEV, optimizer_cfg=OCFG, task="pretrain")
    pre.init_reference(seed=seed)
    with torch.no_grad():
        pre.P("lm_head/output_bias").copy_(torch.randn(cfg["vocab_size"], generator=torch.Generator().manual_seed(seed)))
        pre.P("word_embeddings/word_embeddings").add_(torch.randn(pre.P("word_embeddings/word_embeddings").shape,
                                                                  generator=torch.Generator().manual_seed(seed + 1)).to(DEV))
    pre.sync_bf16()
    pre.global_step = 123
    pre.save_checkpoint(str(path))
    return pre


def test_init_checkpoint_restores_lm_head_and_derives_the_answers(tmp_path, tiny_cfg, capsys):
    """model.init_checkpoint of a pretraining checkpoint: lm_head/* and the embeddings restore by name, fib_cls/answers is
    the float64 mean of the restored embedding rows and output bias (multi-token answers), not its random initial value;
    then resuming from a video_fib checkpoint restores the layer exactly, whatever the store's embeddings were."""
    from merlot_b200 import video_fib as VF
    from merlot_b200.params import ParamStore
    A = 21
    cfg = fib_cfg(tiny_cfg)
    pre = _pretraining_checkpoint(cfg, tmp_path / "pre.ckpt-123")
    path, ans = answers_file(A, max_tokens=3, seed=4)
    config = neat(dict(cfg, init_checkpoint=str(tmp_path / "pre.ckpt-123")), A, path)
    fn = VF.video_fib_model_fn_builder(config)
    out = capsys.readouterr().out
    assert "2 variables not in the checkpoint" in out and "fib_cls/answers: derived" in out
    st = fn.store
    for n in ("lm_head/projection/kernel", "lm_head/projection/bias", "lm_head/LayerNorm/gamma", "lm_head/LayerNorm/beta",
              "word_embeddings/word_embeddings", "encoder/layer01/qkv/kernel"):
        assert torch.equal(st.P(n), pre.P(n)), n
    emb, ob = pre.P("word_embeddings/word_embeddings").double().cpu().numpy(), pre.P("lm_head/output_bias").double().cpu().numpy()
    kern = np.stack([emb[a].mean(0) for a in ans], 1).astype(np.float32)
    bias = np.array([ob[a].mean() for a in ans], np.float32)
    np.testing.assert_array_equal(st.P(f"{ANS}/kernel")[:, :A].cpu().numpy(), kern)
    np.testing.assert_array_equal(st.P(f"{ANS}/bias")[:A].cpu().numpy(), bias)
    assert float(st.P(f"{ANS}/kernel")[:, A:].abs().max()) == 0.0
    fresh = ParamStore(cfg, device=DEV, optimizer_cfg=OCFG, task="video_fib", num_answers=A)
    fresh.init_reference(seed=0)
    assert not torch.equal(fresh.P(f"{ANS}/kernel"), st.P(f"{ANS}/kernel"))
    # a fine-tuning step moves the layer away from its derivation; its checkpoint restores it and derives nothing
    image, mask, ids, blank, target = batch(cfg, 3, A, seed=12)
    fn(feats_of(image, mask, ids, blank, target)).train_op()
    st.save_checkpoint(str(tmp_path / "model.ckpt-1"))
    trained = st.P(f"{ANS}/kernel").clone()
    assert not torch.equal(trained[:, :A].cpu(), torch.from_numpy(kern))
    resumed = ParamStore(cfg, device=DEV, optimizer_cfg=OCFG, task="video_fib", num_answers=A)
    resumed.init_reference(seed=3)
    with torch.no_grad():
        resumed.P("word_embeddings/word_embeddings").mul_(-2.0)
    resumed.restore_checkpoint(str(tmp_path / "model.ckpt-1"))
    assert torch.equal(resumed.P(f"{ANS}/kernel"), trained) and torch.equal(resumed.p, st.p)
    # init_checkpoint of a video_fib checkpoint restores the layer by name and does not derive it either
    fn2 = VF.video_fib_model_fn_builder(neat(dict(cfg, init_checkpoint=str(tmp_path / "model.ckpt-1")), A, path))
    assert "derived" not in capsys.readouterr().out and torch.equal(fn2.store.P(f"{ANS}/kernel"), trained)


def test_padding_columns_stay_zero_through_train_ops(tiny_cfg):
    """A = 13 (16 stored columns): after four train_op() steps with weight decay the padding columns of the kernel and the
    bias, of their bf16 copies and of the first Adam moment are exactly zero while the real columns have moved."""
    from merlot_b200 import video_fib as VF
    cfg = fib_cfg(tiny_cfg)
    _, store = build(cfg, 13)
    fn = VF.video_fib_model_fn_builder(neat(cfg, 13), store=store, seed=5)
    before = store.P(f"{ANS}/kernel").clone()
    for s in range(4):
        fn(feats_of(*batch(cfg, 3, 13, seed=40 + s))).train_op()
    torch.cuda.synchronize()
    assert store.global_step == 4
    for name in (f"{ANS}/kernel", f"{ANS}/bias"):
        e = store.entries[name]
        for buf in (store.p, store.m, store.pb):
            t = buf[e.offset:e.offset + e.numel].view(e.shape)
            assert float(t[..., 13:].float().abs().max()) == 0.0, name
    assert not torch.equal(store.P(f"{ANS}/kernel")[:, :13], before[:, :13])


def test_oov_rows_and_device_blank_positions_in_an_eval_batch(tiny_cfg):
    """Labels [a, -1, b, -1]: eval mode's loss is the mean CE over the two in-vocabulary rows, its accuracy counts the OOV
    rows wrong, and its counts are loss_sum / in_vocab 2 / correct; the head backward gives the OOV rows a zero gradient.
    Without blank_pos the MASK is found on the device and the logits are the same bits."""
    from merlot_b200 import video_fib as VF
    A = 13
    cfg = fib_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    params, store = build(cfg, A)
    fn = VF.video_fib_model_fn_builder(neat(cfg, A), store=store)
    image, mask, ids, blank, target = batch(cfg, 4, A, seed=7, oov=(1, 3))
    spec = fn(feats_of(image, mask, ids, blank, target), None, "eval")
    lg = spec.metrics["logits"].double().cpu()
    again = fn(feats_of(image, mask, ids, blank, target, with_blank=False), None, "eval").metrics["logits"]
    assert torch.equal(again.cpu(), lg.float())
    assert float(spec.metrics["loss"]) == pytest.approx(float(ce_in_vocab(lg, target)), rel=1e-5)
    per = torch.nn.functional.cross_entropy(lg, target.clamp(min=0).long(), reduction="none")
    assert float(spec.metrics["loss_sum"]) == pytest.approx(float(per[[0, 2]].sum()), rel=1e-5)
    assert float(spec.metrics["in_vocab"]) == 2.0
    right = (lg.argmax(-1) == target.long()) & (target >= 0)
    assert float(spec.metrics["correct"]) == float(right.sum())
    assert float(spec.metrics["accuracy"]) == pytest.approx(float(right.sum()) / 4, abs=1e-7)
    m = spec.model
    rows, P = _blank_rows(m, blank)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items() if k in HEAD}
    ce_in_vocab(head_oracle(rows, leaf), target).backward()
    spec = fn(feats_of(image, mask, ids, blank, target), None, "eval")
    store.g.zero_()
    d_hidden = VF.fib_head_backward(spec.model, store)
    grads = store.to_tf_dict("g")
    for k in HEAD:
        assert rel(grads[k], leaf[k].grad) < 4e-2, k
    B, Sj, H = spec.model.encoder_info["hidden_state"].shape
    dh = d_hidden.float().cpu().reshape(B, Sj, H)
    assert float(dh[[1, 3]].abs().max()) == 0.0 and float(dh[[0, 2]].abs().max()) > 0


def test_accumulation_matches_the_whole_batch(tiny_cfg):
    """A = 2 micro-batches of 2 questions against one batch of 4, dropout off: the same loss and the same gradient handed
    to AdamW."""
    from merlot_b200 import video_fib as VF
    from tests.test_gpu_accumulation import capture_applied_gradient
    cfg = fib_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    micro = [feats_of(*batch(cfg, 2, 13, seed=30 + j)) for j in range(2)]
    whole = {k: torch.cat([f[k] for f in micro], 0) for k in micro[0]}
    grads, losses = [], []
    for feats in (micro, whole):
        _, store = build(cfg, 13)
        fn = VF.video_fib_model_fn_builder(neat(cfg, 13), store=store)
        seen = capture_applied_gradient(fn, store)
        spec = fn(feats)
        spec.train_op()
        torch.cuda.synchronize()
        assert store.global_step == 1
        grads.append(torch.cat([v.reshape(-1) for v in seen.values()]))
        losses.append(float(spec.metrics["loss"]))
    print(f"video_fib A=2 x 2 vs 1 x 4: loss {losses[0]:.6f} vs {losses[1]:.6f}, gradient {rel(grads[0], grads[1]):.2e}")
    assert abs(losses[0] - losses[1]) <= 1e-4 * abs(losses[1])
    assert rel(grads[0], grads[1]) <= 1e-3


def test_clipped_accumulation_is_the_mean_of_clipped_micro_batches(tiny_cfg):
    """clip_norm c between the two micro-batches' gradient norms: the gradient AdamW applies is the mean of each
    micro-batch's gradient (run alone) clipped to c."""
    from merlot_b200 import video_fib as VF
    from tests.test_gpu_clip_accumulation import capture_applied, clipped_mean, norm_of
    cfg = fib_cfg(tiny_cfg, hidden_dropout_prob=0.0)
    micro = [feats_of(*batch(cfg, 2, 13, seed=50 + j)) for j in range(2)]
    alone = []
    for f in micro:
        _, store = build(cfg, 13)
        fn = VF.video_fib_model_fn_builder(neat(cfg, 13), store=store)
        seen = capture_applied(fn, store)
        fn(f).train_op()
        torch.cuda.synchronize()
        alone.append(dict(seen))
    norms = [norm_of(g) for g in alone]
    c = (norms[0] * norms[1]) ** 0.5 if max(norms) / min(norms) > 1.02 else 0.5 * min(norms)
    _, store = build(cfg, 13)
    fn = VF.video_fib_model_fn_builder(neat(cfg, 13, clip_norm=c), store=store)
    seen = capture_applied(fn, store)
    spec = fn(micro)
    spec.train_op()
    torch.cuda.synchronize()
    want = clipped_mean(alone, norms, c)
    got, ref = (torch.cat([d[k].reshape(-1) for k in sorted(want)]) for d in (seen, want))
    got_norm = float(spec.metrics["gradnorms/_overall"])
    print(f"video_fib A=2 c={c:.4f}: norms {norms}, gradnorms/_overall {got_norm:.4f}, gradient {rel(got, ref):.2e}")
    assert store.global_step == 1 and store.g_acc is not None and rel(got, ref) <= 1e-3
    assert abs(got_norm - sum(norms) / 2) <= 1e-3 * sum(norms) / 2


# ------------------------------------------------------------------------------------------------------------
# input pipeline and validator
# ------------------------------------------------------------------------------------------------------------
OUT = (48, 64)
A_SMALL = 11


def _config(tmp_path, tiny_cfg, val="val-*.tfrecord", F=3, answers=None, **device):
    model = dict(tiny_cfg, num_imgs=F, num_texts=1, num_chunks_in_group=1, image_size=list(OUT), vocab_size=1000,
                 max_position_embeddings=64, hidden_dropout_prob=0.1, transpose_input=True)
    ans = answers or FR.answers(np.random.default_rng(8), A_SMALL)
    d = {"data": {"train_file": str(tmp_path / "train-*.tfrecord"), "val_file": str(tmp_path / val), "num_threads": 2,
                  "shuffle_buffer_size": 4},
         "model": model, "optimizer": dict(OCFG, num_train_steps=4),
         "device": dict({"use_tpu": False, "output_dir": str(tmp_path / "out"), "train_batch_size": 2, "val_batch_size": 3,
                         "iterations_per_loop": 2}, **device),
         "downstream": {"task": "video_fib", "max_text_len": 40, "answer_tokens": FR.write_answers(tmp_path / "answers.json", ans)},
         "validate": {"eval_samples": 7, "eval_timeout": 0}}
    path = tmp_path / f"fib_{val[:3]}.yaml"
    path.write_text(yaml.safe_dump(d))
    from merlot_b200.config import NeatConfig
    return str(path), NeatConfig.from_dict(d)


def _check_fib_batch(batch, qs, plan, F, draws=None):
    from tests.test_gpu_video_qa import _check_batch
    _check_batch(batch, qs, plan, F, draws)  # pixels, img_mask, lm_input (START + question + END) and lm_targets
    assert batch["blank_pos"].dtype == torch.int32 and batch["blank_pos"].shape == (len(batch["id"]),)
    for i, rid in enumerate(batch["id"]):
        assert int(batch["blank_pos"][i]) == FR.blank_np(qs[rid]) and int(batch["lm_input"][i, batch["blank_pos"][i]]) == 1


def test_pipelines_match_the_restatement(tmp_path, tiny_cfg):
    """Training batches hold no OOV question and count the ones they skip; evaluation batches keep them; every field, the
    blank positions and every pixel match the restatement."""
    from merlot_b200 import video_fib_input as FI
    train_qs = {q["id"]: q for q in FR.write_questions(tmp_path, [4, 3], 3, A_SMALL, prefix="train", seed=1, oov_every=3)}
    val = FR.write_questions(tmp_path, [4, 3], 3, A_SMALL, prefix="val", seed=2, oov_every=3)
    _, config = _config(tmp_path, tiny_cfg)
    with FI.input_fn_builder(config, is_training=True, seed=4, batch_size=2) as pipe:
        for _ in range(4):
            b = next(pipe)
            torch.cuda.synchronize()
            assert (b["lm_targets"] >= 0).all()
            _check_fib_batch(b, train_qs, pipe.last_info["plan"], 3, pipe.last_info["draws"])
        assert pipe.skipped > 0
    seen = []
    with FI.input_fn_builder(config, is_training=False) as pipe:
        for b in pipe:
            torch.cuda.synchronize()
            _check_fib_batch(b, {q["id"]: q for q in val}, None, 3)
            seen += b["id"]
        assert pipe.dropped == 1
    assert seen == ["q-0", "q-4", "q-1", "q-5", "q-2", "q-6"]


def _in_memory(config, store, labelled=True):
    """{accuracy, loss, questions, oov, logits, id} of the first eval_samples // val_batch_size batches, evaluated in this
    process on `store` as it is, one batch per forward, reduced on the host in float64."""
    from merlot_b200 import video_fib_input as FI
    from merlot_b200.video_fib import video_fib_model_fn_builder
    fn = video_fib_model_fn_builder(config, store=store)
    b = config.device["val_batch_size"]
    n = config.validate["eval_samples"] // b
    sums = {"loss_sum": 0.0, "in_vocab": 0.0, "correct": 0.0}
    logits, ids = [], []
    with torch.no_grad(), FI.input_fn_builder(config, is_training=False, labelled=labelled) as pipe:
        for _, batch in zip(range(n), pipe):
            spec = fn({k: batch[k] for k in ("images", "img_mask", "lm_input", "lm_targets", "blank_pos")}, None,
                      "eval" if labelled else "predict")
            if labelled:
                for k in sums:
                    sums[k] += float(spec.metrics[k])
            logits.append(spec.metrics["logits"].float().cpu().numpy())
            ids += batch["id"]
    return {"accuracy": sums["correct"] / (n * b), "loss": sums["loss_sum"] / max(sums["in_vocab"], 1e-30),
            "questions": n * b, "oov": n * b - int(sums["in_vocab"]), "logits": np.concatenate(logits), "id": ids}


def test_save_resume_and_validate(tmp_path, tiny_cfg, capsys):
    """The trainer on records writes checkpoints 2 and 4 with the answer layer's [H, A] and [A] shapes; the validator
    follows them and its results lines equal the in-memory evaluation of each restored checkpoint; --chunk gives the same
    numbers; --predictions holds id, label, prediction and the top-5 answers; a resumed run continues to step 5."""
    from merlot_b200 import train
    from merlot_b200 import vcr_validate as VV
    from merlot_b200 import video_fib_validate as FV
    from merlot_b200.params import ParamStore
    from merlot_b200.tf_checkpoint import load_checkpoint
    FR.write_questions(tmp_path, [3, 3], 3, A_SMALL, prefix="train", seed=4, oov_every=4)
    val = FR.write_questions(tmp_path, [5, 3], 3, A_SMALL, prefix="val", seed=5, oov_every=3)
    path, config = _config(tmp_path, tiny_cfg)
    train.main([path])
    assert "training on synthetic batches" not in capsys.readouterr().out
    out = tmp_path / "out"
    ckpts = [str(out / "model.ckpt-2"), str(out / "model.ckpt-4")]
    saved = load_checkpoint(ckpts[1])
    assert tuple(saved[f"{ANS}/kernel"].shape) == (128, A_SMALL) and tuple(saved[f"{ANS}/bias"].shape) == (A_SMALL,)
    clock = iter(range(10 ** 6))
    res = FV.main([path], clock=lambda: next(clock), sleep=lambda s: None)
    lines = [json.loads(x) for x in (out / "eval" / "results.jsonl").read_text().splitlines()]
    assert [r["global_step"] for r in res] == [x["global_step"] for x in lines] == [2, 4]
    assert all(set(x) == {"global_step", "accuracy", "loss", "questions", "oov"} for x in lines)
    chunked = FV.main([path, "--chunk", "2", "--poll-interval", "0"], clock=lambda: next(clock), sleep=lambda s: None)

    def store_at(prefix):
        st = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer, task="video_fib", num_answers=A_SMALL)
        st.restore_checkpoint(prefix)
        return st
    for prefix, r, c in zip(ckpts, res, chunked):
        mem = _in_memory(config, store_at(prefix))
        assert r["questions"] == mem["questions"] == 6 and r["oov"] == mem["oov"] == 2
        assert r["accuracy"] == pytest.approx(mem["accuracy"], abs=1e-9) and r["loss"] == pytest.approx(mem["loss"], rel=1e-6)
        assert c["oov"] == r["oov"] and c["accuracy"] == pytest.approx(r["accuracy"], abs=1e-9)
        assert c["loss"] == pytest.approx(r["loss"], rel=2e-3)
    resumed = dict(yaml.safe_load(open(path)), optimizer=dict(OCFG, num_train_steps=5))
    rpath = tmp_path / "resume.yaml"
    rpath.write_text(yaml.safe_dump(resumed))
    train.main([str(rpath)])
    assert "restored" in capsys.readouterr().out and (out / "model.ckpt-5.index").exists()
    FV.main([path, "--checkpoint", ckpts[1], "--predictions", str(tmp_path / "p.npz")])
    mem = _in_memory(config, store_at(ckpts[1]))
    by_id = {q["id"]: q for q in val}
    with np.load(tmp_path / "p.npz") as z:
        assert sorted(z.files) == ["id", "label", "prediction", "top_k", "top_k_log_prob"]
        assert list(z["id"]) == mem["id"] == ["q-0", "q-5", "q-1", "q-6", "q-2", "q-7"]
        assert list(z["label"]) == [by_id[i]["answer"] for i in mem["id"]]
        lp = VV.log_softmax(mem["logits"])
        np.testing.assert_array_equal(z["top_k"], np.argsort(-lp, axis=1, kind="stable")[:, :5])
        np.testing.assert_allclose(z["top_k_log_prob"], np.take_along_axis(lp, z["top_k"], 1), atol=1e-6)
        assert (z["prediction"] == lp.argmax(-1)).all()


def test_zero_shot_validation_of_a_pretraining_checkpoint(tmp_path, tiny_cfg):
    """--zero-shot --checkpoint <pretraining prefix>: the accuracy and loss computed from the oracle's zero-shot logits on
    the same records (the multi-image oracle's joint encoder on the restored weights, lm_head, and the answer layer derived
    in float64 from the checkpoint), global_step the checkpoint's; without --zero-shot the strict restore refuses it.  The
    records' answers are set from the oracle's own predictions (right for every other in-vocabulary question, wrong for the
    rest), so the accuracy is neither 0 nor 1."""
    from merlot_b200 import video_fib_input as FI
    from merlot_b200 import video_fib_validate as FV
    from merlot_b200.tf_checkpoint import CheckpointFormatError, load_checkpoint
    from tests import multi_image_oracle as MIO
    from tests import tfrecord_writer as W
    ans = FR.answers(np.random.default_rng(8), A_SMALL, max_tokens=2)
    val = FR.write_questions(tmp_path, [5, 3], 3, A_SMALL, prefix="val", seed=5, oov_every=3)
    path, config = _config(tmp_path, tiny_cfg, answers=ans)
    cfg = dict(config.model, hidden_dropout_prob=0.0)
    _pretraining_checkpoint(cfg, tmp_path / "pre.ckpt-123")
    prefix = str(tmp_path / "pre.ckpt-123")
    d = load_checkpoint(prefix)
    p = {k: (v.float().bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v.float())
         for k, v in d.items()}
    emb, ob = d["word_embeddings/word_embeddings"].double(), d["lm_head/output_bias"].double()
    p[f"{ANS}/kernel"] = torch.stack([emb[a].mean(0) for a in ans], 1).float().bfloat16().float()
    p[f"{ANS}/bias"] = torch.stack([ob[a].mean() for a in ans]).float()
    logits = {}
    with FI.input_fn_builder(config, is_training=False) as pipe:
        for _, b in zip(range(2), pipe):
            image = b["images"].float().cpu()
            om = MIO.MultiImageOracle(cfg, p, image, b["lm_input"].cpu(), img_mask=b["img_mask"].cpu(),
                                      log_attention_probs=False)
            lang = om.encoder_hidden_states["lang"]
            lg = head_oracle(lang[torch.arange(lang.shape[0]), b["blank_pos"].long().cpu()], p).double()
            logits.update(zip(b["id"], lg))
    for k, q in enumerate(val):  # the oracle's answer for even k, another one for odd k; OOV stays OOV
        if q["id"] in logits and q["answer"] >= 0:
            pred = int(logits[q["id"]].argmax())
            q["answer"] = pred if k % 2 == 0 else (pred + 1) % A_SMALL
    W.write_records(tmp_path / "val-000.tfrecord", [FR.example(q) for q in val[:5]])
    W.write_records(tmp_path / "val-001.tfrecord", [FR.example(q) for q in val[5:]])
    (res,) = FV.main([path, "--checkpoint", prefix, "--zero-shot"])
    with pytest.raises(CheckpointFormatError, match="variables the store needs are not in the checkpoint"):
        FV.main([path, "--checkpoint", prefix])
    by_id = {q["id"]: q for q in val}
    correct, ce, iv, close = 0, 0.0, 0, 0
    for rid, lg in logits.items():
        t = by_id[rid]["answer"]
        top2 = lg.topk(2).values
        close += int(float(top2[0] - top2[1]) < 1e-2 * float(top2.abs().max()))  # bf16 may order these two either way
        if t >= 0:
            correct += int(int(lg.argmax()) == t)
            ce += float(torch.nn.functional.cross_entropy(lg[None], torch.tensor([t])))
            iv += 1
    n = len(logits)
    print(f"zero-shot: GPU accuracy {res['accuracy']:.4f} loss {res['loss']:.5f}; oracle {correct / n:.4f} {ce / iv:.5f}; "
          f"{close} near ties")
    assert res["global_step"] == 123 and res["questions"] == n == 6 and res["oov"] == n - iv
    assert 0 < correct < iv and abs(res["accuracy"] * n - correct) <= close + 1e-9, (correct, close)
    assert res["loss"] == pytest.approx(ce / iv, rel=1e-2)


def _rank_main(rank, world, port, path, checkpoint, predictions, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    try:
        from merlot_b200 import video_fib_validate as FV
        clock = iter(range(10 ** 6))
        followed = FV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
        single = FV.main([path, "--checkpoint", checkpoint, "--predictions", predictions])
        q.put({"rank": rank, "out": (followed, single)})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="two-rank validation needs two GPUs")
def test_validation_on_two_ranks_matches_one_process(tmp_path, tiny_cfg):
    """Two processes on two GPUs write the same results lines and predictions file as one, bit for bit."""
    import torch.multiprocessing as mp
    from merlot_b200 import train
    from merlot_b200 import video_fib_validate as FV
    from tests.test_gpu_video_qa import _free_port
    FR.write_questions(tmp_path, [3, 3], 3, A_SMALL, prefix="train", seed=4)
    FR.write_questions(tmp_path, [5, 3, 4], 3, A_SMALL, prefix="val", seed=5, oov_every=3)
    path, _ = _config(tmp_path, tiny_cfg, val_batch_size=2)
    train.main([path])
    out = tmp_path / "out"
    ckpt = str(out / "model.ckpt-4")
    results = out / "eval" / "results.jsonl"
    clock = iter(range(10 ** 6))
    one = FV.main([path, "--chunk", "2"], clock=lambda: next(clock), sleep=lambda s: None)
    one += FV.main([path, "--checkpoint", ckpt, "--predictions", str(tmp_path / "one.npz")])
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
    """8 questions x 6 frames of 192 x 352 (67 viz tokens per frame), 64-token texts with one blank each, A = 1500
    answers: Sj = 6 * 67 + 64 = 466; merlot.yaml widths (ViT-B, 12 joint layers, do_projection), questions holding 1 to
    6 frames.  The eval forward's language rows and logits against the oracle on the same bf16-rounded weights
    (tests/test_gpu_fullsize.py's 1.5e-2 for the hidden states after 12 + 12 bf16 layers, 1e-2 for the logits)."""
    import sys
    from merlot_b200 import video_fib as VF
    from merlot_b200.modeling import MerlotModel
    from tests import multi_image_oracle as MIO
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import bench
    base = bench.load_config().model
    cfg = dict(base, hidden_dropout_prob=0.0, num_imgs=6, num_texts=1, num_chunks_in_group=1, resnet_layers=[],
               do_projection=True)
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    params, store = build(cfg, 1500, encoder_scale=1.0)
    g = torch.Generator().manual_seed(21)
    counts = [6, 5, 4, 3, 2, 1, 6, 6]
    mask = torch.arange(6)[None] < torch.tensor(counts)[:, None]
    image = torch.rand(48, 192, 352, 3, generator=g).bfloat16().float() * mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, 50357, (8, 64), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(24, 65, (8,), generator=g)
    ids = (ids * (torch.arange(64)[None] < lens[:, None])).int()
    blank = 1 + (torch.rand(8, generator=g) * (lens - 1)).long()
    ids[torch.arange(8), blank] = FR.MASK
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                    params=store, log_attention_probs=False, save_for_backward=False)
    logits = VF.fib_head(m, store, blank.int().to(DEV))
    torch.cuda.synchronize()
    assert (m.viz_chunk_length, m._dims["Sj"], m.B) == (67, 466, 8) and tuple(logits.shape) == (8, 1500)
    with torch.no_grad():
        om = MIO.MultiImageOracle(cfg, params, image, ids, img_mask=mask, log_attention_probs=False)
        lang = om.encoder_hidden_states["lang"]
        ref = head_oracle(lang[torch.arange(8), blank], params)
    rep = {"hidden_lang_rel": rel(m.encoder_hidden_states["lang"], lang), "logits_rel": rel(logits, ref),
           "logits_max_abs": float((logits.float().cpu() - ref).abs().max())}
    path = os.environ.get("MERLOT_VIDEO_FIB_REPORT") or os.path.join(tempfile.mkdtemp(prefix="merlot_video_fib_"), "parity.json")
    with open(path, "w") as f:
        json.dump(rep, f, indent=1, sort_keys=True)
    print(f"video_fib parity report: {path}: {rep}")
    assert rep["hidden_lang_rel"] < 1.5e-2 and rep["logits_rel"] < 1e-2, rep
