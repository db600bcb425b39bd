"""GPU parity of the whole hot path through the MerlotModel mirror (pytest -m gpu): forward activations, the three
losses, every parameter gradient, one optimizer step -- against the oracle on identical weights and inputs, in eval mode
(dropout 0) and in training mode (hidden dropout under the kernels' own masks); plus size-independent properties at
merlot.yaml's full sizes."""
import pytest
import torch

from oracle import merlot_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def synth(cfg, batch, nc, Lc, h0, w0, seed):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(batch * nc, h0, w0, 3, generator=g).bfloat16().float()
    ids = torch.randint(100, cfg["vocab_size"], (batch, nc, Lc), generator=g)
    ids[:, :, 0] = O.START
    lens = torch.randint(Lc // 2, Lc + 1, (batch, nc), generator=g)
    ids = (ids * (torch.arange(Lc)[None, None] < lens[..., None])).int()
    ncg = cfg["num_chunks_in_group"]
    B = batch * nc // ncg
    shuf = torch.arange(ncg).repeat(B)
    shuf[:ncg] = 16 + torch.randperm(ncg, generator=g)
    if B > 1:
        shuf[ncg:2 * ncg] = 64 + torch.randperm(ncg, generator=g)
    vid = torch.zeros(B, ncg, dtype=torch.int32)
    vid[0, ncg // 2:] = 1
    return image, ids, shuf.int(), vid


def bf16_operands(params):
    """GEMM operands are the bf16 compute copies (bfloat16_getter): hand the oracle the same rounded matrices."""
    return {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}


def build(cfg, seed=1, ocfg=None):
    from merlot_b200.params import ParamStore
    params = bf16_operands(O.init_params(cfg, seed=seed, perturb=0.05))
    ocfg = ocfg or dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=10, weight_decay_rate=0.1,
                        beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
                        param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]])
    store = ParamStore(cfg, device=DEV, optimizer_cfg=ocfg)
    store.load_tf_dict(params)
    return params, store, ocfg


def _step_parity(cfg, is_training=False, dropout_seed=0, oracle_dropout=None, wrong_dropout=None, batch=2, nc=4, Lc=16, hw=(64, 96)):
    """One pretraining step (forward, the three losses, backward, AdamW) against the oracle on the same weights and inputs:
    `batch` videos of `nc` segments, captions of `Lc` tokens, frames of hw.  Training mode: the model runs with dropout_seed,
    the oracle applies `oracle_dropout` (its hook for the same seed) and an oracle with `wrong_dropout` (another seed) must
    miss the hidden-state or loss bars.  Returns the model."""
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.optimization import build_optimizer_from_config
    image, ids, shuf, vid = synth(cfg, batch, nc, Lc, *hw, 0)
    params, store, ocfg = build(cfg)
    B, Lj = batch * nc // cfg["num_chunks_in_group"], Lc * cfg["num_chunks_in_group"]
    draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), cfg["vocab_size"], seed=5)
    m = MerlotModel(cfg, is_training=is_training, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                    shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, save_for_backward=True, dropout_seed=dropout_seed)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_draws=draws, dropout=oracle_dropout)
    assert rel(m.lang_transformer_info["attention_summs"], om.attention_summs) < 2e-3
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    if not (torch.equal(gm["masked_ids"], om.lang_mask_info["masked_ids"]) and torch.equal(gm["masked_idx"], om.lang_mask_info["masked_idx"])):
        om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm,
                            dropout=oracle_dropout)  # near-tie in attn sums
    for name in ("viz", "lang"):
        assert rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name]) < 1e-2  # rel-Frobenius, bf16 stacks
    for k, v in om.attention_log.items():  # attention_log metrics (model/modeling.py:186-203)
        assert abs(float(m.attention_log[k]) - float(v)) < 2e-3, k
    ll, linfo = m.mask_loss()
    cl, cinfo = m.contrastive_loss()
    tl, tinfo = m.temporal_loss(shuf.to(DEV), vid.to(DEV))
    total_ref, oinfo = O.pretrain_losses(om, shuf, vid)
    for a, b in [(ll, oinfo["lang"]["loss"]), (cinfo["lang_to_viz"], oinfo["contr"]["lang_to_viz"]),
                 (cinfo["viz_to_lang"], oinfo["contr"]["viz_to_lang"]), (cl, oinfo["contr"]["loss_all"]),
                 (tinfo["lang_viz_loss"], oinfo["temporal"]["lang_viz_loss"]), (tinfo["viz_viz_loss"], oinfo["temporal"]["viz_viz_loss"]),
                 (tl, oinfo["temporal"]["loss"])]:
        assert abs(float(a) - float(b)) <= 2e-3 * abs(float(b)), (float(a), float(b))
    total = float(ll) + float(cl) + float(tl)
    assert abs(total - float(total_ref)) <= 1e-3 * abs(float(total_ref))  # north-star bar: losses within 1e-3 rel
    if wrong_dropout is not None:  # the comparison notices a mask that is not the one the step used
        bad = O.MerlotOracle(cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm, dropout=wrong_dropout)
        bad_total, _ = O.pretrain_losses(bad, shuf, vid)
        assert (max(rel(m.encoder_hidden_states[n], bad.encoder_hidden_states[n]) for n in ("viz", "lang")) >= 1e-2
                or abs(total - float(bad_total)) > 1e-3 * abs(float(bad_total)))
    assert float(tinfo["lang_viz_acc"]) == pytest.approx(float(oinfo["temporal"]["lang_viz_acc"]), abs=1e-6)
    store.g.zero_()
    m.backward()
    total_ref.backward()
    grads = store.to_tf_dict("g")
    for k, v in leaf.items():
        if v.grad is None or float(v.grad.norm()) < 1e-7:  # key biases: softmax is shift invariant => exactly zero gradient
            continue
        assert rel(grads[k], v.grad) < 4e-2, k
    # one AdamW step on those gradients vs the oracle optimizer fed the GPU gradients (isolates K10 from bf16 noise), taken at
    # the end of the warm-up: at step 0 the learning rate is 0 and the parameters could not move on either side
    check_adam_step(store, build_optimizer_from_config(None, ocfg, None, store=store)[0], ocfg, grads)
    return m


def check_adam_step(store, opt, ocfg, grads):
    """opt.apply_gradients() at global_step num_warmup_steps against AdamOracle fed `grads` (the gradients in store.g):
    parameters within 2e-6, the moments bit for bit; the parameters move by over 20x that bar (an Adam step from zero
    moments moves a parameter by about 0.7 lr_t, 1.4e-4 at learning_rate 3e-4) and store.g ends zeroed."""
    step = ocfg["num_warmup_steps"]
    store.global_step = step
    p_before = {k: v.clone() for k, v in store.to_tf_dict("p").items()}
    p_ref = {k: v.clone() for k, v in p_before.items()}
    adam = O.AdamOracle(p_ref, ocfg)
    adam.global_step = step
    assert float(adam.step_scalars()["lr"]) > 0
    adam.apply_gradients(p_ref, grads)
    opt.apply_gradients()
    after = store.to_tf_dict("p")
    for k in after:
        assert (after[k] - p_ref[k]).abs().max().item() < 2e-6, k
    assert max((after[k] - p_before[k]).abs().max().item() for k in after) > 20 * 2e-6
    for buf, ref in ((store.m, adam.m), (store.v, adam.v)):
        views = store.tf_views(buf)
        assert len(views) == len(ref)
        for _, nm, t in views:
            assert t.dtype == ref[nm].dtype and torch.equal(bits(t.cpu().contiguous()), bits(ref[nm].contiguous())), nm
    assert float(store.g.abs().max()) == 0.0 and store.global_step == step + 1


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def test_pretrain_step_parity(tiny_cfg):
    _step_parity(tiny_cfg)


def test_pretrain_step_parity_training_mode(tiny_cfg):
    """The training step with hidden dropout on (the headline configuration), against the oracle under the very masks the
    kernels draw (oracle/dropout_mask.py).  ViT and text stacks use different probabilities, so swapped ones are caught; the
    seed has a non-zero high word."""
    from oracle import dropout_mask as DM
    cfg = dict(tiny_cfg, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2)
    seed = 2 ** 32 + 77
    _step_parity(cfg, is_training=True, dropout_seed=seed, oracle_dropout=DM.dropout_hook(seed, 0.1, 0.2),
                 wrong_dropout=DM.dropout_hook(seed + 1, 0.1, 0.2))


def _long_sequence_step_parity(tiny_cfg, Lc, max_pos):
    """The training-mode step of test_pretrain_step_parity_training_mode at tiny width but long sequences: one video of 8
    segments with Lc-token captions and 64x96 frames (7 vision tokens per segment), so the language-only stack runs over
    L = 8 Lc tokens and the joint encoder over Sj = 8 Lc + 56.  Both are longer than 4 key tiles, so every attention backward
    reduces dQ atomically into the one workspace slice that the stack clears once and each layer hands back zeroed to the
    layer below it; with two layers per stack, the lower layer consumes a workspace the upper one used."""
    from merlot_b200._lib import lib
    from oracle import dropout_mask as DM
    cfg = dict(tiny_cfg, num_chunks_in_group=8, max_position_embeddings=max_pos, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2)
    L, Sj = 8 * Lc, 8 * Lc + 56
    assert lib().merlot_attention_bwd_dq_parts(L) == 0 and lib().merlot_attention_bwd_dq_parts(Sj) == 0
    assert cfg["num_hidden_layers"] >= 2 and cfg["num_lang_transformer_hidden_layers"] >= 2
    seed = 2 ** 32 + 78
    m = _step_parity(cfg, is_training=True, dropout_seed=seed, oracle_dropout=DM.dropout_hook(seed, 0.1, 0.2),
                     wrong_dropout=DM.dropout_hook(seed + 1, 0.1, 0.2), batch=1, nc=8, Lc=Lc)
    assert m.lang_transformer_info["hidden_state"].shape[1] == L and m._dims["Sj"] == Sj


def test_pretrain_step_parity_long_sequence(tiny_cfg):
    """80-token captions: L = 640, Sj = 696."""
    _long_sequence_step_parity(tiny_cfg, Lc=80, max_pos=1024)


def test_pretrain_step_parity_config5_lengths(tiny_cfg):
    """configs[4]'s sequence lengths (8 segments x 384-token captions, max_position_embeddings 3072) at tiny width:
    L = 3072, Sj = 3128.  The full-width step is out of reach of the CPU oracle (its attention probabilities alone would
    take 12 x 3608^2 x 4 B = 625 MB per layer before autograd)."""
    _long_sequence_step_parity(tiny_cfg, Lc=384, max_pos=3072)


def test_disable_pairwise_lang_attn(tiny_cfg):
    """model/modeling.py:160-168 through the whole model: with the switch on, the language chunks of the joint encoder see the
    vision tokens and themselves only -- hidden states, attention_log, the three losses and every gradient against the oracle
    (which builds the reference's explicit mask), and the result differs from the unrestricted model."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, disable_pairwise_lang_attn=True, num_chunks_in_group=4)
    batch, nc, Lc = 2, 4, 16
    image, ids, shuf, vid = synth(cfg, batch, nc, Lc, 64, 96, 3)
    params, store, _ = build(cfg)
    B, Lj = batch * nc // cfg["num_chunks_in_group"], Lc * cfg["num_chunks_in_group"]
    draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), cfg["vocab_size"], seed=7)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                    shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, save_for_backward=True)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm)
    for name in ("viz", "lang"):
        assert rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name]) < 1e-2
    for k, v in om.attention_log.items():
        assert abs(float(m.attention_log[k]) - float(v)) < 2e-3, k
    free = O.MerlotOracle(dict(cfg, disable_pairwise_lang_attn=False), params, image, ids, mask_input=True, shuffled_idx_img=shuf,
                          mask_override=gm)
    assert rel(free.encoder_hidden_states["lang"], om.encoder_hidden_states["lang"]) > 3e-3  # the switch changes the function (near-uniform attention at this init: ~1e-2)
    ll, _ = m.mask_loss()
    cl, _ = m.contrastive_loss()
    tl, _ = m.temporal_loss(shuf.to(DEV), vid.to(DEV))
    total_ref, _ = O.pretrain_losses(om, shuf, vid)
    total = float(ll) + float(cl) + float(tl)
    assert abs(total - float(total_ref)) <= 1e-3 * abs(float(total_ref))
    store.g.zero_()
    m.backward()
    total_ref.backward()
    grads = store.to_tf_dict("g")
    for k, v in leaf.items():
        if v.grad is None or float(v.grad.norm()) < 1e-7:
            continue
        assert rel(grads[k], v.grad) < 4e-2, k


def test_forward_only_2d_ids_config1(tiny_cfg):
    """BASELINE config 1 shape family: 2-D input_ids => num_chunks = 1 (model/modeling.py:72-77), no masking, no losses."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg)
    image, ids, _, _ = synth(cfg, 3, 1, 16, 64, 96, 2)
    params, store, _ = build(cfg, seed=3)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids[:, 0].to(DEV), params=store)
    om = O.MerlotOracle(cfg, params, image, ids[:, 0])
    assert m.num_chunks == 1 and m.B == 3 and m.L == 16 and m.P == om.P
    for name in ("viz", "lang"):
        assert m.encoder_hidden_states[name].shape == om.encoder_hidden_states[name].shape
        assert rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name]) < 1e-2
    with pytest.raises(ValueError):
        MerlotModel(cfg, False, False, image.to(DEV), ids[0, 0].to(DEV), params=store)  # rank-1 ids: assert_rank ValueError
    with pytest.raises(AssertionError):
        MerlotModel(cfg, False, False, image[:, :60].to(DEV), ids[:, 0].to(DEV), params=store)  # h % patch != 0


def test_sort_story_temporal_head_config4_shape(tiny_cfg):
    """downstream/sort_story/get_zero_shot_logits.py:55-86: eval forward, shuffled idx + 64, all-pairs temporal softmax."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, num_chunks_in_group=5, max_position_embeddings=128)
    image, ids, _, _ = synth(cfg, 2, 5, 16, 64, 64, 4)
    params, store, _ = build(cfg, seed=5)
    shuf = (torch.stack([torch.randperm(5, generator=torch.Generator().manual_seed(i)) for i in range(2)]) + 64).int().reshape(-1)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=False,
                    shuffled_idx_img=shuf.to(DEV), params=store)
    om = O.MerlotOracle(cfg, params, image, ids, mask_input=False, shuffled_idx_img=shuf)
    H = cfg["hidden_size"]
    h_lang = m.encoder_hidden_states["lang"].reshape(m.B, 5, m.lang_chunk_length, H)[:, :, 0]
    h_viz = m.encoder_hidden_states["viz"].reshape(m.B, 5, m.viz_chunk_length, H)[:, :, 0]
    logits = m.allpairs_temporal_logits(h_lang, h_viz, scope_name="lang_viz_temporal")
    ol = om.encoder_hidden_states["lang"].reshape(om.B, 5, om.lang_chunk_length, H)[:, :, 0]
    ov = om.encoder_hidden_states["viz"].reshape(om.B, 5, om.viz_chunk_length, H)[:, :, 0]
    ref = om.allpairs_temporal_logits(ol, ov, "lang_viz_temporal")
    assert logits.shape == ref.shape == (2 * 25, 4)
    assert rel(torch.softmax(logits.float(), -1)[:, 1:], torch.softmax(ref, -1)[:, 1:]) < 1e-2


def test_dropout_training_mode_is_deterministic_and_changes_output(tiny_cfg):
    from merlot_b200.modeling import MerlotModel
    image, ids, shuf, vid = synth(tiny_cfg, 2, 4, 16, 64, 96, 0)
    _, store, _ = build(tiny_cfg)
    outs = []
    for seed in (11, 11, 12):
        m = MerlotModel(tiny_cfg, is_training=True, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=False,
                        shuffled_idx_img=shuf.to(DEV), params=store, dropout_seed=seed)
        outs.append(m.encoder_hidden_states["lang"].clone())
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])


def test_full_size_properties():
    """merlot.yaml sizes (BASELINE configs[1], batch 2 to stay quick): finite losses at the random-init levels the
    closed forms predict, backward linearity (grad arena accumulates: two backwards == 2x), and loss decreases on a fixed batch."""
    import math
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from merlot_b200.train import model_fn_builder, synthetic_batch
    cfg = bench.load_config()
    cfg.model["hidden_dropout_prob"] = 0.0
    cfg.optimizer["num_warmup_steps"] = 0
    fn = model_fn_builder(cfg)
    feats = synthetic_batch(cfg, 2, seed=0)
    spec = fn(feats)
    lang, contr, temp = (float(x) for x in spec.loss_parts)
    assert abs(lang - math.log(50370)) < 0.5  # random-init MLM loss ~ ln(V)
    assert 0.0 < contr < 0.25 * 2 * math.log(8) + 1.0 and math.isfinite(temp)
    store = fn.store
    store.g.zero_()
    spec.model.backward()
    g1 = store.g.clone()
    spec.model.backward()
    # Accumulation is linear; the backward itself is not bit-reproducible: dQ is reduced with fp32 atomics, its bf16
    # rounding flips on ~1e-5 of the elements and 12 pre-LN layers amplify that to ~3e-3 run-to-run on the earliest
    # layers' gradients (tools/determinism_check.py, tools/op_determinism.py: every other op is bitwise repeatable).
    assert rel(store.g, 2 * g1) < 1e-2
    assert torch.isfinite(g1).all() and float(g1.abs().max()) > 0
    store.g.zero_()
    l0 = spec.loss
    for _ in range(8):
        s = fn(feats)
        s.train_op()
    assert fn(feats).loss < l0  # the step trains


def _partial_backward_equals_full(tiny_cfg, training):
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, num_vision_transformer_hidden_layers=4, vit_hidden_dropout_prob=0.2)
    image, ids, shuf, vid = synth(cfg, 2, 4, 16, 64, 96, 0)
    params, store, _ = build(cfg)
    draws = O.make_mask_draws(4, 32, 6, cfg["vocab_size"], seed=5)
    gs = []
    for groups in (None, [(2, 4), (1, 2), (0, 1)]):
        m = MerlotModel(cfg, is_training=training, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                        shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, save_for_backward=True,
                        dropout_seed=2 ** 32 + 5)
        m.mask_loss(), m.contrastive_loss(), m.temporal_loss(shuf.to(DEV), vid.to(DEV))
        store.g.zero_()
        seen = []
        m.backward(vit_layer_groups=groups, on_vit_group_done=seen.append)
        gs.append(store.g.clone())
        assert seen == ([] if groups is None else [0, 1, 2])
    assert rel(gs[1], gs[0]) < 1e-3
    store.g.zero_()


def test_partial_stack_backward_equals_full(tiny_cfg):
    """merlot_stack_backward walked in layer groups (bwd_lo/bwd_hi; data-parallel bucket overlap) gives the gradients of one
    full call (the only difference allowed is the order of fp32 atomic adds in split-K wgrads / LN column sums)."""
    _partial_backward_equals_full(tiny_cfg, training=False)


def test_partial_stack_backward_equals_full_training_mode(tiny_cfg):
    """The same with hidden dropout on: each layer-group call hands the next one the dropout-masked stream gradient of the
    layer below it (`dmask` in the stack's scratch)."""
    _partial_backward_equals_full(tiny_cfg, training=True)


def test_exported_attention_probabilities(tiny_cfg):
    """encoder_info / lang_transformer_info['self_attn_probs'] (model_fn PREDICT outputs, model/modeling.py:762-770): head-mean
    probabilities [B, layers, S, S] against the oracle's transformer(return_attn_probs=True); rows sum to one."""
    from merlot_b200.modeling import MerlotModel
    cfg = tiny_cfg
    image, ids, shuf, vid = synth(cfg, 2, 4, 16, 64, 96, 0)
    params, store, _ = build(cfg)
    draws = O.make_mask_draws(4, 32, 6, cfg["vocab_size"], seed=5)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                    shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, export_attention_probs=True)
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(4, 32), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    om = O.MerlotOracle(cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm)
    pj, pl = m.encoder_info["self_attn_probs"], m.lang_transformer_info["self_attn_probs"]
    assert tuple(pj.shape) == tuple(om.encoder_info["self_attn_probs"].shape)
    assert tuple(pl.shape) == tuple(om.lang_transformer_info["self_attn_probs"].shape)
    assert rel(pl, om.lang_transformer_info["self_attn_probs"]) < 5e-3
    assert rel(pj, om.encoder_info["self_attn_probs"]) < 1e-2  # second layer sees bf16 activations of the first
    assert float((pj.sum(-1) - 1).abs().max()) < 2e-3


def test_vcr_num_texts_tiling_and_cls_head(tiny_cfg):
    """merlot_vcr.yaml's num_texts: 4 (model/modeling.py:111-119): every image's tokens are tiled to its four candidate texts;
    plus downstream/vcr's validation head and loss.  Forward against the oracle; backward of an external head's gradient
    (d_hidden_state) against autograd: the four texts' gradients meet in the shared image tokens."""
    from merlot_b200 import vcr
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, num_texts=4, num_chunks_in_group=1)
    g = torch.Generator().manual_seed(3)
    nimg, L = 3, 16
    image = torch.rand(nimg, 64, 96, 3, generator=g).bfloat16().float()
    ids = torch.randint(100, cfg["vocab_size"], (nimg * 4, L), generator=g)
    ids[:, 0] = O.START
    ids[:, 12:] = 0
    ids = ids.int()
    params, store, _ = build(cfg)
    head = vcr.init_head(cfg["hidden_size"], "answer", seed=1, device=DEV)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), params=store, save_for_backward=True)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    om = O.MerlotOracle(cfg, leaf, image, ids)
    assert (m.B, m.img_batch_size, m.P) == (12, 3, om.P)
    for name in ("viz", "lang"):
        assert rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name]) < 1e-2
    hp = {k: v.float().cpu() for k, v in head.items()}
    hp = {k: (v.bfloat16().float() if k.endswith("kernel") else v) for k, v in hp.items()}
    logits = vcr.cls_head_val(m, head, "answer")
    ref = O.vcr_cls_head_val(om, hp, "answer")
    assert tuple(logits.shape) == (3, 4) and rel(logits, ref) < 1e-2
    target = torch.tensor([1, 3, 0])
    loss, acc = vcr.cls_loss(logits, target.to(DEV))
    ref_loss = torch.nn.functional.cross_entropy(ref, target, reduction="sum") / 3  # downstream/vcr/modeling.py:141-142
    assert abs(float(loss) - float(ref_loss)) < 2e-3 * abs(float(ref_loss))
    # an external head's gradient through the tiled model: d(sum of first-language-token features . w)
    Sj, H = m._dims["Sj"], cfg["hidden_size"]
    w = (torch.randn(12, Sj, H, generator=g) * 0.05).bfloat16()
    store.g.zero_()
    m.backward(d_hidden_state=w.to(DEV))
    (om.encoder_info["hidden_state"] * w.float()).sum().backward()
    grads = store.to_tf_dict("g")
    worst = {k: rel(grads[k], v.grad) for k, v in leaf.items() if v.grad is not None and float(v.grad.norm()) > 1e-7}
    assert len(worst) > 40 and max(worst.values()) < 4e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    store.g.zero_()
