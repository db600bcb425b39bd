"""share_params: False on the GPU (pytest -m gpu): the language-only pass on its own `langonly_encoder/` stack.
  * one pretraining step against the oracle, in eval mode and with hidden dropout, every langonly_encoder/ gradient checked;
  * with langonly_encoder/ equal to encoder/, the separate model computes what the shared one does: the same forward bits,
    and G(encoder) + G(langonly_encoder) equal to the shared G(encoder);
  * mask_input=False (no language-only pass) is unaffected by the switch; a store without the stack the config asks for raises;
  * checkpoints: the training state round trip, a shared checkpoint restored (raises) or loaded by name (the new variables
    are reported missing and keep their values), and the trainer's save / resume loop;
  * a gradient-accumulation step of two micro-batches against the replica oracle.
"""
import pytest
import torch

from merlot_b200 import tf_checkpoint as T
from oracle import merlot_oracle as O
from tests import share_params_oracle as SO
from tests import test_gpu_checkpoint as TC
from tests import test_gpu_model as TM

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 2 ** 32 + 77


@pytest.fixture(autouse=True)
def separate_oracle(monkeypatch):
    SO.use_separate_oracle(monkeypatch)


def _sep(cfg, **kw):
    """Joint depth 2, language-only depth 3: the two stacks differ in depth as well as in variables."""
    return dict(cfg, share_params=False, num_hidden_layers=2, num_lang_transformer_hidden_layers=3, **kw)


def _lo_names(names):
    return sorted(n for n in names if n.startswith("langonly_encoder/"))


def _model(cfg, store, image, ids, shuf, **kw):
    from merlot_b200.modeling import MerlotModel
    return MerlotModel(cfg, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), shuffled_idx_img=shuf.to(DEV),
                       params=store, **kw)


def _mask_of(m, B, Lj):
    return {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}


# ---- 1. against the oracle -------------------------------------------------------------------------------------------
def _langonly_gradients(cfg, is_training, dropout_seed, oracle_dropout):
    """Every langonly_encoder/ gradient of one step against the oracle's: the 4e-2 bar of _step_parity where the oracle's
    gradient is non-zero; the key biases, whose gradient is zero (softmax is shift invariant), must be ~0 on the GPU too."""
    image, ids, shuf, vid = TM.synth(cfg, 2, 4, 16, 64, 96, 0)
    params, store, _ = TM.build(cfg)
    B, Lj = 2 * 4 // cfg["num_chunks_in_group"], 16 * cfg["num_chunks_in_group"]
    draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), cfg["vocab_size"], seed=5)
    m = _model(cfg, store, image, ids, shuf, is_training=is_training, mask_input=True, mask_draws=draws, save_for_backward=True,
               dropout_seed=dropout_seed)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=_mask_of(m, B, Lj),
                        dropout=oracle_dropout)
    m.mask_loss(), m.contrastive_loss(), m.temporal_loss(shuf.to(DEV), vid.to(DEV))
    store.g.zero_()
    m.backward()
    O.pretrain_losses(om, shuf, vid)[0].backward()
    grads = store.to_tf_dict("g")
    names = _lo_names(leaf)
    assert len(names) == 3 * 16 + 2 and names == _lo_names(grads)
    worst, zero = {}, {}
    for k in names:
        ref = leaf[k].grad
        assert ref is not None, k
        if k.endswith("/key_layer/bias"):
            scale = float(grads[k.replace("/key_layer/", "/value_layer/")].norm())
            assert float(ref.norm()) < 1e-6 * scale + 1e-9, k
            zero[k] = float(grads[k].norm()) / scale
        else:
            assert float(ref.norm()) >= 1e-7, k
            worst[k] = TM.rel(grads[k], ref)
    print(f"langonly_encoder/: worst rel {max(worst.values()):.2e} ({max(worst, key=worst.get)}); key-bias |g| / |g(value bias)| "
          f"<= {max(zero.values()):.2e}")
    assert max(worst.values()) < 4e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    assert max(zero.values()) < 1e-2, zero


@pytest.mark.parametrize("training", [False, True])
def test_step_parity(tiny_cfg, training):
    """_step_parity's forward, loss, gradient and AdamW bars with the separate stack, then its gradients one by one."""
    from oracle import dropout_mask as DM
    cfg = _sep(tiny_cfg)
    kw = {}
    if training:
        cfg = dict(cfg, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2)
        kw = dict(is_training=True, dropout_seed=SEED, oracle_dropout=DM.dropout_hook(SEED, 0.1, 0.2))
    m = TM._step_parity(cfg, wrong_dropout=DM.dropout_hook(SEED + 1, 0.1, 0.2) if training else None, **kw)
    assert m.lang_transformer_info["attention_summs"].shape == (m.B, m.L)
    _langonly_gradients(cfg, training, kw.get("dropout_seed", 0), kw.get("oracle_dropout"))


# ---- 2. separate equals shared on equal weights ------------------------------------------------------------------------
def _equal_weight_stores(cfg_sep):
    """A shared store (encoder/ of max(2, 3) layers) and a separate one whose encoder/ and langonly_encoder/ are copies of
    its encoder/ (the joint pass reads layers 0-1, the language-only pass 0-2 in both)."""
    from merlot_b200.params import ParamStore
    cfg_sh = dict(cfg_sep, share_params=True)
    params, st_sh, ocfg = TM.build(cfg_sh)
    tf = dict(params)
    tf.update({"langonly_encoder/" + k[len("encoder/"):]: v for k, v in params.items() if k.startswith("encoder/")})
    st_sep = ParamStore(cfg_sep, device=DEV, optimizer_cfg=ocfg)
    st_sep.load_tf_dict(tf)
    return cfg_sh, st_sh, st_sep, ocfg


def _rel_max(a, b):
    """max |a - b| over max |b|: the reassociation of fp32 sums shows as a few ulps of the tensor's scale."""
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_separate_equals_shared_on_equal_weights(tiny_cfg):
    """Training mode, hidden dropout 0.1, same inputs, seed and masks.  Forward: the language-only and joint hidden states,
    lang_trg and every loss bit for bit.  attention_summs and attention_log are column sums of the attention maps that K4
    (attention.cu, colsum) adds with float atomics: equal up to their reassociation, max |diff| <= 1e-5 of the scale.
    Backward: G(encoder) + G(langonly_encoder) of the separate store against the shared G(encoder), and every other
    gradient, to fp32 reassociation: the weight-gradient GEMMs red.add their split-K partial sums into the arena in no fixed
    order (and the shared store adds both passes into one tensor), and the LM head's input gradient is a split-K sum too.
    A reordered split-K sum can also flip the bf16 rounding of an element of the joint output's gradient.  Bar, that of
    test_partial_stack_backward_equals_full for the same atomics: rel-Frobenius < 1e-3 per tensor with a non-zero gradient
    and < 1e-4 over all gradients (observed on an H100 in two runs: at most 1.5e-7 and 2.9e-8).  One AdamW step past
    warm-up then moves the two encoders of the separate store apart."""
    from merlot_b200.optimization import build_optimizer_from_config
    cfg_sep = _sep(tiny_cfg, hidden_dropout_prob=0.1)
    cfg_sh, st_sh, st_sep, ocfg = _equal_weight_stores(cfg_sep)
    image, ids, shuf, vid = TM.synth(cfg_sh, 2, 4, 16, 64, 96, 3)
    B, Lj = 2 * 4 // cfg_sh["num_chunks_in_group"], 16 * cfg_sh["num_chunks_in_group"]
    draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), cfg_sh["vocab_size"], seed=5)
    runs = []
    for cfg, st in ((cfg_sh, st_sh), (cfg_sep, st_sep)):
        mask = {"mask_draws": draws} if not runs else {"mask_override": _mask_of(runs[0]["m"], B, Lj)}
        m = _model(cfg, st, image, ids, shuf, is_training=True, mask_input=True, save_for_backward=True, dropout_seed=SEED,
                   **mask)
        (ll, linfo), (cl, cinfo), (tl, tinfo) = m.mask_loss(), m.contrastive_loss(), m.temporal_loss(shuf.to(DEV), vid.to(DEV))
        losses = {"mask": ll, "contrastive": cl, "temporal": tl, **{f"lang/{k}": v for k, v in linfo.items()},
                  **{f"contr/{k}": v for k, v in cinfo.items()}, **{f"temporal/{k}": v for k, v in tinfo.items()}}
        st.g.zero_()
        m.backward()
        torch.cuda.synchronize()
        runs.append({"m": m, "losses": {k: float(v) for k, v in losses.items()}, "g": st.to_tf_dict("g"),
                     "lo_h": m.lang_transformer_info["hidden_state"].clone(), "joint_h": m.encoder_info["hidden_state"].clone(),
                     "lang_trg": m.lang_trg_h.clone(), "summs": m.lang_transformer_info["attention_summs"].clone(),
                     "attn_log": {k: float(v) for k, v in m.attention_log.items()}})
    sh, sep = runs
    report = {k: torch.equal(sh[k], sep[k]) for k in ("lo_h", "joint_h", "lang_trg")}
    report.update({f"loss {k}": sh["losses"][k] == sep["losses"][k] for k in sh["losses"]})
    summs = _rel_max(sep["summs"], sh["summs"])
    logs = max(abs(sep["attn_log"][k] - sh["attn_log"][k]) / max(abs(sh["attn_log"][k]), 1e-30) for k in sh["attn_log"])
    g_sh, g_sep = sh["g"], sep["g"]
    assert set(g_sep) - set(g_sh) == set(_lo_names(g_sep))
    combined = {}
    for k in g_sh:
        parts = [g_sep[n] for n in (k, "langonly_encoder/" + k[len("encoder/"):]) if k.startswith("encoder/") and n in g_sep]
        combined[k] = sum(parts[1:], parts[0]) if parts else g_sep[k]
    per = {k: TM.rel(combined[k], g_sh[k]) for k in g_sh if float(g_sh[k].norm()) >= 1e-7}
    whole = TM.rel(torch.cat([combined[k].reshape(-1) for k in g_sh]), torch.cat([g_sh[k].reshape(-1) for k in g_sh]))
    print(f"forward bit-equal: {report}; attention_summs {summs:.2e}, attention_log {logs:.2e}; gradients: worst per tensor "
          f"{max(per.values()):.2e} ({max(per, key=per.get)}), all {whole:.2e}")
    assert all(report.values()), report
    assert summs <= 1e-5 and logs <= 1e-5
    assert max(per.values()) < 1e-3 and whole < 1e-4, sorted(per.items(), key=lambda kv: -kv[1])[:5]
    # the separate store's two encoders start equal; their gradients differ, so one AdamW step moves them apart
    opt, _ = build_optimizer_from_config(None, ocfg, None, store=st_sep)
    st_sep.global_step = ocfg["num_warmup_steps"]  # the learning rate is 0 at step 0 of the warm-up
    opt.apply_gradients()
    p = st_sep.to_tf_dict("p")
    for name in ("layer00/query_layer/kernel", "layer01/intermediate/bias", "LayerNorm_ln_final/gamma"):
        assert not torch.equal(p[f"encoder/{name}"], p[f"langonly_encoder/{name}"]), name


# ---- 6. mask_input=False, and stores that lack the stack ---------------------------------------------------------------
def test_mask_input_false_forward_is_unchanged(tiny_cfg):
    """Without the language-only pass (the VCR / zero-shot forward) the switch changes nothing: the joint encoder reads
    encoder/ layers 0-1 in both stores, and the hidden states and temporal logits are bit for bit the same."""
    cfg_sep = _sep(tiny_cfg)
    cfg_sh, st_sh, st_sep, _ = _equal_weight_stores(cfg_sep)
    with torch.no_grad():
        for n in _lo_names(st_sep.entries):  # the separate stack is not read: scramble it
            st_sep.P(n).normal_()
    st_sep.sync_bf16()
    image, ids, shuf, vid = TM.synth(cfg_sh, 2, 4, 16, 64, 96, 4)
    outs = []
    for cfg, st in ((cfg_sh, st_sh), (cfg_sep, st_sep)):
        m = _model(cfg, st, image, ids, shuf, is_training=False, mask_input=False, log_attention_probs=False)
        _, tinfo = m.temporal_loss(shuf.to(DEV), vid.to(DEV))
        outs.append((m.encoder_info["hidden_state"].clone(), float(tinfo["lang_viz_loss"]), float(tinfo["viz_viz_loss"])))
    assert torch.equal(outs[0][0], outs[1][0]) and outs[0][1:] == outs[1][1:]


def test_store_without_the_stack_raises(tiny_cfg):
    """The language-only pass checks that the store holds the stack the config asks for, before any launch."""
    from merlot_b200.params import ParamStore
    cfg_sep = _sep(tiny_cfg)
    image, ids, shuf, _ = TM.synth(cfg_sep, 2, 4, 16, 64, 96, 0)
    shared_store = ParamStore(dict(cfg_sep, share_params=True), device=DEV)
    with pytest.raises(ValueError, match="langonly_encoder/"):
        _model(cfg_sep, shared_store, image, ids, shuf, is_training=False, mask_input=True)
    sep_store = ParamStore(cfg_sep, device=DEV)  # encoder/ of 2 layers: too shallow for a shared 3-layer language-only pass
    with pytest.raises(ValueError, match="encoder/"):
        _model(dict(cfg_sep, share_params=True), sep_store, image, ids, shuf, is_training=False, mask_input=True)


# ---- 3, 4. checkpoints and the trainer ---------------------------------------------------------------------------------
def test_training_state_round_trip(tmp_path, tiny_cfg):
    _, _, prefix = TC._round_trip(TC._config(_sep(tiny_cfg)), tmp_path)
    names = dict(T.list_variables(prefix))
    for n in ("langonly_encoder/layer02/key_layer/kernel", "langonly_encoder/LayerNorm_ln_final/beta"):
        assert n in names and f"{n}/adam_m" in names and f"{n}/adam_v" in names, n
    assert "encoder/layer01/query_layer/kernel" in names and "encoder/layer02/query_layer/kernel" not in names


def test_shared_checkpoint_into_a_separate_store(tmp_path, tiny_cfg):
    """restore_checkpoint (Saver.restore) needs every variable: it raises and names the missing langonly_encoder/ ones.
    load_checkpoint (init_checkpoint's restore by name) reports exactly the langonly_encoder/ entries as missing, leaves
    them at their initial values and restores everything else."""
    from merlot_b200.params import ParamStore
    shared = TC._trained(TC._config(tiny_cfg), steps=1).store
    prefix = str(tmp_path / "model.ckpt-1")
    shared.save_checkpoint(prefix)
    sep = ParamStore(_sep(tiny_cfg), device=DEV, optimizer_cfg=TC.OCFG)
    sep.init_reference(seed=4)
    with pytest.raises(T.CheckpointFormatError, match="langonly_encoder/"):
        sep.restore_checkpoint(prefix)
    before = sep.to_tf_dict("p")
    missing = sep.load_checkpoint(prefix)
    assert sorted(missing) == _lo_names(sep.entries)
    after, ref = sep.to_tf_dict("p"), shared.to_tf_dict("p")
    for k, v in after.items():
        assert torch.equal(v, before[k] if k.startswith("langonly_encoder/") else ref[k]), k


def test_trainer_saves_and_resumes(tmp_path, tiny_cfg, capsys):
    from merlot_b200.train import main
    cfg = _sep(tiny_cfg)
    out = tmp_path / "out"
    main([TC._yaml(tmp_path, cfg, 3, out)])
    assert T.latest_checkpoint(str(out)) == str(out / "model.ckpt-3")
    names = dict(T.list_variables(str(out / "model.ckpt-3")))
    for n in ("langonly_encoder/layer02/value_layer/kernel", "langonly_encoder/layer00/LayerNorm_mlp_ln0/gamma"):
        assert n in names and f"{n}/adam_m" in names and f"{n}/adam_v" in names, n
    capsys.readouterr()
    main([TC._yaml(tmp_path, cfg, 5, out)])
    log = capsys.readouterr().out
    assert "continuing from global_step 3" in log and "step 0 loss" not in log, log
    assert T.latest_checkpoint(str(out)) == str(out / "model.ckpt-5")
    assert int(T.load_checkpoint(str(out / "model.ckpt-5"), names=["global_step"])["global_step"]) == 5


# ---- 5. gradient accumulation ------------------------------------------------------------------------------------------
def test_accumulated_step_is_the_replica_oracle(monkeypatch):
    from tests import test_gpu_accumulation as TA
    monkeypatch.setattr(TA, "CFG", dict(TA.CFG, share_params=False, num_lang_transformer_hidden_layers=3))
    TA.test_accumulated_pretraining_step_is_the_replica_oracle(2)
