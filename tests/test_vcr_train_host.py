"""VCR fine-tuning on the host (no GPU): the parameter arena of ParamStore(task="vcr") against the reference graph's variables,
the unchanged pretraining arena, the towers' initial values and checkpoint round trips, init_checkpoint, the synthetic VCR
batch and the CLI's dispatch on downstream.task."""
import hashlib
import math

import pytest
import torch

from tests import vcr_oracle as V

# merlot_vcr.yaml (model/configs/merlot_vcr.yaml) with the model shrunk to the test width: its optimizer, dropout, num_texts,
# transpose_input, downstream and device sections copied as shipped
VCR_YAML_OPTIMIZER = dict(type="adam_optimizer", learning_rate=0.000012, num_train_steps=60000, num_warmup_steps=6000,
                          weight_decay_rate=0.01, beta_2=0.98, clip_norm=0.0, adafactor=False, use_bfloat16_adam=True, verbose=False,
                          param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"],
                                            {"weight_decay_rate": 0}]])


def vcr_config(tiny_cfg, **model):
    from merlot_b200.config import NeatConfig
    m = dict(tiny_cfg, num_texts=4, transpose_input=True, image_size=[64, 96], attention_probs_dropout_prob=0.0,
             hidden_dropout_prob=0.1, num_chunks_in_group=1)
    m.update(model)
    return NeatConfig.from_dict({"data": {"train_file": "", "val_file": "", "draw": "segm"}, "model": m,
                                 "optimizer": dict(VCR_YAML_OPTIMIZER),
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_vcr", "train_batch_size": 64},
                                 "downstream": {"task": "vcr", "mode": "answer"}})


def _fingerprint(st):
    rows = [(e.name, e.shape, e.tf_names, e.offset, e.numel, e.padded, tuple(float(x) for x in e.hyper)) for e in st.entries.values()]
    rows.append(("groups", tuple((tuple(float(x) for x in h), o, c) for h, o, c in st.groups), st.total, st.num_params()))
    return hashlib.sha256(repr(rows).encode()).hexdigest()


# Recorded from the arena before ParamStore had a `task` (every entry's name, shape, reference names, offset, size, padding
# and hyper-parameters, then the group table, the arena size and num_params).
_PRETRAIN_FINGERPRINTS = {
    ("patch", False): "081200d3e3d3b6d72a406751891ed90eb0b8690b1b5613a2d5d397e99c262ea3",
    ("patch", True): "f1098879e0694d8ab178b26ffd60f2f88cfe3d8b67d440022b120a9a8070657f",
    ("hybrid", False): "cacd984d74b4c10961cc8815c91ae221457179f2a46c247e6e8c3a7249a932e0",
    ("hybrid", True): "ed13e4d9e0a4858f2bd3eb6f30e8761035918472104de3a3da9ea9c393f4711e",
}


@pytest.mark.parametrize("stem", ["patch", "hybrid"])
@pytest.mark.parametrize("grouped", [False, True])
def test_default_arena_is_the_pretraining_arena(tiny_cfg, stem, grouped):
    from merlot_b200.params import ParamStore
    cfg = dict(tiny_cfg, resnet_layers=[1, 2] if stem == "hybrid" else [])
    ocfg = VCR_YAML_OPTIMIZER if grouped else None
    st = ParamStore(cfg, device="cpu", optimizer_cfg=ocfg)
    assert st.task == "pretrain"
    assert _fingerprint(st) == _PRETRAIN_FINGERPRINTS[(stem, grouped)]
    explicit = ParamStore(cfg, device="cpu", optimizer_cfg=ocfg, task="pretrain")
    assert _fingerprint(explicit) == _fingerprint(st)
    with pytest.raises(ValueError):
        ParamStore(cfg, device="cpu", task="vqa")


@pytest.mark.parametrize("stem", ["patch", "hybrid"])
def test_vcr_layout_is_the_reference_graph(tiny_cfg, stem):
    from merlot_b200.params import ParamStore
    cfg = dict(tiny_cfg, resnet_layers=[1, 2] if stem == "hybrid" else [], num_lang_transformer_hidden_layers=3)
    st = ParamStore(cfg, device="cpu", optimizer_cfg=VCR_YAML_OPTIMIZER, task="vcr")
    shapes = V.param_shapes(cfg)
    names = set(st.to_tf_dict("p"))
    assert names == set(shapes)
    for bad in ("langonly_embeddings/", "contrastive/", "_temporal/", "lm_head/", "encoder/layer02/"):
        assert not any(bad in n for n in names), bad
    assert st.num_params() == sum(math.prod(s) for s in shapes.values())
    for tower in V.TOWERS:
        k1, b1 = st.entries[f"{tower}/classifier_mlp1/kernel"], st.entries[f"{tower}/classifier_mlp1/bias"]
        assert (k1.shape, k1.ref_cols, b1.shape, b1.ref_cols) == ((cfg["hidden_size"] // 2, 8), 1, (8,), 1)
        # hyper-parameter groups from hyper_for like every other variable: kernels decay, biases do not
        assert st.entries[f"{tower}/classifier_mlp0/kernel"].hyper[1] == pytest.approx(0.01)
        assert st.entries[f"{tower}/classifier_mlp0/bias"].hyper[1] == 0.0 and b1.hyper[1] == 0.0
        assert st.entries[f"{tower}/classifier_mlp0/kernel"].hyper[0] == pytest.approx(1.2e-5)


def test_tower_initial_values_and_round_trip(tiny_cfg):
    from merlot_b200.params import ParamStore
    H = tiny_cfg["hidden_size"]
    st = ParamStore(tiny_cfg, device="cpu", task="vcr")
    st.init_reference(seed=4)
    for tower in V.TOWERS:
        k0, b0 = st.P(f"{tower}/classifier_mlp0/kernel"), st.P(f"{tower}/classifier_mlp0/bias")
        k1, b1 = st.P(f"{tower}/classifier_mlp1/kernel"), st.P(f"{tower}/classifier_mlp1/bias")
        assert k0.abs().max() <= 0.04 and 0.012 < float(k0.std()) < 0.02  # truncated normal(0.02) within 2 sigma
        assert k1[:, 0].abs().max() <= 0.04 and float(k1[:, 0].std()) > 0.01 and torch.all(k1[:, 1:] == 0)
        assert torch.all(b0 == 0)
        assert float(b1[0]) == pytest.approx(-math.log(3.0)) and torch.all(b1[1:] == 0)
    tf = st.to_tf_dict("p")
    assert tuple(tf["answer_cls/classifier_mlp1/kernel"].shape) == (H // 2, 1)
    assert tuple(tf["rationale_cls/classifier_mlp1/bias"].shape) == (1,)
    vals = V.init_params(tiny_cfg, seed=9, perturb=0.1)
    st.load_tf_dict(vals)
    back = st.to_tf_dict("p")
    for k, v in vals.items():
        assert tuple(back[k].shape) == tuple(v.shape) and torch.equal(back[k], v.float()), k
    for tower in V.TOWERS:  # the padding columns stay zero
        assert torch.all(st.P(f"{tower}/classifier_mlp1/kernel")[:, 1:] == 0)
        assert torch.all(st.P(f"{tower}/classifier_mlp1/bias")[1:] == 0)


def test_init_checkpoint_from_a_pretraining_checkpoint(tmp_path, tiny_cfg):
    """A pretraining checkpoint restores every backbone variable of the VCR graph by name; exactly the 8 tower variables are
    reported missing and keep their initial values; its pretraining-only variables are ignored (model/modeling.py:724-740)."""
    from merlot_b200.params import ParamStore
    from oracle import merlot_oracle as O
    from tests.test_tf_checkpoint import _write_checkpoint
    pre = O.init_params(tiny_cfg, seed=3, perturb=0.1)
    prefix = str(tmp_path / "model.ckpt-460000")
    _write_checkpoint(prefix, pre)
    st = ParamStore(tiny_cfg, device="cpu", task="vcr")
    st.init_reference(seed=0)
    towers0 = {k: v.clone() for k, v in st.to_tf_dict("p").items() if k.split("/")[0] in V.TOWERS}
    missing = st.load_checkpoint(prefix)
    assert sorted(missing) == sorted(f"{t}/classifier_mlp{i}/{w}" for t in V.TOWERS for i in (0, 1) for w in ("kernel", "bias"))
    back = st.to_tf_dict("p")
    for k, v in back.items():
        if k in towers0:
            assert torch.equal(v, towers0[k]), k
        else:
            assert torch.equal(v, pre[k]), k


def test_vcr_step_applies_init_checkpoint(tmp_path, tiny_cfg):
    """vcr_model_fn_builder restores model.init_checkpoint into the store it builds, and a prefix without an .index file
    raises instead of training from the initialisers."""
    from merlot_b200.vcr import vcr_model_fn_builder
    from oracle import merlot_oracle as O
    from tests.test_tf_checkpoint import _write_checkpoint
    pre = O.init_params(tiny_cfg, seed=5)
    prefix = str(tmp_path / "model.ckpt-1")
    _write_checkpoint(prefix, pre)
    fn = vcr_model_fn_builder(vcr_config(tiny_cfg, init_checkpoint=prefix), device="cpu")
    got = fn.store.to_tf_dict("p")
    assert torch.equal(got["word_embeddings/word_embeddings"], pre["word_embeddings/word_embeddings"])
    assert fn.store.task == "vcr"
    with pytest.raises(FileNotFoundError):
        vcr_model_fn_builder(vcr_config(tiny_cfg, init_checkpoint=str(tmp_path / "missing.ckpt")), device="cpu")


def test_synthetic_vcr_batch_and_cli_dispatch(tiny_cfg):
    from merlot_b200 import train
    from merlot_b200.config import NeatConfig
    from merlot_b200.modeling import START
    from merlot_b200.vcr import vcr_model_fn_builder
    cfg = vcr_config(tiny_cfg)
    f = train.synthetic_vcr_batch(cfg, 3, seed=1, device="cpu")
    assert tuple(f["images"].shape) == (6, 64, 96, 3) and f["images"].dtype == torch.bfloat16
    assert tuple(f["lm_input"].shape) == (24, 184) and f["lm_input"].dtype == torch.int32
    ids = f["lm_input"]
    assert torch.all(ids[:, 0] == START)
    body = ids[:, 1:]
    assert torch.all((body == 0) | ((body >= 100) & (body < tiny_cfg["vocab_size"])))
    # a zero-padded tail: once a text has ended it stays ended
    nz = (ids != 0).int()
    assert torch.all(nz[:, 1:] <= nz[:, :-1])
    t = f["lm_targets"]
    assert tuple(t.shape) == (6,) and t.dtype == torch.int32 and int(t.min()) >= 0 and int(t.max()) < 4
    assert not torch.equal(train.synthetic_vcr_batch(cfg, 3, seed=2, device="cpu")["lm_input"], ids)
    assert train._step_for(cfg) == (vcr_model_fn_builder, train.synthetic_vcr_batch)
    pre = NeatConfig.from_dict({"data": {}, "model": dict(tiny_cfg), "optimizer": dict(VCR_YAML_OPTIMIZER),
                                "device": {"output_dir": "/tmp/x"}})
    assert train._step_for(pre) == (train.model_fn_builder, train.synthetic_batch)
