"""share_params: False on the host: the separate `langonly_encoder/` stack in the parameter arena against the oracle's
variable list, the full-size counts, the shared layout left as it was, the data-parallel split, the variable lists of the
programs that read checkpoints, and the multi-image refusal."""
import os
import sys

import pytest
import torch

from merlot_b200.params import ParamStore
from tests import share_params_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OCFG = {"learning_rate": 3e-4, "weight_decay_rate": 0.1,
        "param_overrides": [[["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]]}


def _separate(cfg):
    return dict(cfg, share_params=False, num_hidden_layers=2, num_lang_transformer_hidden_layers=3)


def _bench_model():
    sys.path.insert(0, ROOT)
    import bench
    return bench.load_config().model


def _layout(st):
    return [(e.name, e.shape, e.tf_names, e.offset, e.padded, e.hyper) for e in st.entries.values()]


def test_arena_matches_oracle_and_round_trips(tiny_cfg, monkeypatch):
    from oracle import merlot_oracle as O
    SO.use_separate_oracle(monkeypatch)
    cfg = _separate(tiny_cfg)
    shapes = O.param_shapes(cfg)
    lo = [k for k in shapes if k.startswith("langonly_encoder/")]
    assert len(lo) == 3 * 16 + 2 and "langonly_encoder/layer02/key_layer/kernel" in shapes
    assert not any(k.startswith("encoder/layer02/") for k in shapes)
    st = ParamStore(cfg, device="cpu")
    views = {nm: tuple(t.shape) for _, nm, t in st.tf_views(st.p)}
    assert views == {k: tuple(v) for k, v in shapes.items()}
    params = O.init_params(cfg, seed=0, perturb=0.1)
    st.load_tf_dict(params)
    back = st.to_tf_dict("p")
    assert set(back) == set(params)
    for k in params:
        assert torch.equal(back[k], params[k]), k
    assert st.num_params() == sum(v.numel() for v in params.values())


def test_oracle_extension_leaves_the_shared_oracle_alone(tiny_cfg):
    from oracle import merlot_oracle as O
    for cfg in (tiny_cfg, dict(tiny_cfg, share_params=True), dict(tiny_cfg, num_lang_transformer_hidden_layers=3)):
        assert list(SO.param_shapes(cfg).items()) == list(O.param_shapes(cfg).items())


def test_full_size_counts():
    model = _bench_model()
    shared = ParamStore(model, device="meta")
    sep = ParamStore(dict(model, share_params=False), device="meta")
    assert (shared.num_params(), shared.total) == (223_423_946, 223_430_272)
    assert (sep.num_params(), sep.total) == (308_479_946, 308_486_272)
    lo = [e for e in sep.entries.values() if e.name.startswith("langonly_encoder/")]
    assert sum(e.numel for e in lo) == 308_479_946 - 223_423_946 == 85_056_000


def test_shared_layout_unchanged(tiny_cfg):
    model = _bench_model()
    absent = {k: v for k, v in model.items() if k != "share_params"}
    for base in (model, tiny_cfg, dict(tiny_cfg, num_lang_transformer_hidden_layers=3)):
        a = ParamStore({k: v for k, v in base.items() if k != "share_params"}, device="meta", optimizer_cfg=OCFG)
        b = ParamStore(dict(base, share_params=True), device="meta", optimizer_cfg=OCFG)
        assert _layout(a) == _layout(b) and a.total == b.total and a.groups == b.groups
        assert not any(n.startswith("langonly_encoder/") for n in a.entries)
    assert ParamStore(absent, device="meta").total == 223_430_272


def test_vcr_ignores_the_switch(tiny_cfg):
    cfg = dict(tiny_cfg, num_texts=4, num_chunks_in_group=1)
    a = ParamStore(cfg, device="meta", task="vcr")
    b = ParamStore(dict(cfg, share_params=False), device="meta", task="vcr")
    assert _layout(a) == _layout(b) and a.total == b.total


@pytest.mark.parametrize("full", [False, True])
def test_langonly_encoder_is_outside_the_vit_buckets(tiny_cfg, full):
    model = _bench_model() if full else tiny_cfg
    shared = ParamStore(model, device="meta", optimizer_cfg=OCFG)
    sep = ParamStore(dict(model, share_params=False), device="meta", optimizer_cfg=OCFG)
    lo = [e for e in sep.entries.values() if e.name.startswith("langonly_encoder/")]
    assert lo
    for e in lo:
        assert any(a <= e.offset and e.offset + e.padded <= b for a, b in sep.rest_ranges), e.name
        assert not any(a < e.offset + e.padded and e.offset < b for a, b in sep.vit_ranges), e.name
    # the same ViT buckets: same layer groups, each bucket over the same variables (the offsets of the second
    # hyper-parameter group move by the size of the decayed langonly_encoder/ kernels)
    def buckets(st):
        groups, ranges = st.vit_buckets()
        return groups, [sorted(e.name for e in st.entries.values() if any(a <= e.offset < b for a, b in r)) for r in ranges]
    assert buckets(sep) == buckets(shared)
    assert sep.vit_ranges[0] == shared.vit_ranges[0]
    covered = sum(b - a for a, b in sep.vit_ranges + sep.rest_ranges)
    assert covered == sep.total


def test_program_variable_lists(tiny_cfg):
    from merlot_b200.sort_story import zero_shot_variables
    from merlot_b200.train import variables_without_gradient
    for extra in ({}, {"image_shuffle_prob": 0.0}, {"temporal_coef": 0.0}):
        shared_cfg = dict(_separate(tiny_cfg), share_params=True, **extra)
        sep_cfg = dict(_separate(tiny_cfg), **extra)
        shared = ParamStore(shared_cfg, device="meta", optimizer_cfg=OCFG)
        sep = ParamStore(sep_cfg, device="meta", optimizer_cfg=OCFG)
        zs = zero_shot_variables(sep)
        assert not any(n.startswith("langonly_encoder/") for n in zs)
        assert zs == zero_shot_variables(shared)  # the joint encoder's variables, in both layouts
        skip = variables_without_gradient(sep_cfg, sep)
        assert skip == variables_without_gradient(shared_cfg, shared)
        assert not any(n.startswith("langonly_encoder/") for n in skip)
        slotted = {e.name for e in sep.slot_entries(skip)}
        lo = {n for n in sep.entries if n.startswith("langonly_encoder/")}
        assert len(lo) == 3 * 12 + 2 and lo <= slotted


def test_multi_image_refuses_separate_encoder(tiny_cfg):
    from merlot_b200.modeling import check_num_imgs
    cfg = dict(tiny_cfg, share_params=False, num_chunks_in_group=1)
    with pytest.raises(NotImplementedError, match="share_params"):
        check_num_imgs(dict(cfg, num_imgs=2), batch_size=2, num_chunks=1, B=2, n_images=4)
    with pytest.raises(NotImplementedError, match="share_params"):
        check_num_imgs(cfg, batch_size=2, num_chunks=1, B=2, n_images=2, img_mask=torch.ones(2, 1, dtype=torch.bool))
    # one image per text: the switch is the pretraining path's, nothing to refuse
    assert check_num_imgs(cfg, batch_size=2, num_chunks=1, B=2, n_images=2) == 1
    assert check_num_imgs(dict(cfg, num_imgs=2, share_params=True), batch_size=2, num_chunks=1, B=2, n_images=4) == 2
