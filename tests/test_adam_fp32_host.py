"""fp32 Adam moments on the host (no GPU): which moment format a ParamStore keeps for use_bfloat16_adam (the reference
defaults it to False, utils/optimization.py:58,305), AdamOptimizer refusing a store of the other format, ops.adamw_step
refusing mixed moment dtypes before any launch, and the DT_FLOAT slots a checkpoint of such a store lists."""
import pytest
import torch

OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=1, weight_decay_rate=0.1,
            beta_2=0.98, clip_norm=0.0,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]])


def _store(tiny_cfg, ocfg, **kw):
    from merlot_b200.params import ParamStore
    return ParamStore(tiny_cfg, device="cpu", optimizer_cfg=ocfg, **kw)


@pytest.mark.parametrize("flag,dtype", [("missing", torch.float32), (False, torch.float32), (True, torch.bfloat16),
                                        ("no_optimizer_cfg", torch.bfloat16)])
def test_moment_dtype_follows_the_flag(tiny_cfg, flag, dtype):
    if flag == "no_optimizer_cfg":
        st = _store(tiny_cfg, None)
    else:
        st = _store(tiny_cfg, OCFG if flag == "missing" else dict(OCFG, use_bfloat16_adam=flag))
    assert st.moment_dtype == st.m.dtype == st.v.dtype == dtype
    assert st.m.numel() == st.v.numel() == st.total
    assert st.p.dtype == st.g.dtype == torch.float32 and st.pb.dtype == torch.bfloat16


def test_vcr_store_follows_the_flag(tiny_cfg):
    cfg = dict(tiny_cfg, num_texts=4, num_chunks_in_group=1)
    assert _store(cfg, OCFG, task="vcr").m.dtype == torch.float32
    assert _store(cfg, dict(OCFG, use_bfloat16_adam=True), task="vcr").m.dtype == torch.bfloat16


def test_optimizer_refuses_a_store_of_the_other_format(tiny_cfg):
    from merlot_b200.optimization import build_optimizer_from_config
    for store_flag, opt_flag in ((False, True), (True, False)):
        st = _store(tiny_cfg, dict(OCFG, use_bfloat16_adam=store_flag))
        with pytest.raises(ValueError, match="use_bfloat16_adam"):
            build_optimizer_from_config(None, dict(OCFG, use_bfloat16_adam=opt_flag), store=st)
    for flag in (False, True):  # matching formats build
        st = _store(tiny_cfg, dict(OCFG, use_bfloat16_adam=flag))
        opt, _ = build_optimizer_from_config(None, dict(OCFG, use_bfloat16_adam=flag), store=st)
        assert opt.store is st
    opt, _ = build_optimizer_from_config(None, OCFG, store=_store(tiny_cfg, OCFG))  # flag left out on both sides
    assert opt.store.m.dtype == torch.float32


@pytest.mark.parametrize("mdt,vdt", [(torch.float32, torch.bfloat16), (torch.bfloat16, torch.float32),
                                     (torch.float16, torch.float16)])
def test_adamw_step_refuses_mixed_moments_before_launch(monkeypatch, mdt, vdt):
    from merlot_b200 import _lib as L
    from merlot_b200 import ops

    def no_library():
        raise AssertionError("adamw_step reached the library")
    monkeypatch.setattr(L, "lib", no_library)
    n = 16
    p, g, pb = torch.zeros(n), torch.zeros(n), torch.zeros(n, dtype=torch.bfloat16)
    with pytest.raises(L.MerlotError, match="both float32 or both bfloat16"):
        ops.adamw_step(p, g, torch.zeros(n, dtype=mdt), torch.zeros(n, dtype=vdt), pb, n, 0.9, 0.1, 0.98, 0.02, 1e-6, 1e-3,
                       0.0, 1.0, True)


def test_checkpoint_lists_float_slots_for_fp32_moments(tiny_cfg):
    from merlot_b200.tf_checkpoint import DT_BFLOAT16, DT_FLOAT, DT_INT64
    for flag, slot_dt in ((False, DT_FLOAT), (True, DT_BFLOAT16)):
        st = _store(tiny_cfg, dict(OCFG, use_bfloat16_adam=flag))
        ts = st._checkpoint_tensors(())
        assert DT_INT64 not in {dt for _, dt, _ in ts}
        params = [(nm, dt) for nm, dt, _ in ts if not nm.endswith(("/adam_m", "/adam_v"))]
        slots = [(nm, dt, t) for nm, dt, t in ts if nm.endswith(("/adam_m", "/adam_v"))]
        assert len(slots) == 2 * len(params) and all(dt == DT_FLOAT for _, dt in params)
        # data-file order: the parameters, then every adam_m, then every adam_v
        assert [nm for nm, _, _ in ts] == [nm for nm, _ in params] + [f"{nm}/adam_m" for nm, _ in params] + \
            [f"{nm}/adam_v" for nm, _ in params]
        for nm, dt, t in slots:
            assert dt == slot_dt and t.dtype == st.m.dtype, nm
