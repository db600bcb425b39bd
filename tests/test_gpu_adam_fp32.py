"""AdamW with fp32 moments on the GPU (pytest -m gpu): use_bfloat16_adam: False, the reference's default
(utils/optimization.py:58,305).  K10's fp32 instance against AdamOracle bit for bit, the data-parallel bucketed update, a
pretraining step, checkpoints with DT_FLOAT slots (round trip, a reference-default bundle, mismatches with bf16 slots) and
the trainer's save / resume loop."""
import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import ops
from merlot_b200 import tf_checkpoint as T
from oracle import merlot_oracle as O
from tests import test_gpu_checkpoint as CK

pytestmark = pytest.mark.gpu
DEV = "cuda"
OCFG = {k: v for k, v in CK.OCFG.items() if k != "use_bfloat16_adam"}  # the flag left out: the reference's default, False


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _config_dict(model_cfg, task=None, **opt):
    d = {"data": {"num_chunks": 4, "chunk_text_len": 16}, "model": dict(model_cfg, image_size=[64, 96]),
         "optimizer": dict(OCFG, **opt), "device": {"output_dir": "/tmp/unused", "train_batch_size": 2}}
    if task:
        d["downstream"] = {"task": task, "mode": "answer"}
    return d


def _config(model_cfg, task=None, **opt):
    from merlot_b200.config import NeatConfig
    return NeatConfig.from_dict(_config_dict(model_cfg, task, **opt))


# ---- K10 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grad_scale", [1.0, 0.25])
@pytest.mark.parametrize("zero_grad", [True, False])
def test_adamw_f32_moments_vs_oracle(grad_scale, zero_grad):
    """25 steps on n = 100003 (12500 vector threads and a 3-element scalar tail), gradients from 1e-6 to 1, a decayed and a
    no-decay tensor: m and v bit for bit equal to AdamOracle(use_bfloat16_adam=False), p within 1e-6."""
    g = torch.Generator().manual_seed(1)
    n = 100003
    cfg = dict(learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=10, weight_decay_rate=0.1, beta_2=0.98, epsilon=1e-6,
               use_bfloat16_adam=False, param_overrides=[[["bias"], {"weight_decay_rate": 0}]])
    p_ref = {"w/kernel": torch.randn(n, generator=g) * 0.02, "w/bias": torch.randn(n, generator=g) * 0.02}
    opt = O.AdamOracle(p_ref, cfg)
    assert opt.m["w/kernel"].dtype == torch.float32
    dev = {k: dict(p=v.clone().to(DEV), m=torch.zeros(n, device=DEV), v=torch.zeros(n, device=DEV),
                   pb=torch.zeros(n, dtype=torch.bfloat16, device=DEV)) for k, v in p_ref.items()}
    for step in range(25):
        grads = {k: torch.randn(n, generator=g) * (10.0 ** float(torch.randint(-6, 1, (1,), generator=g))) for k in p_ref}
        s = opt.step_scalars()
        opt.apply_gradients(p_ref, {k: v * grad_scale for k, v in grads.items()})  # exact: grad_scale is a power of two
        for k, d in dev.items():
            gd = grads[k].to(DEV)
            wd = 0.1 if "kernel" in k else 0.0
            ops.adamw_step(d["p"], gd, d["m"], d["v"], d["pb"], n, float(s["beta1"]), float(np.float32(1) - s["beta1"]),
                           float(s["beta2"]), float(np.float32(1) - s["beta2"]), float(s["eps"]), float(s["lr_t"]), wd,
                           grad_scale, zero_grad)
            if zero_grad:
                assert float(gd.abs().max()) == 0.0
            else:
                assert torch.equal(gd.cpu(), grads[k])
    for k, d in dev.items():
        assert torch.equal(_bits(d["m"].cpu()), _bits(opt.m[k])), "first moment must be bit-exact"
        assert torch.equal(_bits(d["v"].cpu()), _bits(opt.v[k])), "second moment must be bit-exact"
        assert (d["p"].cpu() - p_ref[k]).abs().max().item() < 1e-6
        assert torch.equal(d["pb"].cpu(), d["p"].cpu().bfloat16())


def _random_store(cfg, seed):
    from merlot_b200.optimization import AdamOptimizer
    from merlot_b200.params import ParamStore
    st = ParamStore(cfg, device=DEV, optimizer_cfg=OCFG)
    assert st.m.dtype == st.v.dtype == torch.float32
    gen = torch.Generator(device=DEV).manual_seed(seed)
    st.p.copy_(torch.randn(st.total, generator=gen, device=DEV) * 0.02)
    st.sync_bf16()
    st.m.copy_(torch.randn(st.total, generator=gen, device=DEV) * 1e-3)
    st.v.copy_(torch.rand(st.total, generator=gen, device=DEV) * 1e-6)
    st.g.copy_(torch.randn(st.total, generator=gen, device=DEV))
    st.global_step = 7
    return st, AdamOptimizer(st, **{k: v for k, v in OCFG.items() if k != "type"})


def test_bucketed_update_equals_one_call(tiny_cfg):
    """The data-parallel call pattern of train.py (rest_ranges, then each ViT bucket, the last one advancing the step) on a
    store with fp32 moments is bitwise the single apply_gradients() call."""
    a, opt_a = _random_store(tiny_cfg, 5)
    b, opt_b = _random_store(tiny_cfg, 5)
    skip = ["viz_viz_temporal/logits/bias"]
    opt_a.apply_gradients(grad_scale=0.5, skip=skip)
    _, vit_ranges = b.vit_buckets(2)
    opt_b.apply_gradients(grad_scale=0.5, skip=skip, only=b.rest_ranges, advance=False)
    assert b.global_step == 7
    for k, rs in enumerate(vit_ranges):
        opt_b.apply_gradients(grad_scale=0.5, skip=skip, only=rs, advance=(k + 1 == len(vit_ranges)))
    torch.cuda.synchronize()
    for x, y in ((a.p, b.p), (a.pb, b.pb), (a.m, b.m), (a.v, b.v), (a.g, b.g)):
        assert torch.equal(_bits(x), _bits(y))
    assert a.global_step == b.global_step == 8
    e = a.entries[skip[0]]
    assert float(a.g[e.offset:e.offset + e.padded].abs().max()) == 0.0  # skipped, its gradient still zeroed


# ---- one pretraining step ------------------------------------------------------------------------------------------
def test_pretrain_step_parity_f32_moments(tiny_cfg):
    """tests/test_gpu_model.py's tiny pretraining step with the moments in fp32: forward, the three losses, backward, then
    one AdamW step against AdamOracle fed the GPU gradients -- parameters within 2e-6, adam_m / adam_v bit for bit."""
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.optimization import build_optimizer_from_config
    from merlot_b200.params import ParamStore
    from tests.test_gpu_model import check_adam_step, rel, synth
    cfg = tiny_cfg
    batch, nc, Lc = 2, 4, 16
    image, ids, shuf, vid = synth(cfg, batch, nc, Lc, 64, 96, 0)
    params = O.init_params(cfg, seed=1, perturb=0.05)
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    ocfg = dict(OCFG, num_warmup_steps=10)
    store = ParamStore(cfg, device=DEV, optimizer_cfg=ocfg)
    store.load_tf_dict(params)
    B, Lj = batch * nc // cfg["num_chunks_in_group"], Lc * cfg["num_chunks_in_group"]
    draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), cfg["vocab_size"], seed=5)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                    shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, save_for_backward=True)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm)
    ll, _ = m.mask_loss()
    cl, _ = m.contrastive_loss()
    tl, _ = m.temporal_loss(shuf.to(DEV), vid.to(DEV))
    total_ref, _ = O.pretrain_losses(om, shuf, vid)
    total = float(ll) + float(cl) + float(tl)
    ref = float(total_ref.detach())
    assert abs(total - ref) <= 1e-3 * abs(ref)
    store.g.zero_()
    m.backward()
    total_ref.backward()
    grads = store.to_tf_dict("g")
    for k, v in leaf.items():
        if v.grad is None or float(v.grad.norm()) < 1e-7:
            continue
        assert rel(grads[k], v.grad) < 4e-2, k
    # taken at the end of the warm-up: at step 0 the learning rate is 0 and the parameters could not move on either side
    check_adam_step(store, build_optimizer_from_config(None, ocfg, None, store=store)[0], ocfg, grads)
    assert store.m.dtype == store.v.dtype == torch.float32


# ---- checkpoints ---------------------------------------------------------------------------------------------------
def _round_trip(config, tmp_path):
    """test_gpu_checkpoint's round trip (2 steps, save, restore into a fresh store, the next forward and AdamW update bit for
    bit) with fp32 moments: every slot is DT_FLOAT and equals the arena bit for bit.  Returns (trained store, prefix); the
    store has taken one more step since the save."""
    fn = CK._trained(config)
    st = fn.store
    assert st.m.dtype == torch.float32
    prefix = str(tmp_path / "model.ckpt-2")
    st.save_checkpoint(prefix)
    got = T.load_checkpoint(prefix, skip_optimizer_slots=False)
    for suffix, buf in (("adam_m", st.m), ("adam_v", st.v)):
        for _, nm, t in st.tf_views(buf):
            g = got[f"{nm}/{suffix}"]
            assert g.dtype == torch.float32 and list(g.shape) == list(t.shape), nm
            assert torch.equal(_bits(g), _bits(t.cpu().contiguous())), nm
    assert all(dt == T.DT_FLOAT for nm, dt, _ in st._checkpoint_tensors(()) if nm.endswith(("/adam_m", "/adam_v")))
    fn2 = CK._trained(config, steps=0)
    st2 = fn2.store
    st2.p.normal_()
    st2.m.fill_(1.0)
    st2.v.fill_(-1.0)
    st2.global_step = 123
    st2.restore_checkpoint(prefix)
    mask = CK._variable_mask(st)
    CK._assert_same_state(st, st2, mask)
    feats = CK._batch(config, 9)
    s1, s2 = fn(feats, None, "train", None), fn2(feats, None, "train", None)
    for x, y in zip(s1.loss_parts, s2.loss_parts):
        assert torch.equal(torch.as_tensor(x).float(), torch.as_tensor(y).float()), (float(x), float(y))
    del s1, s2
    g = torch.randn(st.total, generator=torch.Generator().manual_seed(3)).to(DEV) * mask
    for f in (fn, fn2):
        f.store.g.copy_(g)
        f.optimizer.apply_gradients()
    torch.cuda.synchronize()
    CK._assert_same_state(st, st2, mask)
    return st, prefix


def test_pretrain_state_round_trip_f32_moments(tmp_path, tiny_cfg):
    _round_trip(_config(tiny_cfg), tmp_path)


def test_vcr_state_round_trip_f32_moments(tmp_path, tiny_cfg):
    """The VCR store, and the validator restoring the trainer's checkpoint from the same config."""
    from merlot_b200.config import NeatConfig
    from merlot_b200.vcr_validate import Validator
    d = _config_dict(CK._vcr_cfg(tiny_cfg), task="vcr")
    _, prefix = _round_trip(NeatConfig.from_dict(d), tmp_path)
    d["device"]["val_batch_size"] = 2
    d["validate"] = {"eval_samples": 2}
    val = Validator(NeatConfig.from_dict(d), device=DEV)
    assert val.store.m.dtype == torch.float32
    val.store.restore_checkpoint(prefix)
    got = T.load_checkpoint(prefix, skip_optimizer_slots=False)
    assert val.store.global_step == int(got["global_step"]) == 2
    for suffix, buf in (("", val.store.p), ("/adam_m", val.store.m), ("/adam_v", val.store.v)):
        for _, nm, t in val.store.tf_views(buf):
            assert torch.equal(_bits(t.cpu().contiguous()), _bits(got[nm + suffix])), nm + suffix


def _reference_default_bundle(store, prefix, seed):
    """What the reference's Saver writes with use_bfloat16_adam False: every variable DT_FLOAT, every slot DT_FLOAT (seeded
    random moments, v > 0), global_step int64.  Returns the variables and slots as reference-named CPU tensors."""
    g = torch.Generator().manual_seed(seed)
    params = {nm: (torch.randn(t.shape, generator=g) * 0.02) for _, nm, t in store.tf_views(store.p)}
    slots = {}
    for _, nm, t in store.tf_views(store.p):
        slots[f"{nm}/adam_m"] = torch.randn(t.shape, generator=g) * 1e-3
        slots[f"{nm}/adam_v"] = torch.rand(t.shape, generator=g) * 1e-6
    entries = [("global_step", T.DT_INT64, (), np.int64(11).tobytes(), None)]
    for nm, t in list(params.items()) + list(slots.items()):
        entries.append((nm, T.DT_FLOAT, tuple(t.shape), t.contiguous().numpy().tobytes(), None))
    T.write_bundle(prefix, entries)
    return params, slots


def test_restore_reference_default_checkpoint(tmp_path, tiny_cfg):
    """A bundle with fp32 slots as the reference writes them by default restores, and the next update of every variable
    matches AdamOracle started from those moments: m and v bit for bit, parameters within 2e-6."""
    from merlot_b200.optimization import AdamOptimizer
    from merlot_b200.params import ParamStore
    ocfg = dict(OCFG, num_warmup_steps=1)
    st = ParamStore(tiny_cfg, device=DEV, optimizer_cfg=ocfg)
    prefix = str(tmp_path / "model.ckpt-11")
    params, slots = _reference_default_bundle(st, prefix, 0)
    st.restore_checkpoint(prefix)
    assert st.global_step == 11
    opt = AdamOptimizer(st, **{k: v for k, v in ocfg.items() if k != "type"})
    adam = O.AdamOracle({k: v.clone() for k, v in params.items()}, ocfg)
    ref_p = {k: v.clone() for k, v in params.items()}
    for nm in params:
        adam.m[nm], adam.v[nm] = slots[f"{nm}/adam_m"].clone(), slots[f"{nm}/adam_v"].clone()
    adam.global_step = 11
    gen = torch.Generator().manual_seed(1)
    grads = {nm: torch.randn(t.shape, generator=gen) for nm, t in params.items()}
    for _, nm, t in st.tf_views(st.g):
        t.copy_(grads[nm])
    adam.apply_gradients(ref_p, grads)
    opt.apply_gradients()
    torch.cuda.synchronize()
    for (_, nm, tm), (_, _, tv), (_, _, tp) in zip(st.tf_views(st.m), st.tf_views(st.v), st.tf_views(st.p)):
        assert torch.equal(_bits(tm.cpu().contiguous()), _bits(adam.m[nm].contiguous())), nm
        assert torch.equal(_bits(tv.cpu().contiguous()), _bits(adam.v[nm].contiguous())), nm
        assert (tp.cpu() - ref_p[nm]).abs().max().item() < 2e-6, nm
    assert st.global_step == 12


def test_slot_format_mismatches(tmp_path, tiny_cfg):
    """bf16 slots into an fp32 store and fp32 slots into a bf16 store both raise, naming a slot and the flag; an fp32 VCR
    store still initialises from a bf16-slot pretraining checkpoint (init_checkpoint skips slots) and trains."""
    f32 = CK._trained(_config(tiny_cfg), steps=1)
    b16 = CK._trained(CK._config(tiny_cfg), steps=1)
    assert f32.store.m.dtype == torch.float32 and b16.store.m.dtype == torch.bfloat16
    p32, p16 = str(tmp_path / "f32.ckpt-1"), str(tmp_path / "bf16.ckpt-1")
    f32.store.save_checkpoint(p32)
    b16.store.save_checkpoint(p16)
    with pytest.raises(T.CheckpointFormatError, match=r"/adam_[mv]: .*use_bfloat16_adam: True.*use_bfloat16_adam: False"):
        f32.store.restore_checkpoint(p16)
    with pytest.raises(T.CheckpointFormatError, match=r"/adam_[mv]: .*use_bfloat16_adam: False.*use_bfloat16_adam: True"):
        b16.store.restore_checkpoint(p32)
    vcfg = _config(CK._vcr_cfg(tiny_cfg), task="vcr")
    fn = CK._trained(vcfg, steps=0)
    st = fn.store
    assert st.m.dtype == torch.float32
    missing = st.load_checkpoint(p16)
    assert missing and all(n.startswith(("answer_cls/", "rationale_cls/")) for n in missing)
    e = st.entries["encoder/layer00/intermediate/kernel"]
    assert torch.equal(st.P(e.name).cpu(), b16.store.P(e.name).cpu())
    fn(CK._batch(vcfg, 0), None, "train", None).train_op()
    torch.cuda.synchronize()
    assert st.global_step == 1 and float(st.m.abs().max()) > 0 and torch.isfinite(st.p).all()


# ---- the trainer ---------------------------------------------------------------------------------------------------
def _yaml(tmp_path, tiny_cfg, steps, out):
    cfg = {"data": {"num_chunks": 4, "chunk_text_len": 16}, "model": dict(tiny_cfg, image_size=[64, 96], vocab_size=50370),
           "optimizer": dict(OCFG, num_train_steps=steps),
           "device": {"output_dir": str(out), "train_batch_size": 2, "iterations_per_loop": 2}}
    assert "use_bfloat16_adam" not in cfg["optimizer"]
    path = tmp_path / f"run{steps}.yaml"
    path.write_text(yaml.safe_dump(cfg))
    return str(path)


def test_trainer_saves_and_resumes_f32_moments(tmp_path, tiny_cfg, capsys):
    """A YAML without use_bfloat16_adam trains, saves fp32 slots and resumes from its own checkpoint."""
    from merlot_b200.train import main
    out = tmp_path / "out"
    main([_yaml(tmp_path, tiny_cfg, 3, out)])
    assert T.latest_checkpoint(str(out)) == str(out / "model.ckpt-3")
    slots = {nm: dt for nm, dt in ((nm, e["dtype"]) for nm, e in T._index(str(out / "model.ckpt-3"), True)[1].items())
             if nm.endswith(("/adam_m", "/adam_v"))}
    assert slots and all(int(dt) == T.DT_FLOAT for dt in slots.values())
    capsys.readouterr()
    main([_yaml(tmp_path, tiny_cfg, 5, out)])
    log = capsys.readouterr().out
    assert "continuing from global_step 3" in log, log
    assert int(T.load_checkpoint(str(out / "model.ckpt-5"), names=["global_step"])["global_step"]) == 5


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_resume_f32_moments(tmp_path, tiny_cfg):
    """test_gpu_checkpoint's two-rank save and resume with fp32 moments: after the resume both ranks hold bitwise the same
    parameters and moments."""
    import torch.multiprocessing as mp
    out = tmp_path / "out"
    y3, y4 = _yaml(tmp_path, tiny_cfg, 3, out), _yaml(tmp_path, tiny_cfg, 4, out)
    world, port = 2, CK._free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=CK._dist_worker, args=(r, world, port, y3, y4, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in ps:
        p.join(timeout=120)
    for r in res:
        assert "error" not in r, r.get("error")
    assert all(r["identical"] and r["step"] == 4 for r in res)
    assert T._index(str(out / "model.ckpt-4"), True)[1]["encoder/layer00/intermediate/kernel/adam_v"]["dtype"] == T.DT_FLOAT
