"""Saving and resuming training on the GPU (pytest -m gpu): K15 (merlot_crc32c_multi) against the NumPy CRC-32C, the whole
training state through ParamStore.save_checkpoint / restore_checkpoint (pretraining, VCR, hybrid stem), corruption and
mismatch errors, and the trainer's save / resume loop."""
import os
import socket

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import ops
from merlot_b200 import tf_checkpoint as T

pytestmark = pytest.mark.gpu
DEV = "cuda"
OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=1, weight_decay_rate=0.1,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]])


# ---- K15 ----------------------------------------------------------------------------------------------------------
def _dev(b: bytes) -> torch.Tensor:
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(DEV) if b else torch.empty(0, dtype=torch.uint8, device=DEV)


def test_crc32c_known_answers():
    vecs = {b"123456789": 0xE3069283, bytes(32): 0x8A9136AA, b"\xff" * 32: 0x62A8AB43,  # RFC 3720 B.4
            bytes(range(32)): 0x46DD794E, bytes(range(31, -1, -1)): 0x113FDB5C, b"": 0}
    got = ops.crc32c_multi([_dev(v) for v in vecs])
    assert got == list(vecs.values()) == [T.crc32c(v) for v in vecs]


def test_crc32c_every_short_length_and_offset():
    """Every length 0..300 at every start offset 0..15 (4816 segments, one launch): heads, tails and the 16-byte body."""
    rng = np.random.default_rng(0)
    host = rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()
    buf = _dev(host)
    segs = [(o, n) for o in range(16) for n in range(301)]
    got = ops.crc32c_multi([buf[o:o + n] for o, n in segs])
    want = [T.crc32c(host[o:o + n]) for o, n in segs]
    assert got == want
    out = torch.full((len(segs),), 7, dtype=torch.int32, device=DEV)  # device-resident result, old contents overwritten
    assert ops.crc32c_multi([buf[o:o + n] for o, n in segs], out=out) is out
    assert out.cpu().numpy().view(np.uint32).tolist() == want


def test_crc32c_long_segments_across_chunk_boundaries():
    """Lengths at the kernel's lane (1 KiB) and chunk (32 KiB) boundaries +-1 and random lengths up to 6 MB at random
    unaligned starts, all in one launch."""
    rng = np.random.default_rng(1)
    host = rng.integers(0, 256, 8 << 20, dtype=np.uint8).tobytes()
    buf = _dev(host)
    segs = [(3, k * 1024 + d) for k in (1, 2, 31, 32, 33) for d in (-1, 0, 1)]
    segs += [(o, k * 32768 + d) for o in (0, 5) for k in (1, 2, 3, 64) for d in (-1, 0, 1)]
    segs += [(int(rng.integers(0, 1 << 20)), int(rng.integers(1, 6 << 20))) for _ in range(12)]
    segs += [(0, len(host)), (1, len(host) - 1)]
    got = ops.crc32c_multi([buf[o:o + n] for o, n in segs])
    assert got == [T.crc32c(host[o:o + n]) for o, n in segs]


def test_crc32c_one_launch_over_more_than_4_gib():
    """65 aliases of one 64 MiB buffer plus shifted ones: more than 2^32 bytes in one launch, every result exact."""
    rng = np.random.default_rng(2)
    host = rng.integers(0, 256, 64 << 20, dtype=np.uint8)
    buf = torch.from_numpy(host).to(DEV)
    full = T.crc32c(host)
    views = [buf] * 65 + [buf[1:], buf[:-3], buf[4096:]]
    assert sum(v.numel() for v in views) > 2 ** 32
    got = ops.crc32c_multi(views)
    assert got[:65] == [full] * 65
    assert got[65:] == [T.crc32c(host[1:]), T.crc32c(host[:-3]), T.crc32c(host[4096:])]


# ---- training state ----------------------------------------------------------------------------------------------
def _config(model_cfg, tmp_path=None, task=None, **opt):
    from merlot_b200.config import NeatConfig
    d = {"data": {"num_chunks": 4, "chunk_text_len": 16}, "model": dict(model_cfg, image_size=[64, 96]),
         "optimizer": dict(OCFG, **opt), "device": {"output_dir": str(tmp_path or "/tmp/unused"), "train_batch_size": 2}}
    if task:
        d["downstream"] = {"task": task, "mode": "answer"}
    return NeatConfig.from_dict(d)


def _vcr_cfg(tiny_cfg):
    return dict(tiny_cfg, num_texts=4, num_chunks_in_group=1, hidden_dropout_prob=0.1)


def _batch(config, seed):
    """Features of the configured task at the tiny config (ids inside its vocabulary)."""
    m = config.model
    if config.downstream.get("task") == "vcr":
        from tests.test_gpu_vcr_train import batch
        image, ids, target = batch(m, 2, seed=seed)
        return {"images": image.bfloat16().to(DEV), "lm_input": ids.to(DEV), "lm_targets": target.to(DEV)}
    from tests.test_gpu_model import synth
    image, ids, shuf, vid = synth(m, 2, 4, 16, 64, 96, seed)
    return {"images": image.bfloat16().to(DEV), "input_ids": ids.to(DEV), "shuffled_idx_img": shuf.to(DEV),
            "video_src_ids": vid.to(DEV)}


def _trained(config, steps=2):
    from merlot_b200.train import _step_for
    builder, _ = _step_for(config)
    fn = builder(config, device=DEV)
    for s in range(steps):
        fn(_batch(config, s), None, "train", None).train_op()
    torch.cuda.synchronize()
    return fn


def _variable_mask(store):
    """True on the arena elements that belong to a reference variable (not PAD padding, not zero-padded columns)."""
    mask = torch.zeros(store.total, dtype=torch.bool, device=DEV)
    for e in store.entries.values():
        v = mask[e.offset:e.offset + e.numel].view(e.shape)
        if e.ref_cols:
            v[..., :e.ref_cols] = True
        else:
            v.fill_(True)
    return mask


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _assert_same_state(a, b, mask):
    assert torch.equal(_bits(a.p), _bits(b.p)) and torch.equal(_bits(a.pb), _bits(b.pb)) and torch.equal(_bits(a.m), _bits(b.m))
    # AdamW's 1e-30 floor leaves a residue in the second moment of padding elements, which belong to no variable: those
    # restore as zero, every variable's bits match
    assert torch.equal(_bits(a.v)[mask], _bits(b.v)[mask])
    assert a.global_step == b.global_step


def _close(x, y, exact):
    x, y = torch.as_tensor(x).float(), torch.as_tensor(y).float()
    return torch.equal(x, y) if exact else bool(torch.allclose(x, y, rtol=1e-2, atol=1e-5))


def _round_trip(config, tmp_path, exact_forward=True):
    """Train 2 steps, save, check the file against the arenas, restore into a fresh store and check the state, the next
    forward and the next AdamW update bit for bit.  exact_forward=False compares the forward at the model parity bar (1e-2)
    instead: the hybrid stem's GroupNorm statistics are summed with float atomics, so its forward is not bitwise repeatable
    (one loss was seen to differ by 2.6e-4 relative between a saved and a restored store whose state is bitwise equal).
    Returns (trained store, restored store, prefix)."""
    fn = _trained(config)
    st = fn.store
    prefix = str(tmp_path / "model.ckpt-2")
    timing = st.save_checkpoint(prefix)
    assert timing["bytes"] == os.path.getsize(prefix + ".data-00000-of-00001")
    got = T.load_checkpoint(prefix, skip_optimizer_slots=False)
    ref = st.to_tf_dict("p")
    for nm, t in ref.items():
        assert got[nm].dtype == torch.float32 and torch.equal(_bits(got[nm]), _bits(t)), nm
    for suffix, buf in (("adam_m", st.m), ("adam_v", st.v)):
        for _, nm, t in st.tf_views(buf):
            g = got[f"{nm}/{suffix}"]
            assert g.dtype == torch.bfloat16 and list(g.shape) == list(t.shape) and torch.equal(_bits(g), _bits(t.cpu().contiguous())), nm
    assert got["global_step"].dtype == torch.int64 and int(got["global_step"]) == 2
    assert set(got) == set(ref) | {f"{n}/adam_{s}" for n in ref for s in "mv"} | {"global_step"}

    fn2 = _trained(config, steps=0)
    st2 = fn2.store
    st2.p.normal_()  # everything must come from the checkpoint
    st2.m.fill_(1.0)
    st2.v.fill_(-1.0)
    st2.global_step = 123
    st2.restore_checkpoint(prefix)
    mask = _variable_mask(st)
    _assert_same_state(st, st2, mask)
    assert not torch.any(st2.p[~mask]) and not torch.any(st2.m[~mask]) and not torch.any(st2.v[~mask])
    # the next step's forward on the same batch: bitwise equal losses and metrics
    feats = _batch(config, 9)
    s1, s2 = fn(feats, None, "train", None), fn2(feats, None, "train", None)
    for x, y in zip(s1.loss_parts, s2.loss_parts):
        assert _close(x, y, exact_forward), (float(x), float(y))
    assert s1.metrics.keys() == s2.metrics.keys()
    for k in s1.metrics:
        assert _close(s1.metrics[k], s2.metrics[k], exact_forward), k
    del s1, s2
    # the same injected gradient through apply_gradients
    g = torch.randn(st.total, generator=torch.Generator().manual_seed(3)).to(DEV) * mask
    for f in (fn, fn2):
        f.store.g.copy_(g)
        f.optimizer.apply_gradients()
    torch.cuda.synchronize()
    _assert_same_state(st, st2, mask)
    assert st.global_step == 3
    return st, st2, prefix


def test_pretrain_state_round_trip(tmp_path, tiny_cfg):
    st, _, prefix = _round_trip(_config(tiny_cfg), tmp_path)
    # one flipped byte in a tensor: restore raises and names it
    entries = T._index(prefix, True)[1]
    victim = "encoder/layer01/intermediate/kernel/adam_v"
    with open(prefix + ".data-00000-of-00001", "r+b") as f:
        f.seek(int(entries[victim]["offset"]) + 5)
        b = f.read(1)
        f.seek(int(entries[victim]["offset"]) + 5)
        f.write(bytes([b[0] ^ 0x01]))
    with pytest.raises(T.CheckpointFormatError, match=victim):
        st.restore_checkpoint(prefix)


def test_vcr_state_round_trip_and_mismatches(tmp_path, tiny_cfg):
    from merlot_b200.params import ParamStore
    cfg = _vcr_cfg(tiny_cfg)
    st, st2, prefix = _round_trip(_config(cfg, task="vcr"), tmp_path)
    for tower in ("answer_cls", "rationale_cls"):
        e = st2.entries[f"{tower}/classifier_mlp1/kernel"]
        for buf in (st2.p, st2.m):  # still zero after the restored store's AdamW step (v holds the 1e-30 floor there)
            assert not torch.any(st2._view(buf, e.name)[:, e.ref_cols:])
    # a VCR store cannot resume from a pretraining checkpoint: the towers' variables are missing
    pre = _trained(_config(tiny_cfg), steps=1)
    pprefix = str(tmp_path / "pretrain.ckpt-1")
    pre.store.save_checkpoint(pprefix)
    with pytest.raises(T.CheckpointFormatError, match="answer_cls"):
        st2.restore_checkpoint(pprefix)
    # and a pretraining store needs variables a VCR checkpoint lacks (the language-only embeddings, the pretraining heads)
    with pytest.raises(T.CheckpointFormatError, match="not in the checkpoint"):
        pre.store.restore_checkpoint(prefix)
    # shape mismatch: same names, other hidden size
    other = ParamStore(dict(cfg, hidden_size=64, intermediate_size=128, contrastive_size=64), device=DEV, optimizer_cfg=OCFG,
                       task="vcr")
    with pytest.raises(T.CheckpointFormatError, match="shape"):
        other.restore_checkpoint(prefix)


def test_hybrid_stem_state_round_trip(tmp_path, tiny_cfg):
    st, _, prefix = _round_trip(_config(dict(tiny_cfg, resnet_layers=[1, 2, 1])), tmp_path, exact_forward=False)
    names = dict(T.list_variables(prefix))
    assert names["vision_backbone/vision_transformer/resnet50lite/stem/conv2d/kernel"] == [3, 3, 3, 32]
    assert names["vision_backbone/vision_transformer/resnet50lite/stem/conv2d/kernel/adam_v"] == [3, 3, 3, 32]


def test_slot_rule(tmp_path, tiny_cfg):
    """Slots exist for exactly the variables AdamW updates: not the viz_viz temporal head (no gradient without image
    shuffling) and not a learning-rate-0 group; every variable whose first moment moved has its slots."""
    from merlot_b200.train import variables_without_gradient
    cfg = dict(tiny_cfg, image_shuffle_prob=0.0)
    over = OCFG["param_overrides"] + [[["^lm_head"], {"learning_rate": 0}]]
    config = _config(cfg, param_overrides=over)
    fn = _trained(config)
    st = fn.store
    skip = variables_without_gradient(config.model, st)
    assert skip and all(n.startswith("viz_viz_temporal/") for n in skip)
    slotted = {e.name for e in st.slot_entries(skip)}
    frozen = {n for n, e in st.entries.items() if e.hyper[0] == 0}
    assert frozen and all(n.startswith("lm_head/") for n in frozen)
    assert slotted == set(st.entries) - set(skip) - frozen
    moved = {n for n, e in st.entries.items() if torch.any(st.m[e.offset:e.offset + e.padded])}
    assert moved <= slotted and len(moved) > 0.9 * len(slotted)
    prefix = str(tmp_path / "model.ckpt-2")
    st.save_checkpoint(prefix, skip=skip)
    names = {n for n, _ in T.list_variables(prefix)}
    for n, e in st.entries.items():
        for tf in e.tf_names:
            assert (f"{tf}/adam_m" in names) == (n in slotted) and (f"{tf}/adam_v" in names) == (n in slotted), n
    fresh = _trained(config, steps=0)
    fresh.store.restore_checkpoint(prefix, skip=skip)
    _assert_same_state(st, fresh.store, _variable_mask(st))
    with pytest.raises(T.CheckpointFormatError, match="viz_viz_temporal"):  # a store that wants slots the file lacks
        fresh.store.restore_checkpoint(prefix)


# ---- the trainer -------------------------------------------------------------------------------------------------
def _yaml(tmp_path, tiny_cfg, steps, out):
    cfg = {"data": {"num_chunks": 4, "chunk_text_len": 16}, "model": dict(tiny_cfg, image_size=[64, 96], vocab_size=50370),
           "optimizer": dict(OCFG, num_train_steps=steps),
           "device": {"output_dir": str(out), "train_batch_size": 2, "iterations_per_loop": 2}}
    path = tmp_path / f"run{steps}.yaml"
    path.write_text(yaml.safe_dump(cfg))
    return str(path)


def test_trainer_saves_and_resumes(tmp_path, tiny_cfg, capsys):
    from merlot_b200.train import main
    out = tmp_path / "out"
    main([_yaml(tmp_path, tiny_cfg, 5, out)])
    files = sorted(os.listdir(out))
    assert [f for f in files if f.endswith(".index")] == ["model.ckpt-2.index", "model.ckpt-4.index", "model.ckpt-5.index"]
    assert T.latest_checkpoint(str(out)) == str(out / "model.ckpt-5")
    assert (out / "checkpoint").read_text().startswith('model_checkpoint_path: "model.ckpt-5"\n')
    first = (out / "model.ckpt-4.index").stat().st_mtime_ns
    capsys.readouterr()
    main([_yaml(tmp_path, tiny_cfg, 7, out)])
    log = capsys.readouterr().out
    assert "continuing from global_step 5" in log and "step 0 loss" not in log, log
    assert T.latest_checkpoint(str(out)) == str(out / "model.ckpt-7")
    assert int(T.load_checkpoint(str(out / "model.ckpt-7"), names=["global_step"])["global_step"]) == 7
    assert os.path.exists(out / "model.ckpt-6.index") and (out / "model.ckpt-4.index").stat().st_mtime_ns == first
    with pytest.raises(ValueError, match="local"):
        main([_yaml(tmp_path, tiny_cfg, 3, "gs://bucket/run")])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dist_worker(rank, world, port, yaml3, yaml4, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                          LOCAL_RANK=str(rank))
        torch.cuda.set_device(rank)
        from merlot_b200 import params as P
        from merlot_b200 import train
        saves, real = [], P.ParamStore.save_checkpoint

        def counting(self, prefix, skip=()):
            saves.append(os.path.basename(prefix))
            return real(self, prefix, skip)
        P.ParamStore.save_checkpoint = counting
        train.main([yaml3])
        restored = []
        real_restore = P.ParamStore.restore_checkpoint

        def keep(self, prefix, skip=()):
            real_restore(self, prefix, skip)
            restored.append(self)
        P.ParamStore.restore_checkpoint = keep
        train.main([yaml4])
        st = restored[0]
        import torch.distributed as dist
        state = torch.cat([st.p.view(torch.int32), st.m.view(torch.int32), st.v.view(torch.int32)])
        allst = [torch.empty_like(state) for _ in range(world)]
        dist.all_gather(allst, state)
        q.put({"rank": rank, "saves": saves, "identical": all(torch.equal(allst[0], x) for x in allst[1:]),
               "step": st.global_step})
        dist.barrier()
    except Exception:
        import traceback
        q.put({"rank": rank, "error": traceback.format_exc()})
        raise


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_save_and_resume(tmp_path, tiny_cfg):
    import torch.multiprocessing as mp
    out = tmp_path / "out"
    y3, y4 = _yaml(tmp_path, tiny_cfg, 3, out), _yaml(tmp_path, tiny_cfg, 4, out)
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_dist_worker, args=(r, world, port, y3, y4, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in ps:
        p.join(timeout=120)
    for r in res:
        assert "error" not in r, r.get("error")
    res = {r["rank"]: r for r in res}
    assert res[0]["saves"] == ["model.ckpt-2", "model.ckpt-3", "model.ckpt-4"] and res[1]["saves"] == []
    assert all(res[r]["identical"] and res[r]["step"] == 4 for r in range(world))
    assert T.latest_checkpoint(str(out)) == str(out / "model.ckpt-4")
