"""GPU tests of zero-shot story unshuffling (pytest -m gpu): K14 with the evaluation plan against tests/input_oracle.py,
story records -> batch against the oracle input, the one-ViT-pass forward (frame_copies) against the tiled forward, both
modality pairs' probabilities against the oracle model, independence from the other stories of a batch, the driver end to
end, and one batch at merlot_5segments.yaml sizes."""
import io
import os
import threading

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import ops
from merlot_b200 import sort_story as S
from merlot_b200.config import NeatConfig
from oracle import merlot_oracle as MO
from tests import input_oracle as O
from tests import story_records as R

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _check_bilinear(got, ref, what):
    # the bar of tests/test_gpu_input.py: K14 and the oracle round every float32 operation in the same order, bit-exact
    bad = got != ref
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ, first at {np.argwhere(bad)[0].tolist()}"


def _oracle_frame(u8, out):
    sh, sw, oy, ox = R.eval_plan(u8.shape[0], u8.shape[1], out)
    return O.bf16_round(O.resize_and_pad(u8.astype(np.float32) * O.INV255, out, sh, sw, oy, ox, 0))


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _cfg(tiny_cfg, **over):
    c = dict(tiny_cfg, num_chunks_in_group=5, image_size=[64, 64], max_position_embeddings=256, hidden_dropout_prob=0.1)
    c.update(over)
    return c


def _store(cfg, seed=1):
    from merlot_b200.params import ParamStore
    params = MO.init_params(cfg, seed=seed, perturb=0.05)
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    store = ParamStore(cfg, device=DEV, with_optimizer_state=False)
    store.load_tf_dict(params)
    return params, store


def _stories(cfg, b, seed):
    g = torch.Generator().manual_seed(seed)
    Hh, Ww = cfg["image_size"]
    images = torch.rand(b * 5, Hh, Ww, 3, generator=g).to(torch.bfloat16)
    sents = torch.randint(100, cfg["vocab_size"], (b, 5, 32), generator=g, dtype=torch.int32)
    sents[:, :, 0] = 2
    lens = torch.randint(4, 33, (b, 5), generator=g)
    sents = sents * (torch.arange(32)[None, None] < lens[..., None]).int()
    return images.to(DEV), sents.to(DEV)


def _tiled(images, dup):
    """The reference's frames, one copy per duplicate, in the story-major layout: [story 0 copy 0 | story 0 copy 1 | ...]."""
    n = images.shape[0] // 5
    return images.view(n, 5, *images.shape[1:]).repeat_interleave(dup, 0).reshape(n * dup * 5, *images.shape[1:]).contiguous()


def _forward(cfg, store, images, ids, shuf, copies, dup=2):
    """(viz hidden, lang hidden, lang_viz probs, viz_viz probs) of one eval forward of `dup` story-major copies of every story,
    copied out of the store's buffers (the next forward reuses them)."""
    from merlot_b200.modeling import MerlotModel
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=images, input_ids=ids, mask_input=False, shuffled_idx_img=shuf,
                    params=store, log_attention_probs=False, frame_copies=copies)
    out = (m.encoder_hidden_states["viz"].clone(), m.encoder_hidden_states["lang"].clone(),
           S.temporal_probs(m, dup, "lang_viz_temporal").clone(), S.temporal_probs(m, dup, "viz_viz_temporal").clone())
    torch.cuda.synchronize()
    return out


# ---- K14 with the evaluation plan ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("out", [(40, 56), (64, 64)])
def test_frames_prepare_eval_plan_matches_oracle(out):
    rng = np.random.default_rng(8)
    srcs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in R.SIZES + [(out[0], out[1]), (1, 3)]][:10]
    srcs = srcs + [rng.integers(0, 256, (out[0] // 2, out[1], 3), dtype=np.uint8)] * (15 - len(srcs))  # 2:1 frames
    staging, offsets, hw = S.stage_frames(srcs)
    plan = S.eval_frame_plan(hw, [0, 1, 2], out)
    plan["src_offset"] = offsets
    got = ops.frames_prepare(staging.cuda(), plan, *out).float().cpu().numpy()
    for i, u8 in enumerate(srcs):
        ref = _oracle_frame(u8, out)
        _check_bilinear(got[i], ref, f"{u8.shape[:2]} -> {out}")
        sh, sw = int(plan["scaled_h"][i]), int(plan["scaled_w"][i])
        assert (got[i][sh:] == 0).all() and (got[i][:, sw:] == 0).all()  # zero padding, bottom and right


def _write_config(tmp_path, cfg, val_batch_size, **data):
    d = {"data": dict({"val_file": str(tmp_path / "val-*.tfrecord"), "num_threads": 4}, **data), "model": cfg,
         "optimizer": {"learning_rate": 1e-4}, "device": {"output_dir": str(tmp_path / "out"), "val_batch_size": val_batch_size}}
    path = tmp_path / "sortstory.yaml"
    path.write_text(yaml.safe_dump(d))
    return path, NeatConfig.from_dict(d)


def test_story_pipeline_batch_matches_oracle(tmp_path, tiny_cfg):
    from PIL import Image
    cfg = _cfg(tiny_cfg, image_size=[48, 64])
    stories = R.write_stories(tmp_path, [3, 4], seed=5, max_sentence=50)
    _, config = _write_config(tmp_path, cfg, 3)
    by_id = {s["story_id"]: s for s in stories}
    seen = []
    with S.input_fn_builder(config) as pipe:
        for batch in pipe:
            torch.cuda.synchronize()
            assert batch["images"].shape == (15, 48, 64, 3) and batch["images"].dtype == torch.bfloat16
            assert batch["sentences"].shape == (3, 5, 32) and batch["sentences"].dtype == torch.int32
            imgs = batch["images"].float().cpu().numpy().reshape(3, 5, 48, 64, 3)
            for k, sid in enumerate(batch["story_id"]):
                s = by_id[int(sid)]
                assert batch["permutation_identity_encode"][k] == s["permutation_identity_encode"]
                np.testing.assert_array_equal(batch["sentences"][k].cpu().numpy(), R.sentences_np(s["sentences"]))
                for i, jpg in enumerate(s["frames"]):
                    u8 = np.asarray(Image.open(io.BytesIO(jpg)).convert("RGB"))
                    _check_bilinear(imgs[k, i], _oracle_frame(u8, (48, 64)), f"story {sid} image {i}")
            seen += [int(x) for x in batch["story_id"]]
        assert pipe.dropped == 1
    assert seen == [0, 3, 1, 4, 2, 5]  # two files interleaved one record at a time, the seventh story dropped
    assert not [t.name for t in threading.enumerate() if t.name.startswith("merlot-")]


def test_broken_image_raises_from_pipeline(tmp_path, tiny_cfg):
    rng = np.random.default_rng(0)
    s = R.story(rng, 77)
    s["frames"][4] = b"\xff\xd8 broken"
    from tests import tfrecord_writer as W
    W.write_records(tmp_path / "val-000.tfrecord", [R.story_example(s)])
    _, config = _write_config(tmp_path, _cfg(tiny_cfg), 1)
    with S.input_fn_builder(config) as pipe:
        with pytest.raises(ValueError, match="story 77: image 4 cannot be decoded"):
            next(pipe)


# ---- one ViT pass per story -------------------------------------------------------------------------------------------
def test_frame_copies_bitwise_equals_tiled_forward(tiny_cfg):
    cfg = _cfg(tiny_cfg)
    _, store = _store(cfg)
    images, sents = _stories(cfg, 3, seed=2)
    ids, shuf = S.tiled_inputs(sents, 2, seed=5)
    one = _forward(cfg, store, images, ids, shuf, copies=2)
    tiled = _forward(cfg, store, _tiled(images, 2), ids, shuf, copies=1)
    # every forward kernel computes each output in an order that does not depend on the batch: bitwise equal
    for name, a, b in zip(("viz", "lang", "lang_viz_probs", "viz_viz_probs"), one, tiled):
        assert torch.equal(a, b), (name, float((a - b).abs().max()))


def test_frame_copies_hybrid_stem_matches_tiled_forward(tiny_cfg):
    cfg = _cfg(tiny_cfg, resnet_layers=[1, 1, 1])
    _, store = _store(cfg)
    images, sents = _stories(cfg, 2, seed=3)
    ids, shuf = S.tiled_inputs(sents, 2, seed=6)
    one = _forward(cfg, store, images, ids, shuf, copies=2)
    tiled = _forward(cfg, store, _tiled(images, 2), ids, shuf, copies=1)
    # Not bitwise: the stem's GroupNorm statistics (gn_stats_kernel, csrc/stem.cu) are float atomicAdds whose order depends
    # on block scheduling (and on the batch size through the grid), so the stem is not bit-reproducible even between two runs
    # of the same batch; a flipped bf16 rounding carried through the ViT and the joint encoder measured 6.3e-3 on the viz
    # states.  The bar is the project's bar for bf16 hidden states, 1.5e-2; the patch-embed test above is the exact check.
    for name, a, b in zip(("viz", "lang", "lang_viz_probs", "viz_viz_probs"), one, tiled):
        assert rel(a, b) < 1.5e-2, (name, rel(a, b))


def test_zero_shot_probs_match_oracle(tiny_cfg):
    cfg = _cfg(tiny_cfg)
    params, store = _store(cfg)
    images, sents = _stories(cfg, 2, seed=4)
    config = NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {}, "device": {"output_dir": "/nonexistent"}})
    batch = {"images": images, "sentences": sents, "story_id": np.array([5, 9]), "permutation_identity_encode": np.array([1, 2])}
    got = S.zero_shot_predict(config, store, batch, duplication_factor=2, seed=7)
    assert got["lang_viz_probs"].shape == (2, 5, 5, 3) and got["viz_viz_probs"].shape == (2, 5, 5, 3)
    assert got["sentences"] is sents and list(got["story_id"]) == [5, 9]
    ids, shuf = S.tiled_inputs(sents, 2, seed=7)
    om = MO.MerlotOracle(cfg, params, _tiled(images, 2).float().cpu(), ids.cpu().long(), mask_input=False,
                         shuffled_idx_img=shuf.cpu().long())
    H = cfg["hidden_size"]
    hl = om.encoder_hidden_states["lang"].reshape(om.B, 5, om.lang_chunk_length, H)[:, :, 0]
    hv = om.encoder_hidden_states["viz"].reshape(om.B, 5, om.viz_chunk_length, H)[:, :, 0]
    for name, xa, xb in (("lang_viz", hl, hv), ("viz_viz", hv, hv)):
        ref = torch.softmax(om.allpairs_temporal_logits(xa, xb, f"{name}_temporal"), -1)[:, 1:].reshape(2, 2, 5, 5, 3).mean(1)
        assert rel(got[f"{name}_probs"], ref) < 1e-2, (name, rel(got[f"{name}_probs"], ref))


def test_story_probs_do_not_depend_on_batch_mates(tiny_cfg):
    cfg = _cfg(tiny_cfg)
    _, store = _store(cfg)
    images, sents = _stories(cfg, 4, seed=6)
    ids, shuf = S.tiled_inputs(sents, 2, seed=8)
    base = _forward(cfg, store, images, ids, shuf, copies=2)
    perm = torch.tensor([2, 0, 3, 1])
    rows = (perm[:, None] * 2 + torch.arange(2)[None]).reshape(-1)  # a story's two copies move with it, with their orders
    img_p = images.view(4, 5, *images.shape[1:])[perm.to(DEV)].reshape(images.shape)
    moved = _forward(cfg, store, img_p, ids[rows.to(DEV)], shuf.view(8, 5)[rows.to(DEV)].reshape(-1), copies=2)
    for name, a, b in zip(("lang_viz_probs", "viz_viz_probs"), base[2:], moved[2:]):
        assert torch.equal(a[perm.to(DEV)], b), name
    alone = _forward(cfg, store, images[5:10], ids[2:4], shuf[10:20], copies=2)  # story 1 in a batch of its own
    assert torch.equal(alone[2][0], base[2][1]) and torch.equal(alone[3][0], base[3][1])


# ---- the driver ---------------------------------------------------------------------------------------------------------
def _save_checkpoint(cfg, out_dir, drop=None):
    from merlot_b200.params import ParamStore
    from merlot_b200.tf_checkpoint import DT_FLOAT, update_checkpoint_state, write_bundle
    os.makedirs(out_dir, exist_ok=True)
    store = ParamStore(cfg, device=DEV)
    store.init_reference(seed=3)
    store.global_step = 11
    prefix = os.path.join(out_dir, "model.ckpt-11")
    if drop is None:
        store.save_checkpoint(prefix)
    else:
        write_bundle(prefix, [(nm, DT_FLOAT, tuple(t.shape), t.numpy().tobytes(), None)
                              for nm, t in store.to_tf_dict().items() if nm != drop])
    update_checkpoint_state(out_dir, prefix)
    return prefix


def test_driver_end_to_end(tmp_path, tiny_cfg, capsys, monkeypatch):
    cfg = _cfg(tiny_cfg)
    R.write_stories(tmp_path, [4, 3], seed=9)
    path, config = _write_config(tmp_path, cfg, 2)
    prefix = _save_checkpoint(cfg, str(tmp_path / "out"))
    monkeypatch.delenv("SORTSTORY_PATH", raising=False)
    out = str(tmp_path / "logits_val.npz")
    res = S.main([str(path), "--out", out])
    printed = capsys.readouterr().out
    groups = S.read_logits_npz(out)
    assert len(groups) == 6 and "scored 6 stories, dropped 1" in printed
    for g in groups.values():
        assert sorted(g) == ["lang_viz_probs", "permutation_identity_encode", "sentences", "viz_viz_probs"]
        assert g["lang_viz_probs"].shape == (5, 5, 3) and g["viz_viz_probs"].shape == (5, 5, 3)
        assert g["sentences"].shape == (5, 32) and g["permutation_identity_encode"].shape == ()
    store = S.restore_for_zero_shot(config, prefix)
    with S.input_fn_builder(config) as pipe:
        for batch in pipe:
            pred = S.zero_shot_predict(config, store, batch)
            for row in S._story_rows(pred):
                g = groups[str(row["story_id"])]
                for k in ("lang_viz_probs", "viz_viz_probs", "sentences", "permutation_identity_encode"):
                    np.testing.assert_array_equal(g[k], row[k], err_msg=k)
    ref = S.score_file(out)
    assert res == ref
    tail = printed.split("Spearman:")[1].split()
    assert [float(tail[0]), float(tail[3]), float(tail[5])] == [ref["spearman"], ref["absolute_distance"], ref["pairwise"]]
    # SORTSTORY_PATH takes precedence over data.val_file; a pattern matching nothing raises
    monkeypatch.setenv("SORTSTORY_PATH", str(tmp_path / "nothing-*.tfrecord"))
    with pytest.raises(ValueError, match="matches no file"):
        S.main([str(path), "--out", out])


def test_driver_writes_h5(tmp_path, tiny_cfg, monkeypatch):
    pytest.importorskip("h5py", reason="h5py is not installed here: the HDF5 writer cannot be exercised")
    cfg = _cfg(tiny_cfg)
    R.write_stories(tmp_path, [2], seed=1)
    path, _ = _write_config(tmp_path, cfg, 2)
    _save_checkpoint(cfg, str(tmp_path / "out"))
    monkeypatch.delenv("SORTSTORY_PATH", raising=False)
    res = S.main([str(path), "--out", str(tmp_path / "logits_val.h5")])
    assert res == S.score_file(str(tmp_path / "logits_val.h5"))


def test_checkpoint_missing_temporal_head_raises(tmp_path, tiny_cfg, monkeypatch):
    cfg = _cfg(tiny_cfg)
    R.write_stories(tmp_path, [2], seed=1)
    path, _ = _write_config(tmp_path, cfg, 2)
    _save_checkpoint(cfg, str(tmp_path / "out"), drop="lang_viz_temporal/logits/kernel")
    monkeypatch.delenv("SORTSTORY_PATH", raising=False)
    with pytest.raises(ValueError, match="lang_viz_temporal/logits/kernel"):
        S.main([str(path), "--out", str(tmp_path / "x.npz")])


# ---- merlot_5segments.yaml sizes ------------------------------------------------------------------------------------
def test_one_batch_at_five_segments_sizes():
    from merlot_b200.params import ParamStore
    cfg = R.five_segments_model()
    store = ParamStore(cfg, device=DEV, with_optimizer_state=False)
    store.init_reference(seed=0)
    config = NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {}, "device": {"output_dir": "/nonexistent"}})
    images, sents = _stories(cfg, 16, seed=1)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = S.zero_shot_predict(config, store, {"images": images, "sentences": sents, "story_id": np.arange(16),
                                              "permutation_identity_encode": np.zeros(16, np.int64)}, duplication_factor=2)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print(f"merlot_5segments sizes, 16 stories x 2 copies, 384x384, hybrid stem: peak {peak / 2**30:.2f} GiB allocated "
          f"({(peak - base) / 2**30:.2f} GiB above the weights and inputs)")
    for k in ("lang_viz_probs", "viz_viz_probs"):
        p = got[k]
        assert p.shape == (16, 5, 5, 3) and torch.isfinite(p).all()
        assert (p > 0).all() and (p.sum(-1) < 1).all()  # three of the four classes of a softmax
