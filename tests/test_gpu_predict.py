"""GPU tests of model_fn's PREDICT mode (pytest -m gpu): the accumulating attention-probability export against the mean of
the per-layer exports and a float64 restatement, the per-layer export against its recorded bits, MerlotModel's layer-mean
export against the oracle, the "predict" mode against the "eval" mode, and `python -m merlot_b200.predict` on one and on
two ranks against pretrain_validate.

Bitwise comparisons run with masking_use_attn: False (see tests/test_gpu_pretrain_validate.py: mask_inputs ranks tokens by
attention sums that K4 adds up with float atomics)."""
import json
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import ops
from merlot_b200.config import NeatConfig
from tests import export_cases as X

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
LAYERS = 3


def _u8(valid):
    return None if valid is None else valid.to(torch.uint8).reshape(-1).contiguous().to(DEV)


def _layers(B, S, heads, i, ragged, pair):
    """LAYERS seeded layers of one shape with one validity mask: [(qkv, lse)], valid."""
    out, valid = [], None
    for l in range(LAYERS):
        qkv, lse, v = X.case(B, S, heads, seed=1000 * i + l, ragged=ragged, pair=pair)
        valid = v if l == 0 else valid
        if valid is not None:  # every layer of a stack sees the same mask: recompute lse under layer 0's
            lse = torch.logsumexp(X.scores(qkv, B, S, heads, valid, pair), -1).float()
        out.append((qkv, lse))
    return out, valid


def _max_rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float(((a - b).abs() / b.abs().clamp_min(1e-30)).max())


def _rel_fro(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


# ---- kernel ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("i", range(len(X.SHAPES)))
def test_layer_mean_export(i, p):
    """out = beta*out + alpha*mean_h P with alpha = 1/layers, beta 0 then 1: the mean of the per-layer exports to fp32
    summation order, and the float64 head-and-layer mean, with and without attention dropout.  The exports never read a
    beta = 0 output (it starts as NaN)."""
    B, S, heads, ragged, pair = X.SHAPES[i]
    layers, valid = _layers(B, S, heads, i, ragged, pair)
    vd = _u8(valid)
    mean = torch.full((B, S, S), float("nan"), device=DEV)
    per, ref64 = [], torch.zeros(B, S, S, dtype=torch.float64)
    for l, (qkv, lse) in enumerate(layers):
        drop = (p, X.SEED, X.SITE + l)
        qd, ld = qkv.to(DEV), lse.to(DEV)
        per.append(ops.attention_probs(qd, ld, B, S, heads, vd, out=torch.full((B, S, S), float("nan"), device=DEV),
                                       pair=pair, dropout=drop))
        ops.attention_probs(qd, ld, B, S, heads, vd, out=mean, pair=pair, dropout=drop, alpha=1.0 / LAYERS,
                            beta=0.0 if l == 0 else 1.0)
        ref64 += X.head_mean(qkv, lse, B, S, heads, valid, pair, drop) / LAYERS
    torch.cuda.synchronize()
    assert torch.isfinite(mean).all()
    acc = per[0] * (1.0 / LAYERS)  # the accumulation order of the stack, in fp32
    for t in per[1:]:
        acc = acc + t * (1.0 / LAYERS)
    e_sum, e_64 = _max_rel(mean, acc), _rel_fro(mean, ref64)
    print(f"\n{X.SHAPES[i]} p={p}: layer mean vs fp32 mean of per-layer exports max rel {e_sum:.2e}, "
          f"vs float64 rel-Frobenius {e_64:.2e}")
    assert e_sum < 1e-5
    assert e_64 < 1e-4


def test_per_layer_export_is_bit_identical_to_the_recorded_one():
    """alpha = 1, beta = 0 (the per-layer export, `ops.attention_probs` defaults) reproduces, bit for bit, the exports the
    kernel produced before it took alpha and beta, recorded as SHA-256 digests on the same seeded inputs."""
    with open(os.path.join(HERE, "golden", "export_parent_digests.json")) as f:
        golden = json.load(f)
    assert len(golden) == 2 * len(X.SHAPES)
    for i, (B, S, heads, ragged, pair) in enumerate(X.SHAPES):
        qkv, lse, valid = X.case(B, S, heads, seed=100 + i, ragged=ragged, pair=pair)
        for p in (0.0, 0.1):
            out = torch.full((B, S, S), float("nan"), device=DEV)
            ops.attention_probs(qkv.to(DEV), lse.to(DEV), B, S, heads, _u8(valid), out=out, pair=pair,
                                dropout=(p, X.SEED, X.SITE))
            key = f"{B}x{S}x{heads}/ragged={int(ragged)}/pair={pair[0]},{pair[1]}/p={p}"
            assert X.digest(out) == golden[key], key


def test_attention_log_of_a_layer_mean_map():
    """merlot_attention_log_probs: the reference's block sums (model/modeling.py:190-203) of a map against float64, and the
    same bits on a second call."""
    B, S, P = 3, 300, 77
    g = torch.Generator().manual_seed(5)
    probs = torch.rand(B, S, S, generator=g)
    valid = torch.rand(B, S, generator=g) > 0.2
    got = ops.attention_log_probs(probs.to(DEV), _u8(valid), P)
    again = ops.attention_log_probs(probs.to(DEV), _u8(valid), P)
    m = probs.double() * valid[:, None].double() * valid[:, :, None].double()
    m = m.mean(0)
    m = m / m.sum()
    ref = [m[P:, P:].sum(), m[:P, P:].sum(), m[P:, :P].sum(), m[:P, :P].sum()]  # lang2lang, lang2viz, viz2lang, viz2viz
    assert torch.equal(got, again)
    for a, b in zip(got.cpu().tolist(), ref):
        assert a == pytest.approx(float(b), rel=1e-5)


# ---- MerlotModel ------------------------------------------------------------------------------------------------------
def test_model_layer_mean_export(tiny_cfg):
    """export_attention_probs="layer_mean": encoder_info holds the [B, S, S] layer mean of the joint maps (against the oracle
    and against the per-layer export's mean), the language-only maps stay per layer, attention_log matches the oracle, and
    no [layers, B, S, S] buffer of the joint encoder exists."""
    from oracle import merlot_oracle as O
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import ParamStore
    from tests.test_gpu_model import build, rel, synth
    cfg = tiny_cfg
    image, ids, shuf, _ = synth(cfg, 2, 4, 16, 64, 96, 0)
    params, store, _ = build(cfg)
    draws = O.make_mask_draws(4, 32, 6, cfg["vocab_size"], seed=5)
    kw = dict(is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
              shuffled_idx_img=shuf.to(DEV), mask_draws=draws)
    m = MerlotModel(cfg, params=store, export_attention_probs="layer_mean", **kw)
    B, Sj, layers = m.B, m._dims["Sj"], cfg["num_hidden_layers"]
    pj, pl = m.encoder_info["self_attn_probs"], m.lang_transformer_info["self_attn_probs"]
    assert tuple(pj.shape) == (B, Sj, Sj)
    shapes = [tuple(t.shape) for t in store._bufs.values() if torch.is_tensor(t)]
    assert (layers, B, Sj, Sj) not in shapes and not any(s[-2:] == (Sj, Sj) and len(s) == 4 for s in shapes)
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(4, 32), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    om = O.MerlotOracle(cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm)
    assert tuple(pl.shape) == tuple(om.lang_transformer_info["self_attn_probs"].shape)
    assert rel(pl, om.lang_transformer_info["self_attn_probs"]) < 5e-3
    e = rel(pj, om.encoder_info["self_attn_probs"].mean(1))
    print(f"\nlayer-mean joint map vs oracle: rel-Frobenius {e:.2e}")
    assert e < 1e-2
    assert float((pj.sum(-1) - 1).abs().max()) < 2e-3
    for k, v in om.attention_log.items():  # the bar of tests/test_gpu_model.py
        assert abs(float(m.attention_log[k]) - float(v)) < 2e-3, k
    pj = pj.clone()
    # the per-layer export of a second store with the same weights: its layer mean to fp32 summation order
    store2 = ParamStore(cfg, device=DEV, optimizer_cfg=build(cfg)[2])
    store2.load_tf_dict(params)
    m2 = MerlotModel(cfg, params=store2, export_attention_probs=True, **kw)
    per = m2.encoder_info["self_attn_probs"]  # [B, layers, S, S]
    acc = per[:, 0] * (1.0 / layers)
    for l in range(1, layers):
        acc = acc + per[:, l] * (1.0 / layers)
    assert torch.equal(m2.lang_mask_info["masked_ids"].cpu().reshape(4, 32), gm["masked_ids"])
    assert _max_rel(pj, acc) < 1e-5
    with pytest.raises(ValueError):
        MerlotModel(cfg, params=store, export_attention_probs="mean", **kw)


# ---- model_fn PREDICT ---------------------------------------------------------------------------------------------------
def _tiny(tiny_cfg, **over):
    return dict(tiny_cfg, image_size=[64, 96], masking_use_attn=False, **over)


def _restated_shapes(raw_shapes, bsz):
    """modeling.py:774-784 restated in NumPy on arrays of the given shapes: the shapes each entry ends with."""
    out = {}
    for k in sorted(raw_shapes):
        a = np.zeros(raw_shapes[k], dtype=np.float32)
        if a.ndim == 0:
            a = np.tile(a[None], [bsz])
        elif a.shape[0] != bsz:
            a = np.reshape(a, [bsz, -1])
        out[k] = a.shape
    return out


def test_predict_equals_eval(tmp_path, tiny_cfg):
    """For the same store, seed and batch, "predict" has eval's losses (lang/ contr/ temporal/ to the bit; attn/ from the
    exported map within 1e-4 of K4's column sums), eval's masked_ids, and the shapes of the reference's PREDICT dict."""
    from merlot_b200.train import model_fn_builder
    from tests.test_gpu_model import synth
    from tests.test_gpu_pretrain_validate import _config_dict
    model = _tiny(tiny_cfg, vit_hidden_dropout_prob=0.2, attention_probs_dropout_prob=0.1)
    config = NeatConfig.from_dict(_config_dict(tmp_path, model))
    bsz, n, Lc = 2, 4, 16
    image, ids, shuf, vid = synth(model, bsz, n, Lc, 64, 96, 3)
    feats = {"images": image.to(DEV).bfloat16(), "input_ids": ids.to(DEV), "shuffled_idx_img": shuf.to(DEV),
             "video_src_ids": vid.to(DEV), "is_eoc": torch.zeros(bsz, n, dtype=torch.bool, device=DEV),
             "mean_time": torch.rand(bsz, n, device=DEV)}
    fn = model_fn_builder(config, seed=7)
    k = 5
    ev = fn(feats, None, "eval", {"eval_batch": k})
    ev_metrics = {name: float(v) for name, v in ev.metrics.items()}
    ev_masked = ev.model.lang_mask_info["masked_ids"].cpu().clone()
    B, Sj = ev.model.B, ev.model._dims["Sj"]
    out = fn(feats, None, "predict", {"eval_batch": k, "batch_size": bsz})
    assert set(ev_metrics) <= set(out) and "images" not in out
    for name, v in ev_metrics.items():
        assert out[name].shape == (bsz,) and out[name].dtype == np.float32 and (out[name] == out[name][0]).all()
        if name.startswith("attn/"):
            assert float(out[name][0]) == pytest.approx(v, rel=1e-4, abs=1e-6), name
        else:
            assert float(out[name][0]) == v, (name, float(out[name][0]), v)
    np.testing.assert_array_equal(out["masked_ids"].reshape(-1), ev_masked.numpy().reshape(-1))
    layers, Llo = model["num_lang_transformer_hidden_layers"], Lc * n
    raw = {"self_attn_probs": (bsz, B // bsz, Sj, Sj), "lang_attn_probs": (bsz, layers, Llo, Llo),
           "masked_ids": tuple(ev.model.lang_mask_info["masked_ids"].shape), "input_ids": tuple(ids.shape),
           "shuffled_idx_img": tuple(shuf.shape), "video_src_ids": tuple(vid.shape), "is_eoc": (bsz, n), "mean_time": (bsz, n)}
    raw.update({name: () for name in ev_metrics})
    assert {name: a.shape for name, a in out.items()} == _restated_shapes(raw, bsz)
    for name, a in out.items():
        assert a.dtype in (np.float32, np.int32), (name, a.dtype)
    np.testing.assert_array_equal(out["input_ids"], ids.numpy())
    assert out["is_eoc"].dtype == np.int32


# ---- the program ---------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, argv, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    try:
        from merlot_b200 import predict
        q.put({"rank": rank, "out": predict.main(argv)})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


def test_predict_program_one_and_two_ranks(tmp_path, tiny_cfg):
    """python -m merlot_b200.predict on synthetic records and a checkpoint written by ParamStore.save_checkpoint: one batch
    file per global batch, the same bytes on two ranks as on one, batch k's losses those pretrain_validate computes for
    batch k, and read_predictions yields the videos in global order."""
    import torch.multiprocessing as mp
    from merlot_b200 import predict
    from merlot_b200.pretrain_validate import Validator
    from merlot_b200.tf_checkpoint import update_checkpoint_state
    from merlot_b200.train import variables_without_gradient
    from tests.test_gpu_model import build
    from tests.test_gpu_pretrain_validate import _config_dict, _write
    _write(tmp_path, "val", 3, 3, seed=21)  # 9 records: 4 batches of 2, 1 dropped
    model = _tiny(tiny_cfg)
    cfg = _config_dict(tmp_path, model)
    path = tmp_path / "tiny.yaml"
    path.write_text(yaml.safe_dump(cfg))
    config = NeatConfig.from_dict(cfg)
    _, store, _ = build(model, seed=3)
    out_dir = tmp_path / "out"
    os.makedirs(out_dir)
    prefix = str(out_dir / "model.ckpt-6")
    store.save_checkpoint(prefix, skip=variables_without_gradient(model, store))
    update_checkpoint_state(str(out_dir), prefix)
    one = tmp_path / "pred1"
    files = predict.main([str(path), "--out", str(one)])  # the latest checkpoint of device.output_dir
    assert [os.path.basename(f) for f in files] == [f"batch-{k:06d}.npz" for k in range(4)]
    with pytest.raises(ValueError, match="already holds"):
        predict.main([str(path), "--out", str(one)])
    # two ranks sharing the GPU round-robin
    two = tmp_path / "pred2"
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    argv = [str(path), "--out", str(two), "--checkpoint", prefix]
    ps = [ctx.Process(target=_rank_main, args=(r, 2, port, argv, q)) for r in range(2)]
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
    assert sorted(os.listdir(one)) == sorted(os.listdir(two)) == [f"batch-{k:06d}.npz" for k in range(4)]
    for name in os.listdir(one):
        assert (one / name).read_bytes() == (two / name).read_bytes(), name
    # batch k's losses are pretrain_validate's values for batch k
    v = Validator(config, seed=0)
    keys, vecs = v._own_batches(prefix)
    assert len(vecs) == 4
    for k, vec in enumerate(vecs):
        with np.load(one / f"batch-{k:06d}.npz") as z:
            for j, key in enumerate(keys):
                got = float(z[key][0])
                if key.startswith("attn/"):
                    assert got == pytest.approx(float(vec[j + 1]), rel=1e-4, abs=1e-6), (k, key)
                else:
                    assert got == float(vec[j + 1]), (k, key, got, float(vec[j + 1]))
    videos = list(predict.read_predictions(str(one)))
    assert len(videos) == 8
    with np.load(one / "batch-000001.npz") as z:
        for name in z.files:
            np.testing.assert_array_equal(videos[3][name], z[name][1])
