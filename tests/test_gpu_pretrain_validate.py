"""GPU tests of pretraining validation (pytest -m gpu), at tiny width: model_fn's eval mode against its training mode and
against the oracle, the evaluation input's pixels against the NumPy resize oracle, the validator over two trainer
checkpoints against a per-batch loop, and two ranks against one.

Bitwise comparisons run with masking_use_attn: False.  With it on, mask_inputs ranks tokens by attention sums that K4 adds
up with float atomics, so two runs may pick different tokens at a near tie.  The attn/* metrics come from the joint
encoder's K4 column sums, also float atomics, and are compared to a relative bound instead (ATTN_REL)."""
import io
import json
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import dataloader as D
from merlot_b200 import pretrain_validate as PV
from merlot_b200.config import NeatConfig
from tests import input_oracle as O
from tests import tfrecord_writer as W
from tests.gemm_exact_oracle import bf16_ulps

pytestmark = pytest.mark.gpu
DEV = "cuda"
# K4's float atomics add a few hundred fp32 terms per column in an order that varies between runs: a relative difference of
# a few ulps (1e-7 each), bounded here with a wide margin
ATTN_REL = 1e-5


def _tiny(tiny_cfg, **over):
    return dict(tiny_cfg, image_size=[64, 96], masking_use_attn=False, **over)


def _config_dict(tmp_path, model, steps=4, val_batch_size=2, **validate):
    return {"data": {"train_file": str(tmp_path / "train-*.tfrecord"), "val_file": str(tmp_path / "val-*.tfrecord"),
                     "num_chunks": 4, "chunk_text_len": 16, "random_scale_min": 1.125, "random_scale_max": 1.5,
                     "augment_prob": 0.8, "clean_asr_prob": 0.5, "shuffle_chunks": True, "num_threads": 2,
                     "shuffle_buffer_size": 4},
            "model": model,
            "optimizer": {"type": "adam_optimizer", "learning_rate": 3e-4, "num_train_steps": steps, "num_warmup_steps": 1,
                          "weight_decay_rate": 0.1, "beta_2": 0.98, "clip_norm": 0.0, "use_bfloat16_adam": True},
            "device": {"output_dir": str(tmp_path / "out"), "train_batch_size": 2, "iterations_per_loop": 2,
                       "val_batch_size": val_batch_size},
            "validate": dict(validate)}


def _write(tmp_path, prefix, files, per_file, seed):
    """files x per_file pretraining records of 4 chunks with frames of mixed sizes; returns {record: chunks}."""
    rng = np.random.default_rng(seed)
    sizes = [(70, 100), (66, 99), (81, 123), (64, 96)]
    by_record = {}
    for fi in range(files):
        recs = []
        for e in range(per_file):
            chunks = W.video_chunks(rng, 4, frame_hw=lambda i: sizes[(i + e) % len(sizes)], max_caption=24, video=f"{prefix}{fi}e{e}",
                                    vocab=1000)
            rec = W.chunks_example(chunks)
            by_record[rec] = chunks
            recs.append(rec)
        W.write_records(tmp_path / f"{prefix}-{fi:02d}.tfrecord", recs)
    return by_record


def _vector(spec, keys):
    return torch.stack([spec.total_loss.float()] + [spec.metrics[k].float() for k in keys])


def _assert_lines_equal(got, ref):
    """Results lines equal to the last bit, except attn/* (K4's atomics) within ATTN_REL."""
    assert sorted(got) == sorted(ref)
    for k in ref:
        if k.startswith("attn/"):
            assert got[k] == pytest.approx(ref[k], rel=ATTN_REL), k
        else:
            assert got[k] == ref[k], (k, got[k], ref[k])


# ---- eval mode of model_fn ------------------------------------------------------------------------------------------------
def test_eval_forward_equals_training_forward_and_keeps_state(tmp_path, tiny_cfg):
    from merlot_b200.train import eval_seed, model_fn_builder
    from tests.test_gpu_model import synth
    model = _tiny(tiny_cfg, vit_hidden_dropout_prob=0.2)
    config = NeatConfig.from_dict(_config_dict(tmp_path, model))
    image, ids, shuf, vid = synth(model, 2, 4, 16, 64, 96, 3)  # token ids in [100, vocab_size)
    feats = {"images": image.to(DEV).bfloat16(), "input_ids": ids.to(DEV), "shuffled_idx_img": shuf.to(DEV),
             "video_src_ids": vid.to(DEV)}
    seed, k = 101, 3
    fn_eval = model_fn_builder(config, seed=seed)
    store = fn_eval.store
    before = {n: getattr(store, n).clone() for n in ("p", "g", "m", "v")}
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ev = fn_eval(feats, None, "eval", {"eval_batch": k})
    assert ev.train_op is None and "learning_rate" not in ev.metrics
    keys = sorted(ev.metrics)
    got = _vector(ev, keys).cpu()
    peak_eval = torch.cuda.max_memory_allocated() - base
    for n, t in before.items():  # parameters, gradient arena and moments untouched
        assert torch.equal(getattr(store, n), t), n
    assert store.global_step == 0
    # the training step of a run seeded eval_seed(seed, k) at global_step 0 draws the same dropout and masks
    fn_train = model_fn_builder(config, seed=eval_seed(seed, k))  # a store of its own: its buffers are the training forward's
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    tr = fn_train(feats, None, "train")
    lang, contr, temp = tr.loss_parts
    tr.total_loss = lang + contr + temp
    ref = _vector(tr, keys).cpu()
    peak_train = torch.cuda.max_memory_allocated() - base
    print(f"\npeak memory of one forward: eval {peak_eval / 2**20:.2f} MiB, training {peak_train / 2**20:.2f} MiB")
    assert set(tr.metrics) - set(keys) == {"learning_rate"}
    for i, name in enumerate(["loss"] + keys):
        if name.startswith("attn/"):
            assert float(got[i]) == pytest.approx(float(ref[i]), rel=ATTN_REL), name
        else:
            assert got[i].item() == ref[i].item(), (name, got[i].item(), ref[i].item())
    assert peak_eval < peak_train


def test_eval_metrics_match_oracle(tiny_cfg):
    """Eval mode keeps dropout and masking on (the reference's is_training=True, mask_input=True).  The oracle runs under
    the masks the kernels drew for seed eval_seed(seed, k) (oracle/dropout_mask.py) and the GPU-chosen token mask."""
    from oracle import dropout_mask as DM
    from oracle import merlot_oracle as OM
    from merlot_b200.train import eval_seed, model_fn_builder
    from tests.test_gpu_model import build, rel, synth
    cfg = dict(tiny_cfg, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2)
    image, ids, _, vid = synth(cfg, 2, 4, 16, 64, 96, 0)
    ncg = cfg["num_chunks_in_group"]
    shuf = torch.arange(ncg, dtype=torch.int32).repeat(2 * 4 // ncg)  # the evaluation input's identity order
    params, store, ocfg = build(cfg)
    config = NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": ocfg, "device": {"output_dir": "."}})
    seed, k = 2 ** 32 + 5, 6
    model_fn = model_fn_builder(config, store=store, seed=seed)
    feats = {"images": image.to(DEV).bfloat16(), "input_ids": ids.to(DEV), "shuffled_idx_img": shuf.to(DEV),
             "video_src_ids": vid.to(DEV)}
    spec = model_fn(feats, None, "eval", {"eval_batch": k})
    m = spec.model
    B, Lj = 2 * 4 // ncg, 16 * ncg
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    om = OM.MerlotOracle(cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm,
                         dropout=DM.dropout_hook(eval_seed(seed, k), 0.1, 0.2))
    for name in ("viz", "lang"):
        assert rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name]) < 1e-2  # rel-Frobenius, bf16 stacks
    total_ref, oinfo = OM.pretrain_losses(om, shuf, vid)
    got = {k: float(v) for k, v in spec.metrics.items()}
    # DESIGN 3's bars: each loss head within 2e-3 relative, the summed loss within 1e-3 relative
    for name, ref in (("lang/loss", oinfo["lang"]["loss"]), ("contr/loss_all", oinfo["contr"]["loss_all"]),
                      ("contr/lang_to_viz", oinfo["contr"]["lang_to_viz"]), ("temporal/loss", oinfo["temporal"]["loss"]),
                      ("temporal/lang_viz_loss", oinfo["temporal"]["lang_viz_loss"])):
        assert abs(got[name] - float(ref)) <= 2e-3 * abs(float(ref)), (name, got[name], float(ref))
    assert abs(float(spec.total_loss) - float(total_ref)) <= 1e-3 * abs(float(total_ref))
    for key, v in om.attention_log.items():  # attention_log metrics, the bar of tests/test_gpu_model.py
        assert abs(got[f"attn/{key}"] - float(v)) < 2e-3, key


# ---- evaluation input -----------------------------------------------------------------------------------------------------
def test_eval_pipeline_images_match_oracle(tmp_path, tiny_cfg):
    from PIL import Image
    by_record = _write(tmp_path, "val", 3, 3, seed=21)
    config = NeatConfig.from_dict(_config_dict(tmp_path, _tiny(tiny_cfg)))
    with D.input_fn_builder(config, is_training=False, seed=4) as pipe:
        batches = [(feats, pipe.last_info) for feats in pipe]
        torch.cuda.synchronize()
        assert len(batches) == 4 and pipe.dropped == 1
        for feats, info in batches:
            assert feats["images"].shape == (2 * 4, 64, 96, 3) and feats["images"].dtype == torch.bfloat16
            got = feats["images"].float().cpu().numpy()
            fd = info["frame_draws"]
            for e, rec in enumerate(info["records"]):
                text = O.dataset_parser_text(by_record[rec], 16, bool(info["do_clean"][e]))
                for key in ("input_ids", "video_src_ids", "youtube_id", "chunk_num", "mean_time", "is_eoc"):
                    np.testing.assert_array_equal(feats[key][e].cpu().numpy(), text[key], err_msg=key)
                for j, c in enumerate(by_record[rec]):
                    i = e * 4 + j
                    u8 = np.asarray(Image.open(io.BytesIO(c["image/encoded"])).convert("RGB"))
                    ref, _ = O.load_and_resize_img(u8, (64, 96), fd["scale"][i], fd["u_y"][i], fd["u_x"][i], fd["method"][i],
                                                   fd["augment"][i], fd["factor"][i])
                    d = bf16_ulps(got[i], ref)
                    assert d.max() <= 1 and (d > 0).mean() <= 0.005, (int(d.max()), float((d > 0).mean()))  # the K14 bars
            assert feats["shuffled_idx_img"].tolist() == [0, 1] * 4


# ---- validator ------------------------------------------------------------------------------------------------------------
def _trained_run(tmp_path, tiny_cfg, **validate):
    from merlot_b200 import train
    _write(tmp_path, "train", 2, 3, seed=17)
    _write(tmp_path, "val", 3, 3, seed=21)  # 9 records: 4 batches of 2, 1 dropped
    cfg = _config_dict(tmp_path, _tiny(tiny_cfg), **validate)
    path = tmp_path / "tiny.yaml"
    path.write_text(yaml.safe_dump(cfg))
    train.main([str(path)])
    return str(path), NeatConfig.from_dict(cfg)


def _results(out_dir):
    path = out_dir / "eval" / "results.jsonl"
    lines = [json.loads(x) for x in path.read_text().splitlines()]
    path.unlink()
    return lines


def _per_batch_loop(config, prefix, seed=0):
    """model_fn(..., "eval") over the evaluation input, one batch at a time, and the per-batch means."""
    from merlot_b200.params import ParamStore
    from merlot_b200.train import model_fn_builder, variables_without_gradient
    store = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer)
    model_fn = model_fn_builder(config, store=store, seed=seed)
    store.restore_checkpoint(prefix, skip=variables_without_gradient(config.model, store))
    vecs, keys = [], None
    with torch.no_grad(), D.input_fn_builder(config, is_training=False, seed=seed) as pipe:
        for k, batch in enumerate(pipe):
            spec = model_fn(batch, None, "eval", {"eval_batch": k})
            keys = keys or sorted(spec.metrics)
            vecs.append(_vector(spec, keys).cpu())
    return PV.reduce_batches(keys, vecs, config.device["val_batch_size"], store.global_step, DEV)


def test_validator_follows_trainer_checkpoints(tmp_path, tiny_cfg):
    path, config = _trained_run(tmp_path, tiny_cfg)
    out = tmp_path / "out"
    clock = iter(range(10 ** 6))
    res = PV.main([path], clock=lambda: next(clock), sleep=lambda s: None)
    lines = _results(out)
    assert [r["global_step"] for r in res] == [x["global_step"] for x in lines] == [2, 4]
    keys = {"lang/loss", "lang/acc", "contr/loss_all", "contr/lang_to_viz", "contr/viz_to_lang", "temporal/loss",
            "temporal/lang_viz_loss", "temporal/lang_viz_acc", "temporal/viz_viz_loss", "temporal/viz_viz_acc"}
    keys |= {f"attn/encoder/{p}" for p in ("lang2lang", "lang2viz", "viz2lang", "viz2viz")}
    for r, line, step in zip(res, lines, (2, 4)):
        assert r == line and line["videos"] == 8
        assert set(line) - {"global_step", "loss", "videos"} >= keys and "learning_rate" not in line
        _assert_lines_equal(line, _per_batch_loop(config, str(out / f"model.ckpt-{step}")))
    assert lines[0]["loss"] != lines[1]["loss"]  # two checkpoints, two sets of weights
    # eval_samples truncates: the first batch only
    cfg = yaml.safe_load(open(path))
    cfg["validate"] = {"eval_samples": 3}
    one = tmp_path / "one.yaml"
    one.write_text(yaml.safe_dump(cfg))
    (r,) = PV.main([str(one), "--checkpoint", str(out / "model.ckpt-4")])
    assert r["videos"] == 2 and r["global_step"] == 4


# ---- two ranks --------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, path, ckpt, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    try:
        clock = iter(range(10 ** 6))
        followed = PV.main([path], clock=lambda: next(clock), sleep=lambda s: None)
        q.put({"rank": rank, "out": followed + PV.main([path, "--checkpoint", ckpt])})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


def test_two_ranks_write_the_lines_of_one(tmp_path, tiny_cfg):
    import torch.multiprocessing as mp
    path, _ = _trained_run(tmp_path, tiny_cfg)
    out = tmp_path / "out"
    ckpt = str(out / "model.ckpt-4")
    clock = iter(range(10 ** 6))
    one = PV.main([path], clock=lambda: next(clock), sleep=lambda s: None) + PV.main([path, "--checkpoint", ckpt])
    one_lines = _results(out)
    assert [r["global_step"] for r in one] == [2, 4, 4]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_rank_main, args=(r, 2, port, path, ckpt, q)) for r in range(2)]
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
    two_lines = _results(out)
    assert len(two_lines) == len(one_lines) == 3  # rank 0 alone appended
    for got, ref in zip(two_lines, one_lines):
        _assert_lines_equal(got, ref)
    for r in res:  # every rank returns the result
        for got, ref in zip(r["out"], one):
            _assert_lines_equal(got, ref)
