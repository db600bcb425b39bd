"""GPU tests of frame <-> transcript retrieval (pytest -m gpu): K17 element by element against tests/retrieval_oracle.py on
integer-valued scores with planted ties and NaNs; K16 scores + K17 ranks against float64 cosine ranks; the features against
the oracle's contrastive towers; the validator following a trainer's checkpoints, its predictions file, and two ranks on one
GPU against one rank."""
import os
import traceback

import numpy as np
import pytest
import torch
import yaml

from merlot_b200 import _lib
from merlot_b200 import ops
from merlot_b200 import retrieval_validate as RV
from tests import retrieval_oracle as RO

pytestmark = pytest.mark.gpu
DEV = "cuda"
# K16's three-term split misses only xl.yl (|xl| <= 2^-9 |x|) and adds in fp32: over unit vectors its error is far below
# 1e-5.  Queries whose positive is this far from every other key must get the float64 rank.
SEP = 1e-4


def _planted(rows, cols, ld, seed, nan_frac=0.05, levels=7):
    """Integer-valued fp32 scores in [-levels, levels] (many exact ties) with NaNs, in a [rows, ld] buffer; pos random."""
    rng = np.random.default_rng(seed)
    s = rng.integers(-levels, levels + 1, (rows, ld)).astype(np.float32)
    s[rng.random((rows, ld)) < nan_frac] = np.nan
    s[:, cols:] = 1e9  # past the row: must never be read as a column
    pos = rng.integers(0, cols, rows).astype(np.int32)
    return s, pos


def _check_k17(s, pos, cols, k):
    dev = torch.from_numpy(s).to(DEV)[:, :cols]
    got = ops.rank_topk(dev, torch.from_numpy(pos).to(DEV), k)
    got = [t.cpu().numpy() for t in got]
    ref = RO.rank_topk(s[:, :cols], pos, k)
    for name, g, r in zip(("greater", "ties", "topk_idx"), got[:3], ref[:3]):
        assert np.array_equal(g, r), (name, np.argwhere(g != r)[:5])
    assert np.array_equal(got[3], ref[3], equal_nan=True)
    return got


@pytest.mark.parametrize("cols,ld", [(1, 1), (3, 3), (5, 8), (7, 7), (9, 12), (13, 13), (100, 104), (1001, 1003), (4099, 4100),
                                     (5000, 5000)])
def test_k17_matches_oracle_on_ties_and_nans(cols, ld):
    s, pos = _planted(64, cols, ld, seed=cols)
    s[0, pos[0]] = np.nan  # a NaN positive
    got = _check_k17(s, pos, cols, 10)
    assert got[0][0] == -1 and got[1][0] == 0


def test_k17_every_k():
    s, pos = _planted(48, 777, 780, seed=5, levels=3)
    for k in range(1, 33):
        _check_k17(s, pos, 777, k)
    s, pos = _planted(8, 20, 20, seed=6, nan_frac=0.6)  # fewer non-NaN entries than k: index -1, value NaN
    got = _check_k17(s, pos, 20, 32)
    assert (got[2] == -1).any()


def test_k17_long_row_and_many_short_rows():
    s, pos = _planted(1, 1 << 20, 1 << 20, seed=7, levels=1000)
    _check_k17(s, pos, 1 << 20, 32)
    s, pos = _planted(20000, 5, 6, seed=8)
    _check_k17(s, pos, 5, 3)


def test_k17_positive_outside_row_and_shape_errors():
    s, pos = _planted(4, 10, 10, seed=9)
    pos[1], pos[2] = -1, 10
    got = _check_k17(s, pos, 10, 2)
    assert got[0][1] == got[0][2] == -2
    x = torch.zeros(2, 8, device=DEV)
    p = torch.zeros(2, dtype=torch.int32, device=DEV)
    for k in (0, 33):
        with pytest.raises(_lib.MerlotShapeError, match="rank_topk"):
            ops.rank_topk(x, p, k)


def test_k17_is_deterministic():
    s, pos = _planted(300, 3000, 3000, seed=10, levels=2)
    x, p = torch.from_numpy(s).to(DEV), torch.from_numpy(pos).to(DEV)
    a = [t.clone() for t in ops.rank_topk(x, p, 32)]
    for _ in range(3):
        b = ops.rank_topk(x, p, 32)
        assert all(torch.equal(u, v) for u, v in zip(a[:3], b[:3])) and torch.equal(a[3].nan_to_num(7), b[3].nan_to_num(7))


# ---- K16 scores + K17 against float64 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,Cs,chunk", [(3000, 128, 1024), (1029, 256, 100)])
def test_scores_and_ranks_match_float64(n, Cs, chunk):
    g = torch.Generator().manual_seed(n)
    lang = torch.randn(n, Cs, generator=g)
    viz = lang + 1.5 * torch.randn(n, Cs, generator=g)  # noisy pairs: ranks spread over [1, n]
    viz[7] = viz[8]  # two identical keys
    lang, viz = [torch.nn.functional.normalize(t, dim=1) for t in (lang, viz)]
    chunks = [(c, s, e) for c, (s, e) in enumerate(RV.query_chunks(n, chunk))]
    for d, q, k in (("lang_to_viz", lang, viz), ("viz_to_lang", viz, lang)):
        res = RV.rank_chunks(q.to(DEV), k.to(DEV), chunks, chunk, top_k=5)
        greater = np.concatenate([res[c][0] for c, _, _ in chunks])
        idx = np.concatenate([res[c][2] for c, _, _ in chunks])
        val = np.concatenate([res[c][3] for c, _, _ in chunks])
        s64, rank64, gap = RO.cosine_ranks(q.numpy(), k.numpy())
        ok = gap > SEP
        print(f"\n{d}: {ok.sum()} of {n} queries separated by more than {SEP}; median rank {np.median(rank64)}")
        assert ok.mean() > 0.9
        assert np.array_equal(1 + greater[ok], rank64[ok])
        assert np.abs(val - np.take_along_axis(s64, idx, 1)).max() < 1e-5  # the reported scores are the cosines
        assert (np.diff(val, axis=1) <= 0).all()
        if d == "lang_to_viz":  # queries 7 and 8 find their positive tied with the other copy of the key
            ties = np.concatenate([res[c][1] for c, _, _ in chunks])
            assert ties[7] == ties[8] == 1


# ---- features ------------------------------------------------------------------------------------------------------------
def test_features_match_oracle_towers(tiny_cfg):
    from merlot_b200.modeling import MerlotModel
    from oracle import merlot_oracle as O
    from tests.test_gpu_model import build, synth
    cfg = dict(tiny_cfg, hidden_dropout_prob=0.3)  # is_training=False: no dropout whatever the config says
    image, ids, shuf, _ = synth(cfg, 3, 4, 16, 64, 96, 11)
    params, store, _ = build(cfg)
    feats = []
    for seed in (0, 99):  # the masking seed does not reach the features
        m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV).bfloat16(), input_ids=ids.to(DEV),
                        mask_input=True, shuffled_idx_img=shuf.to(DEV), params=store, dropout_seed=seed, features_only=True,
                        log_attention_probs=False)
        lang, viz = m.contrastive_features()
        feats.append((lang.feat.cpu().clone(), viz.feat.cpu().clone()))
    assert all(torch.equal(a, b) for a, b in zip(*feats))
    draws = O.make_mask_draws(6, 32, int(32 * 0.2), cfg["vocab_size"], seed=3)  # 3 videos x 4 chunks in groups of 2
    om = O.MerlotOracle(cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_draws=draws)
    om.contrastive_loss()
    for name, got in zip(("lang", "viz"), feats[0]):
        ref = om.contrastive_feats[name].float()
        cos = (got * ref).sum(1) / ref.norm(dim=1)
        err = (got - ref).abs().max().item()
        print(f"\n{name}: {got.shape[0]} rows, min cosine to the oracle {cos.min().item():.6f}, max abs error {err:.2e}")
        assert got.shape == ref.shape == (12, cfg["contrastive_size"])
        assert cos.min().item() > 0.999 and err < 2e-2


# ---- validator -------------------------------------------------------------------------------------------------------------
def _own_loop(config, prefix, seed=0):
    """The held-out features by a plain loop over the evaluation input, one MerlotModel per batch."""
    from merlot_b200 import dataloader as D
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import ParamStore
    from merlot_b200.train import eval_seed, variables_without_gradient
    store = ParamStore(config.model, device=DEV, optimizer_cfg=config.optimizer)
    store.restore_checkpoint(prefix, skip=variables_without_gradient(config.model, store))
    lang, viz = [], []
    with torch.no_grad(), D.input_fn_builder(config, is_training=False, seed=seed) as pipe:
        for k, b in enumerate(pipe):
            m = MerlotModel(config.model, is_training=False, use_tpu=False, image=b["images"], input_ids=b["input_ids"],
                            mask_input=True, shuffled_idx_img=b["shuffled_idx_img"], params=store, dropout_seed=eval_seed(seed, k),
                            features_only=True, log_attention_probs=False)
            lf, vf = m.contrastive_features()
            lang.append(lf.feat.cpu().clone())
            viz.append(vf.feat.cpu().clone())
    return torch.cat(lang), torch.cat(viz)


def _lines(out_dir):
    import json
    path = out_dir / "eval" / "retrieval.jsonl"
    lines = [json.loads(x) for x in path.read_text().splitlines()]
    path.unlink()
    return lines


def test_validator_follows_trainer_checkpoints_and_writes_predictions(tmp_path, tiny_cfg):
    from merlot_b200.config import NeatConfig
    from tests.test_gpu_pretrain_validate import _trained_run
    path, config = _trained_run(tmp_path, tiny_cfg)  # 9 held-out records of 4 chunks: 4 batches of 2 videos, N = 32
    out = tmp_path / "out"
    clock = iter(range(10 ** 6))
    res = RV.main([path, "--chunk", "5"], clock=lambda: next(clock), sleep=lambda s: None)
    lines = _lines(out)
    assert res == lines and [x["global_step"] for x in lines] == [2, 4] and all(x["segments"] == 32 for x in lines)
    # features: the validator's arenas are the plain loop's rows, bit for bit
    v = RV.Validator(NeatConfig.from_dict(yaml.safe_load(open(path))), chunk=5, top_k=8)
    ckpt = str(out / "model.ckpt-4")
    lang, viz = v.features(ckpt)
    ref_lang, ref_viz = _own_loop(config, ckpt)
    assert torch.equal(lang.cpu(), ref_lang) and torch.equal(viz.cpu(), ref_viz)
    # the chunk size does not change the line
    (r1,) = RV.main([path, "--checkpoint", ckpt, "--chunk", "1024", "--predictions", str(tmp_path / "p.npz"), "--top-k", "8"])
    assert r1 == lines[1] == _lines(out)[0]
    # predictions against float64 cosines of the plain loop's features
    z = np.load(tmp_path / "p.npz")
    assert z["segment"].tolist() == list(range(32)) and z["video"].max() == 1 and z["chunk"].max() == 3 and z["batch"].max() == 3
    for d, q, k in (("lang_to_viz", ref_lang, ref_viz), ("viz_to_lang", ref_viz, ref_lang)):
        s64, rank64, gap = RO.cosine_ranks(q.numpy(), k.numpy())
        ok = gap > SEP
        assert ok.sum() >= 16, ok.sum()
        assert np.array_equal(z[f"{d}_rank"][ok], rank64[ok])
        idx, val = z[f"{d}_topk_idx"], z[f"{d}_topk_score"]
        assert idx.shape == val.shape == (32, 8)
        assert np.abs(val - np.take_along_axis(s64, idx, 1)).max() < 1e-5
        order = np.argsort(-s64, axis=1, kind="stable")[:, :8]
        sep = np.abs(np.diff(np.sort(s64, axis=1)[:, ::-1][:, :9], axis=1)).min(1) > SEP
        assert np.array_equal(idx[sep], order[sep])
        ranks = z[f"{d}_rank"]
        assert r1[d]["r1"] == float(np.mean(ranks <= 1)) and r1[d]["median_rank"] == float(np.median(ranks))


# ---- two ranks on one GPU ----------------------------------------------------------------------------------------------------
def _rank_main(rank, world, port, path, ckpt, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    try:
        clock = iter(range(10 ** 6))
        followed = RV.main([path, "--chunk", "5"], clock=lambda: next(clock), sleep=lambda s: None)
        q.put({"rank": rank, "out": followed + RV.main([path, "--checkpoint", ckpt, "--chunk", "7"])})
    except Exception:
        q.put({"rank": rank, "error": traceback.format_exc()})


def test_two_ranks_write_the_lines_of_one(tmp_path, tiny_cfg):
    import torch.multiprocessing as mp
    from tests.test_gpu_pretrain_validate import _free_port, _trained_run
    path, _ = _trained_run(tmp_path, tiny_cfg)
    out = tmp_path / "out"
    ckpt = str(out / "model.ckpt-4")
    clock = iter(range(10 ** 6))
    one = RV.main([path, "--chunk", "5"], clock=lambda: next(clock), sleep=lambda s: None) + \
        RV.main([path, "--checkpoint", ckpt, "--chunk", "7"])
    one_lines = _lines(out)
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
    assert _lines(out) == one_lines  # rank 0 alone appended, the one-rank lines
    for r in res:
        assert r["out"] == one
