"""Gradient accumulation on one GPU (pytest -m gpu): an optimizer step of A micro-batches is the data-parallel step of A
replicas.
  * K16, the contrastive head on tensor cores, against float64 at (n, nW) = (32, 32), (40, 120) and (2048, 16384), with a
    label offset and a coefficient, and bitwise-equal repeat runs;
  * pretraining (train.model_fn_builder over a list of micro-batches) against oracle.pretrain_losses_replicas over A oracle
    models, each with its replica's masks: the mean total loss, the contrastive term taken over every micro-batch's features,
    and the gradient AdamW applies; bars of the two-rank data-parallel test (1e-3, 2e-3, 4e-2 relative);
  * with hidden dropout on, the features-only first pass and the training forward give the same features;
  * peak memory does not grow with A beyond the step's feature and head buffers, and stays below the unaccumulated batch;
  * VCR: A = 2 micro-batches of m questions against one batch of 2m at dropout 0;
  * `python -m merlot_b200.train` with device.micro_batch_size writes its checkpoints;
  * on two GPUs (skipped otherwise): world 2 x A 2 against the 4-replica oracle, parameters bit-identical across ranks.
"""
import socket
import os

import pytest
import torch
import yaml

from oracle import merlot_oracle as O
from tests.test_gpu_model import synth

pytestmark = pytest.mark.gpu
DEV = "cuda"
CFG = dict(use_bfloat16=True, hidden_size=128, vocab_size=1000, patch_size=16, spatial_pool_size=2, num_attention_heads=2,
           num_hidden_layers=2, num_vision_transformer_hidden_layers=4, num_lang_transformer_hidden_layers=2,
           intermediate_size=256, initializer_range=0.02, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
           max_position_embeddings=64, num_chunks_in_group=2, do_projection=True, do_bias=True, contrastive_size=128,
           contrast_coef=0.25, contrast_temp=0.05, image_shuffle_prob=0.4, masking_rate=0.2, resnet_layers=[])
OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=10, weight_decay_rate=0.1,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]])
NC, LC = 4, 16


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def neat(cfg, **device):
    from merlot_b200.config import NeatConfig
    return NeatConfig.from_dict({"data": {"num_chunks": NC, "chunk_text_len": LC}, "model": dict(cfg, image_size=[64, 96]),
                                 "optimizer": OCFG, "device": dict({"use_tpu": False, "output_dir": "/tmp/unused"}, **device)})


def params_and_store(cfg):
    from merlot_b200.params import ParamStore
    params = O.init_params(cfg, seed=1, perturb=0.05)
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    store = ParamStore(cfg, device=DEV, optimizer_cfg=OCFG)
    store.load_tf_dict(params)
    return params, store


def micro_batches(cfg, A, batch, seed=10):
    data = [synth(cfg, batch, NC, LC, 64, 96, seed + j) for j in range(A)]
    feats = [{"images": im.to(DEV).bfloat16(), "input_ids": ids.to(DEV), "shuffled_idx_img": sh.to(DEV),
              "video_src_ids": vid.to(DEV)} for im, ids, sh, vid in data]
    return data, feats


def capture_applied_gradient(fn, store):
    """Wrap fn.optimizer.apply_gradients: record {name: gradient AdamW applies} (store.g times grad_scale)."""
    seen = {}
    apply = fn.optimizer.apply_gradients

    def capture(*a, grad_scale=1.0, **kw):
        seen.update({k: v * grad_scale for k, v in store.to_tf_dict("g").items()})
        return apply(*a, grad_scale=grad_scale, **kw)

    fn.optimizer.apply_gradients = capture
    return seen


@pytest.mark.parametrize("A", [2, 3])
def test_accumulated_pretraining_step_is_the_replica_oracle(A):
    from merlot_b200.train import model_fn_builder
    params, store = params_and_store(CFG)
    fn = model_fn_builder(neat(CFG), store=store, device=DEV, seed=3)
    data, feats = micro_batches(CFG, A, batch=2)
    seen = capture_applied_gradient(fn, store)
    spec = fn(feats)
    contr = float(spec.metrics["contr/loss_all"])
    spec.train_op()
    torch.cuda.synchronize()
    assert store.global_step == 1 and len(spec.loss_parts) == 3
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    oms = []
    for (im, ids, sh, _), mk in zip(data, spec.mask_info):
        B, Lj = 2 * NC // CFG["num_chunks_in_group"], LC * CFG["num_chunks_in_group"]
        gm = {"masked_ids": mk["masked_ids"].cpu().reshape(B, Lj), "masked_idx": mk["masked_idx"].cpu().reshape(B, -1)}
        oms.append(O.MerlotOracle(CFG, leaf, im, ids, mask_input=True, shuffled_idx_img=sh, mask_override=gm))
    mean_loss, per = O.pretrain_losses_replicas(oms, [d[2] for d in data], [d[3] for d in data])
    mean_loss.backward()
    ref_total = float(mean_loss.detach())
    ref_contr = sum(float(O.contrastive_loss_replicas(oms, v)[0]) for v in range(A)) / A
    worst = {k: rel(seen[k], v.grad) for k, v in leaf.items() if v.grad is not None and float(v.grad.norm()) >= 1e-7}
    print(f"A={A}: total {spec.loss:.6f} vs {ref_total:.6f}, contrastive {contr:.6f} vs {ref_contr:.6f}, "
          f"worst gradient {max(worst.values()):.2e} ({max(worst, key=worst.get)})")
    assert abs(spec.loss - ref_total) <= 1e-3 * abs(ref_total)
    assert abs(contr - ref_contr) <= 2e-3 * abs(ref_contr)
    assert max(worst.values()) < 4e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:5]


def test_features_only_towers_match_the_training_forward():
    """hidden_dropout_prob 0.1: the first pass (features_only) and the second (the training forward with the first pass's
    masks) compute the same contrastive features under the same seed."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(CFG, hidden_dropout_prob=0.1)
    _, store = params_and_store(cfg)
    (im, ids, sh, _), = micro_batches(cfg, 1, batch=2)[0]
    kw = dict(is_training=True, use_tpu=False, image=im.to(DEV), input_ids=ids.to(DEV), mask_input=True,
              shuffled_idx_img=sh.to(DEV), params=store, dropout_seed=77)
    m1 = MerlotModel(cfg, features_only=True, **kw)
    l1, v1 = (t.feat.clone() for t in m1.contrastive_features())
    masks = {k: v.clone() for k, v in m1.lang_mask_info.items()}
    m2 = MerlotModel(cfg, mask_override=masks, **kw)
    l2, v2 = (t.feat.clone() for t in m2.contrastive_features())
    torch.cuda.synchronize()
    for k in masks:
        assert torch.equal(m2.lang_mask_info[k].reshape(-1), masks[k].reshape(-1))
    print(f"pass 1 vs pass 2 features: lang {rel(l1, l2):.2e}, viz {rel(v1, v2):.2e}, bitwise "
          f"{torch.equal(l1, l2) and torch.equal(v1, v2)}")
    assert torch.equal(l1, l2) and torch.equal(v1, v2)
    # and dropout is on: another seed gives other features
    m3 = MerlotModel(cfg, features_only=True, **dict(kw, dropout_seed=78))
    assert rel(m3.contrastive_features()[0].feat, l1) > 1e-3
    with pytest.raises(RuntimeError, match="save_for_backward"):
        m1.backward()


def _step_peak(cfg, A, batch):
    from merlot_b200.train import model_fn_builder
    _, store = params_and_store(cfg)
    fn = model_fn_builder(neat(cfg), store=store, device=DEV, log_attention_probs=False)
    _, feats = micro_batches(cfg, A, batch)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    spec = fn(feats if A > 1 else feats[0])
    spec.train_op()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del fn, store, spec, feats
    torch.cuda.empty_cache()
    return peak


def test_peak_memory_does_not_grow_with_micro_batches():
    cfg = dict(CFG, hidden_size=256, num_attention_heads=4, intermediate_size=1024, contrastive_size=256)
    m = 4
    p1 = _step_peak(cfg, 1, m)
    p4 = _step_peak(cfg, 4, m)
    p1_big = _step_peak(cfg, 1, 4 * m)
    rows, Cs = 4 * m * NC, cfg["contrastive_size"]  # A n contrastive rows: one per segment
    # the step's buffers: features and their gradients [A n, Cs] x 2 x 2 directions, the all-gathered copies, and the head's
    # logits / their gradients [A n, A n] x 2 x 2 directions, in fp32
    head = 4 * (8 * rows * Cs + 4 * rows * rows)
    print(f"peak above the parameters: A=1 m={m}: {p1 / 2**20:.1f} MiB, A=4 m={m}: {p4 / 2**20:.1f} MiB "
          f"(head buffers {head / 2**20:.2f} MiB), A=1 m={4 * m}: {p1_big / 2**20:.1f} MiB")
    assert p4 <= 1.05 * p1 + head
    assert p4 < p1_big


def test_accumulated_vcr_step_matches_the_whole_batch(tiny_cfg):
    from merlot_b200 import vcr
    from tests.test_gpu_vcr_train import batch, build, neat as vcr_neat, vcr_cfg
    cfg = vcr_cfg(tiny_cfg)
    cfg["hidden_dropout_prob"] = 0.0
    m = 2
    parts = [batch(cfg, m, seed=30 + j) for j in range(2)]
    micro = [{"images": im.to(DEV).bfloat16(), "lm_input": ids.to(DEV), "lm_targets": t.to(DEV)} for im, ids, t in parts]
    whole = {k: torch.cat([f[k] for f in micro], 0) for k in micro[0]}
    grads, losses = [], []
    for feats in (micro, whole):
        _, store = build(cfg)
        fn = vcr.vcr_model_fn_builder(vcr_neat(cfg), store=store)
        seen = capture_applied_gradient(fn, store)
        spec = fn(feats)
        spec.train_op()
        torch.cuda.synchronize()
        assert store.global_step == 1
        grads.append(torch.cat([v.reshape(-1) for v in seen.values()]))
        losses.append(float(spec.metrics["loss"]))
    print(f"VCR A=2 x {m} vs 1 x {2 * m}: loss {losses[0]:.6f} vs {losses[1]:.6f}, gradient {rel(grads[0], grads[1]):.2e}")
    assert abs(losses[0] - losses[1]) <= 1e-4 * abs(losses[1])
    assert rel(grads[0], grads[1]) <= 1e-3


def test_trainer_with_micro_batches_writes_checkpoints(tmp_path, tiny_cfg):
    from merlot_b200.tf_checkpoint import latest_checkpoint
    from merlot_b200.train import main
    out = tmp_path / "out"
    cfg = {"data": {"num_chunks": 4, "chunk_text_len": 16}, "model": dict(tiny_cfg, image_size=[64, 96], vocab_size=50370),
           "optimizer": dict(OCFG, num_train_steps=3),
           "device": {"output_dir": str(out), "train_batch_size": 4, "micro_batch_size": 2, "iterations_per_loop": 100}}
    path = tmp_path / "run.yaml"
    path.write_text(yaml.safe_dump(cfg))
    main([str(path)])
    assert "model.ckpt-3.index" in os.listdir(out)
    assert latest_checkpoint(str(out)) == str(out / "model.ckpt-3")


class _Store:
    device = DEV


class _FakeGather:
    """Rank `rank` of `world` whose all-gather returns the full feature matrices; its reduce-scatter records the gradient of
    all columns (d_y_all) and contributes zeros, so that d_feat is d_x alone."""

    def __init__(self, world, rank, local, full, n):
        self.world, self.rank, self.n, self.local, self.full = world, rank, n, local, full
        self.cols = []

    def all_gather_rows(self, x):
        return next(self.full[k] for k in self.local if self.local[k] is x).clone()

    def reduce_scatter_rows(self, x_all):
        self.cols.append(x_all.clone())
        return torch.zeros(self.n, x_all.shape[1], device=x_all.device)


def _k16_reference(x, y, labels, temp, coeff):
    """float64: per-row loss, d_x and d_y_all of sum_i coeff * CE(x_i . Y^T / temp, label_i)."""
    s = x.double() @ y.double().t() / temp
    lse = torch.logsumexp(s, 1)
    per = lse - s.gather(1, labels.long()[:, None])[:, 0]
    ds = torch.softmax(s, 1)
    ds[torch.arange(x.shape[0]), labels.long()] -= 1.0
    ds *= coeff / temp
    return per, ds @ y.double(), ds.t() @ x.double()


@pytest.mark.parametrize("n,world,rank", [(32, 1, 0), (40, 3, 2), (2048, 8, 5)])
def test_k16_contrastive_head_against_float64(n, world, rank):
    from merlot_b200.modeling import _Buffers, contrastive_head, contrastive_head_bwd
    Cs, temp, coef = 768, 0.05, 0.25
    per_replica = n // 2 if n % 2 == 0 else n
    g = torch.Generator(device=DEV).manual_seed(n)
    full = {k: torch.nn.functional.normalize(torch.randn(world * n, Cs, device=DEV, generator=g), dim=1) for k in ("lang", "viz")}
    mine = slice(rank * n, (rank + 1) * n)
    local = {k: v[mine].clone() for k, v in full.items()}
    cfg = {"contrast_temp": temp, "contrast_coef": coef}
    runs = []
    for _ in range(2):
        bufs = _Buffers(_Store())
        dist = _FakeGather(world, rank, local, full, n) if world > 1 else None
        info, outs = contrastive_head(bufs, cfg, dist, local["lang"], local["viz"], per_replica)
        d_feat = contrastive_head_bwd(bufs, dist, info)
        torch.cuda.synchronize()
        runs.append(dict(l2v=outs["lang_to_viz"].clone(), v2l=outs["viz_to_lang"].clone(),
                         d={k: v.clone() for k, v in d_feat.items()}, cols=list(dist.cols) if dist else []))
    assert torch.equal(runs[0]["l2v"], runs[1]["l2v"]) and torch.equal(runs[0]["v2l"], runs[1]["v2l"])
    assert all(torch.equal(runs[0]["d"][k], runs[1]["d"][k]) for k in ("lang", "viz"))
    assert all(torch.equal(a, b) for a, b in zip(runs[0]["cols"], runs[1]["cols"]))
    labels = torch.arange(n, device=DEV) + rank * n
    r, ref, errs = runs[0], {}, {}
    for name, xk, yk, key in (("lang_to_viz", "lang", "viz", "l2v"), ("viz_to_lang", "viz", "lang", "v2l")):
        per, ref[f"{name} d_x"], ref[f"{name} d_y_all"] = _k16_reference(local[xk], full[yk], labels, temp,
                                                                           coef / 2.0 / per_replica)
        errs[f"{name} loss"] = abs(float(r[key]) - float(per.mean())) / float(per.mean())
    if world > 1:  # d_feat holds d_x; the reduce-scatter received d_y_all (lang_to_viz's columns are viz rows)
        cols = dict(zip(("lang", "viz"), r["cols"]))
        errs["lang_to_viz d_x"] = rel(r["d"]["lang"], ref["lang_to_viz d_x"])
        errs["viz_to_lang d_x"] = rel(r["d"]["viz"], ref["viz_to_lang d_x"])
        errs["lang_to_viz d_y_all"] = rel(cols["viz"], ref["lang_to_viz d_y_all"])
        errs["viz_to_lang d_y_all"] = rel(cols["lang"], ref["viz_to_lang d_y_all"])
    else:  # one rank: d_feat = d_x + d_y_all of the other direction
        errs["d_lang"] = rel(r["d"]["lang"], ref["lang_to_viz d_x"] + ref["viz_to_lang d_y_all"])
        errs["d_viz"] = rel(r["d"]["viz"], ref["viz_to_lang d_x"] + ref["lang_to_viz d_y_all"])
    print(f"K16 n={n} nW={world * n}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v <= (2e-5 if k.endswith("loss") else 2e-4), (k, v)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _two_rank_worker(rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                          LOCAL_RANK=str(rank))
        torch.cuda.set_device(rank)
        global DEV
        DEV = f"cuda:{rank}"
        from merlot_b200.train import DataParallel, model_fn_builder
        dp = DataParallel("nccl")
        A = 2
        params, store = params_and_store(CFG)
        fn = model_fn_builder(neat(CFG), store=store, dist=dp, device=DEV, seed=3, vit_grad_buckets=2)
        data = [synth(CFG, 2, NC, LC, 64, 96, 10 + v) for v in range(world * A)]  # replica v = rank * A + j
        feats = [{"images": im.to(DEV).bfloat16(), "input_ids": ids.to(DEV), "shuffled_idx_img": sh.to(DEV),
                  "video_src_ids": vid.to(DEV)} for im, ids, sh, vid in data[rank * A:(rank + 1) * A]]
        seen = torch.zeros_like(store.g)
        apply = fn.optimizer.apply_gradients

        def capture(*a, grad_scale=1.0, only=None, **kw):
            for lo, hi in (only if only is not None else [(0, store.total)]):
                seen[lo:hi] = store.g[lo:hi] * grad_scale
            return apply(*a, grad_scale=grad_scale, only=only, **kw)

        fn.optimizer.apply_gradients = capture
        spec = fn(feats)
        contr = float(spec.metrics["contr/loss_all"])
        spec.train_op()
        fn.optimizer.apply_gradients = apply
        torch.cuda.synchronize()
        total = torch.tensor([spec.loss, contr], device=DEV)
        mk = torch.cat([torch.cat([m["masked_ids"].reshape(-1), m["masked_idx"].reshape(-1)]) for m in spec.mask_info]).int()
        all_mk = [torch.empty_like(mk) for _ in range(world)]
        dp.dist.all_gather(all_mk, mk)
        all_tot = [torch.empty_like(total) for _ in range(world)]
        dp.dist.all_gather(all_tot, total)
        out = {"rank": rank}
        if rank == 0:
            g_saved = store.g.clone()
            store.g.copy_(seen)
            applied = store.to_tf_dict("g")
            store.g.copy_(g_saved)
            B, Lj = 2 * NC // CFG["num_chunks_in_group"], LC * CFG["num_chunks_in_group"]
            leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
            oms = []
            for v, (im, ids, sh, _) in enumerate(data):
                flat = all_mk[v // A].cpu().view(A, -1)[v % A]
                gm = {"masked_ids": flat[:B * Lj].reshape(B, Lj), "masked_idx": flat[B * Lj:].reshape(B, -1)}
                oms.append(O.MerlotOracle(CFG, leaf, im, ids, mask_input=True, shuffled_idx_img=sh, mask_override=gm))
            mean_loss, per = O.pretrain_losses_replicas(oms, [d[2] for d in data], [d[3] for d in data])
            mean_loss.backward()
            worst = {k: rel(applied[k], v.grad) for k, v in leaf.items() if v.grad is not None and float(v.grad.norm()) >= 1e-7}
            contr_ref = [float(O.contrastive_loss_replicas(oms, v)[0]) for v in range(world * A)]
            out.update(totals=[float(t[0]) for t in all_tot], contrs=[float(t[1]) for t in all_tot],
                       ref_totals=[sum(float(per[r * A + j].detach()) for j in range(A)) / A for r in range(world)],
                       ref_contrs=[sum(contr_ref[r * A:(r + 1) * A]) / A for r in range(world)],
                       grad_max=max(worst.values()), grad_worst=sorted(worst.items(), key=lambda kv: -kv[1])[:5])
        for _ in range(2):
            fn(feats).train_op()
        torch.cuda.synchronize()
        pl = [torch.empty_like(store.p) for _ in range(world)]
        dp.dist.all_gather(pl, store.p)
        out["params_identical"] = all(torch.equal(pl[0], x) for x in pl[1:])
        out["step"] = store.global_step
        q.put(out)
        dp.barrier()
    except Exception:
        import traceback
        q.put({"rank": rank, "error": traceback.format_exc()})
        raise


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_two_micro_batches_against_four_replicas():
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_two_rank_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in ps:
        p.join(timeout=120)
    for r in res:
        assert "error" not in r, r.get("error")
    res = {r["rank"]: r for r in res}
    r0 = res[0]
    for r in range(world):
        assert abs(r0["totals"][r] - r0["ref_totals"][r]) <= 1e-3 * abs(r0["ref_totals"][r]), r
        assert abs(r0["contrs"][r] - r0["ref_contrs"][r]) <= 2e-3 * abs(r0["ref_contrs"][r]), r
    assert r0["grad_max"] < 4e-2, r0["grad_worst"]
    assert all(res[r]["params_identical"] and res[r]["step"] == 3 for r in range(world))


def test_k16_operand_kernels_write_the_split_layouts():
    """ops.ctr_split / ops.ctr_dlogits element by element: hi = bf16(v), lo = bf16(v - hi), in the side-by-side and stacked
    layouts the K16 GEMMs read."""
    from merlot_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(0)
    rows, C = 40, 24
    x = torch.randn(rows, C, device=DEV, generator=g)
    h = x.bfloat16()
    lo = (x - h.float()).bfloat16()
    side = torch.zeros(rows, 3 * C + 8, dtype=torch.bfloat16, device=DEV)
    ops.ctr_split(x, side, side.stride(0), C, 0b100)
    assert torch.equal(side[:, :C], h) and torch.equal(side[:, C:2 * C], h) and torch.equal(side[:, 2 * C:3 * C], lo)
    stack = torch.zeros(3 * rows, C, dtype=torch.bfloat16, device=DEV)
    ops.ctr_split(x, stack, C, rows * C, 0b010)
    assert torch.equal(stack[:rows], h) and torch.equal(stack[rows:2 * rows], lo) and torch.equal(stack[2 * rows:], h)
    n, nW = 40, 120
    logits = torch.randn(n, 128, device=DEV, generator=g) * 4
    labels = (torch.arange(n, device=DEV, dtype=torch.int32) * 3) % nW
    lse = torch.logsumexp(logits[:, :nW], 1).float()
    coeff = torch.rand(n, device=DEV, generator=g)
    dsh = torch.zeros(n, 3 * nW, dtype=torch.bfloat16, device=DEV)
    dsv = torch.zeros(3 * n, 128, dtype=torch.bfloat16, device=DEV)
    ops.ctr_dlogits(logits, labels, nW, lse, coeff, 20.0, dsh, dsv)
    p = torch.softmax(logits[:, :nW].double(), 1)
    p[torch.arange(n), labels.long()] -= 1.0
    ds = p * coeff.double()[:, None] * 20.0
    got = dsh[:, :nW].double() + dsh[:, 2 * nW:].double()
    assert ((got - ds).norm() / ds.norm()).item() < 1e-5
    assert torch.equal(dsh[:, :nW], dsh[:, nW:2 * nW])
    assert torch.equal(dsv[:n, :nW], dsh[:, :nW]) and torch.equal(dsv[n:2 * n, :nW], dsh[:, :nW])
    assert torch.equal(dsv[2 * n:, :nW], dsh[:, 2 * nW:])
