"""Per-micro-batch gradient clipping under accumulation on the GPU (pytest -m gpu): with clip_norm = c > 0 an optimizer step of
A micro-batches on `world` ranks applies (1 / (world A)) sum_v min(1, c / |g_v|) g_v over the virtual replicas v, as the
reference clips every core's gradient before CrossShardOptimizer averages them.
  * ops.clip_accumulate against float64: odd lengths, c below / at / above the norm, an accumulator that holds values;
  * pretraining at A = 2 and 3 against the replica oracle, each replica with its own copy of the parameters so that its
    gradient g_v includes the contrastive terms every other replica's loss sends into its features; c below every norm and
    between them; A = 1 with clipping active against the single-replica oracle;
  * the hybrid stem (resnet_layers): the gradient of each micro-batch, stem included, is the one that gets clipped;
  * VCR at A = 2 against its two micro-batches run alone, clipped in float64 and averaged;
  * `python -m merlot_b200.train` with micro-batches and clip_norm 1.0;
  * on two GPUs (skipped otherwise): world 2 x A 2 against the 4-replica oracle, parameters bit-identical across ranks."""
import os

import pytest
import torch
import yaml

from oracle import merlot_oracle as O
from tests.test_gpu_accumulation import CFG, LC, NC, OCFG, _free_port, neat, params_and_store, rel
from tests.test_gpu_model import synth

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---- the kernel
@pytest.mark.parametrize("n", [1, 7, 4099, 1 << 20 | 3])
def test_clip_accumulate_against_float64(n):
    from merlot_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(n)
    scratch = torch.zeros(1, dtype=torch.float64, device=DEV)
    norm_out = torch.zeros(1, dtype=torch.float32, device=DEV)
    for case in ("below", "equal", "above"):
        x = torch.randn(n, device=DEV, generator=g) * 3.0
        acc0 = torch.randn(n, device=DEV, generator=g)
        norm = float(x.double().norm())
        c = {"below": 0.25 * norm, "equal": float(torch.tensor(norm, dtype=torch.float32)), "above": 4.0 * norm}[case]
        acc, gd = acc0.clone(), x.clone()
        ops.clip_accumulate(acc, gd, c, scratch, norm_out)
        torch.cuda.synchronize()
        want = acc0.double() + x.double() * (c / max(norm, c))
        assert torch.count_nonzero(gd) == 0, case
        assert abs(float(norm_out) - norm) <= 1e-5 * norm, case
        assert ((acc.double() - want).norm() / want.norm()).item() <= 1e-6, case
    with pytest.raises(Exception, match="different arenas"):
        ops.clip_accumulate(gd, gd, 1.0, scratch, norm_out)


# ---- pretraining against the replica oracle
def micro_batches(cfg, A, batch=2, seed=10):
    """A micro-batches; the odd ones repeat one text token, so that their gradients' norms are some 25 % above the others'
    and a clip_norm between them has a margin."""
    data = []
    for j in range(A):
        im, ids, sh, vid = synth(cfg, batch, NC, LC, 64, 96, seed + j)
        if j % 2:
            keep = (ids != 0) & (ids != O.START)
            ids[keep] = 100
        data.append((im, ids, sh, vid))
    feats = [{"images": im.to(DEV).bfloat16(), "input_ids": ids.to(DEV), "shuffled_idx_img": sh.to(DEV),
              "video_src_ids": vid.to(DEV)} for im, ids, sh, vid in data]
    return data, feats


def capture_applied(fn, store):
    """Wrap fn.optimizer.apply_gradients: record {name: gradient AdamW applies} from the arena it reads (grads), times
    grad_scale."""
    seen = {}
    apply = fn.optimizer.apply_gradients

    def capture(*a, grad_scale=1.0, grads=None, **kw):
        buf = store.g if grads is None else grads
        seen.update({nm: t.detach().double().cpu() * grad_scale for _, nm, t in store.tf_views(buf)})
        return apply(*a, grad_scale=grad_scale, grads=grads, **kw)

    fn.optimizer.apply_gradients = capture
    return seen


def oracle_replica_gradients(cfg, params, data, mask_info, dropouts=None):
    """g_v of every replica: each replica holds its own leaf copy of the parameters and the SUM of the per-replica losses is
    differentiated, so leaf_v.grad also carries what the other replicas' contrastive losses send into v's features.
    `dropouts`: each replica's oracle dropout hook (training mode), or None.  Returns ([{name: g_v float64}], mean loss)."""
    B, Lj = 2 * NC // cfg["num_chunks_in_group"], LC * cfg["num_chunks_in_group"]
    leaves = [{k: v.clone().requires_grad_(True) for k, v in params.items()} for _ in data]
    oms = []
    for (im, ids, sh, _), mk, leaf, dropout in zip(data, mask_info, leaves, dropouts or [None] * len(data)):
        gm = {"masked_ids": mk["masked_ids"].cpu().reshape(B, Lj), "masked_idx": mk["masked_idx"].cpu().reshape(B, -1)}
        oms.append(O.MerlotOracle(cfg, leaf, im, ids, mask_input=True, shuffled_idx_img=sh, mask_override=gm, dropout=dropout))
    mean_loss, per = O.pretrain_losses_replicas(oms, [d[2] for d in data], [d[3] for d in data])
    sum(per).backward()
    return [{k: v.grad.double() for k, v in leaf.items() if v.grad is not None} for leaf in leaves], float(mean_loss.detach())


def norm_of(gs):
    return sum(float(t.pow(2).sum()) for t in gs.values()) ** 0.5


def choose_clip(norms, which):
    """c below every norm, or in the widest gap between two of them (some replicas clip, some do not), with margin."""
    s = sorted(norms)
    if which == "all":
        return 0.5 * s[0]
    lo, hi = max(zip(s, s[1:]), key=lambda p: p[1] / p[0])
    assert hi / lo > 1.08, f"norms {s} leave no margin for a clip_norm between them"
    return (lo * hi) ** 0.5


def clipped_mean(gs, norms, c):
    out = {}
    for g, n in zip(gs, norms):
        for k, t in g.items():
            out[k] = out.get(k, 0.0) + t * min(1.0, c / n) / len(gs)
    return out


def run_clipped_step(cfg, A, which):
    from merlot_b200.train import model_fn_builder
    params, store = params_and_store(cfg)
    config = neat(cfg)
    config.optimizer["clip_norm"] = 1.0
    fn = model_fn_builder(config, store=store, device=DEV, seed=3)
    data, feats = micro_batches(cfg, A)
    seen = capture_applied(fn, store)
    r = clipped_step(fn, cfg, params, data, feats, which)
    assert store.global_step == 1 and len(r["snaps"]) == A
    return dict(r, seen=seen)


def clipped_step(fn, cfg, params, data, feats, which, dropouts=None):
    """One optimizer step of fn (clip_norm > 0) over the micro-batches `feats`, whose host copies are `data`: pass 1 draws
    the masks, the replica oracle's gradients at `params` (with `dropouts`) set clip_norm = choose_clip(norms, which), then
    train_op.  Returns the spec, each micro-batch's gradient as clip_accumulate found it in store.g ("snaps"), the oracle's
    gradients, norms and mean loss, and c; checks that both gradient arenas end zeroed."""
    store, snaps = fn.store, []
    clip = fn.optimizer.clip_accumulate

    def snap():
        fn.optimizer.zero_frozen_grads()
        snaps.append({nm: t.detach().double().cpu() for _, nm, t in store.tf_views(store.g)})
        return clip()

    fn.optimizer.clip_accumulate = snap
    spec = fn(feats)  # pass 1 draws the masks the oracle needs
    gs, ref_loss = oracle_replica_gradients(cfg, params, data, spec.mask_info, dropouts)
    norms = [norm_of(g) for g in gs]
    c = choose_clip(norms, which)
    fn.optimizer.clip_norm = c
    spec.train_op()
    torch.cuda.synchronize()
    fn.optimizer.clip_accumulate = clip
    assert len(snaps) == len(feats)
    assert store.g_acc is not None and float(store.g.abs().sum()) == 0.0 and float(store.g_acc.abs().sum()) == 0.0
    return dict(spec=spec, snaps=snaps, gs=gs, norms=norms, c=c, ref_loss=ref_loss)


@pytest.mark.parametrize("A", [2, 3])
@pytest.mark.parametrize("which", ["all", "some"])
def test_clipped_accumulated_pretraining_step_is_the_replica_oracle(A, which):
    r = run_clipped_step(CFG, A, which)
    norms, c = r["norms"], r["c"]
    clipped = sum(n > c for n in norms)
    assert clipped == A if which == "all" else 0 < clipped < A
    want = clipped_mean(r["gs"], norms, c)
    worst = {k: rel(r["seen"][k], v) for k, v in want.items() if float(v.norm()) >= 1e-7}
    got_norm = float(r["spec"].metrics["gradnorms/_overall"])
    print(f"A={A} c={c:.4f} ({clipped} of {A} clip): oracle norms {[round(n, 4) for n in norms]}, gradnorms/_overall "
          f"{got_norm:.4f}; total {r['spec'].loss:.6f} vs {r['ref_loss']:.6f}; worst gradient {max(worst.values()):.2e} "
          f"({max(worst, key=worst.get)})")
    assert abs(r["spec"].loss - r["ref_loss"]) <= 1e-3 * abs(r["ref_loss"])
    assert max(worst.values()) < 4e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    assert abs(got_norm - sum(norms) / A) <= 2e-2 * sum(norms) / A


def test_clipped_pretraining_step_without_accumulation_is_the_oracle():
    """A = 1 with clipping active: clip the local gradient in place, then AdamW (the path of every clipped single-batch step)."""
    from merlot_b200.train import model_fn_builder
    params, store = params_and_store(CFG)
    config = neat(CFG)
    config.optimizer["clip_norm"] = 1.0
    fn = model_fn_builder(config, store=store, device=DEV, seed=3)
    data, feats = micro_batches(CFG, 1)
    seen = capture_applied(fn, store)
    spec = fn(feats[0])
    mk = spec.model.lang_mask_info
    gs, ref_loss = oracle_replica_gradients(CFG, params, data, [mk])
    n = norm_of(gs[0])
    fn.optimizer.clip_norm = c = 0.5 * n
    spec.train_op()
    torch.cuda.synchronize()
    assert store.g_acc is None  # nothing new is allocated at A = 1
    want = clipped_mean(gs, [n], c)
    worst = {k: rel(seen[k], v) for k, v in want.items() if float(v.norm()) >= 1e-7}
    got_norm = float(spec.metrics["gradnorms/_overall"])
    print(f"A=1 c={c:.4f}: oracle norm {n:.4f}, gradnorms/_overall {got_norm:.4f}, worst gradient {max(worst.values()):.2e}")
    assert abs(spec.loss - ref_loss) <= 1e-3 * abs(ref_loss)
    assert max(worst.values()) < 4e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    assert abs(got_norm - n) <= 2e-2 * n


def test_clipped_accumulation_with_the_hybrid_stem(tiny_cfg):
    """resnet_layers set: the stem's conv kernels get their gradients through a cached table of arena pointers (WsPlan).
    Each micro-batch's gradient, stem included, must be what is clipped and folded: AdamW applies (1/A) sum_j clip(g_j) of
    the gradients clip_accumulate found, at fp32 rounding, and those gradients match the replica oracle at the bf16 noise
    floor of a whole graph with a ResNet stem.  test_gpu_stem.py explains that floor: the bf16 stem's output sits ~4e-2 from
    fp32 and that noise reaches every gradient downstream (single tensors up to ~1e-1, the contrastive biases worst), and
    whole-graph stem gradients sit ~30 % from fp32.  So the non-stem gradients are held to 4e-2 as one vector and the stem
    gradients to 0.5; a missing or misdirected stem gradient is 100 % off."""
    cfg = dict(CFG, resnet_layers=[1, 1, 1], hidden_dropout_prob=0.0)
    A = 2
    r = run_clipped_step(cfg, A, "some")
    norms, c, snaps = r["norms"], r["c"], r["snaps"]
    gpu_norms = [norm_of(s) for s in snaps]
    fold = clipped_mean(snaps, gpu_norms, c)
    assert max(rel(r["seen"][k], v) for k, v in fold.items() if float(v.norm()) > 0) < 1e-5
    for j in range(A):
        stem = [k for k in r["gs"][j] if "resnet50lite" in k]
        assert stem and all(float(snaps[j][k].norm()) > 0 for k in stem)
        rest = [k for k in r["gs"][j] if k not in stem]
        rest_rel = rel(torch.cat([snaps[j][k].reshape(-1) for k in rest]), torch.cat([r["gs"][j][k].reshape(-1) for k in rest]))
        stem_rel = rel(torch.cat([snaps[j][k].reshape(-1) for k in stem]), torch.cat([r["gs"][j][k].reshape(-1) for k in stem]))
        print(f"stem, micro-batch {j}: norm {gpu_norms[j]:.4f} vs oracle {norms[j]:.4f}, non-stem gradients {rest_rel:.2e}, "
              f"stem gradients {stem_rel:.2e}")
        assert rest_rel < 4e-2
        assert stem_rel < 0.5
        assert abs(gpu_norms[j] - norms[j]) <= 2e-2 * norms[j]
    assert float(r["spec"].metrics["gradnorms/_overall"]) == pytest.approx(sum(gpu_norms) / A, rel=1e-4)


# ---- VCR
def test_clipped_accumulated_vcr_step_is_the_mean_of_clipped_micro_batches(tiny_cfg):
    from merlot_b200 import vcr
    from tests.test_gpu_vcr_train import batch, build, neat as vcr_neat, vcr_cfg
    cfg = vcr_cfg(tiny_cfg)
    cfg["hidden_dropout_prob"] = 0.0
    parts = [batch(cfg, 2, seed=30 + j) for j in range(2)]
    micro = [{"images": im.to(DEV).bfloat16(), "lm_input": ids.to(DEV), "lm_targets": t.to(DEV)} for im, ids, t in parts]
    alone = []
    for f in micro:  # each micro-batch alone at clip_norm 0: its gradient g_j (grad_scale 1)
        _, store = build(cfg)
        fn = vcr.vcr_model_fn_builder(vcr_neat(cfg), store=store)
        seen = capture_applied(fn, store)
        fn(f).train_op()
        torch.cuda.synchronize()
        alone.append(dict(seen))
    norms = [norm_of(g) for g in alone]
    c = (norms[0] * norms[1]) ** 0.5 if max(norms) / min(norms) > 1.02 else 0.5 * min(norms)
    _, store = build(cfg)
    fn = vcr.vcr_model_fn_builder(vcr_neat(cfg, clip_norm=c), store=store)
    seen = capture_applied(fn, store)
    spec = fn(micro)
    spec.train_op()
    torch.cuda.synchronize()
    assert store.global_step == 1 and store.g_acc is not None
    want = clipped_mean(alone, norms, c)
    got, ref = (torch.cat([d[k].reshape(-1) for k in sorted(want)]) for d in (seen, want))
    got_norm = float(spec.metrics["gradnorms/_overall"])
    print(f"VCR A=2 c={c:.4f}: norms {norms}, gradnorms/_overall {got_norm:.4f}, gradient {rel(got, ref):.2e}")
    assert rel(got, ref) <= 1e-3
    assert abs(got_norm - sum(norms) / 2) <= 1e-3 * sum(norms) / 2


def test_trainer_with_micro_batches_and_clipping_writes_checkpoints(tmp_path, tiny_cfg):
    from merlot_b200.tf_checkpoint import latest_checkpoint
    from merlot_b200.train import main
    out = tmp_path / "out"
    cfg = {"data": {"num_chunks": 4, "chunk_text_len": 16}, "model": dict(tiny_cfg, image_size=[64, 96], vocab_size=50370),
           "optimizer": dict(OCFG, num_train_steps=3, clip_norm=1.0),
           "device": {"output_dir": str(out), "train_batch_size": 4, "micro_batch_size": 2, "iterations_per_loop": 100}}
    path = tmp_path / "run.yaml"
    path.write_text(yaml.safe_dump(cfg))
    main([str(path)])
    assert "model.ckpt-3.index" in os.listdir(out)
    assert latest_checkpoint(str(out)) == str(out / "model.ckpt-3")


# ---- two GPUs
def _two_rank_worker(rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                          LOCAL_RANK=str(rank))
        torch.cuda.set_device(rank)
        dev = f"cuda:{rank}"
        from merlot_b200.params import ParamStore
        from merlot_b200.train import DataParallel, model_fn_builder
        dp = DataParallel("nccl")
        A = 2
        params = O.init_params(CFG, seed=1, perturb=0.05)
        params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v)
                  for k, v in params.items()}
        config = neat(CFG)
        config.optimizer["clip_norm"] = 1.0
        store = ParamStore(CFG, device=dev, optimizer_cfg=config.optimizer)
        store.load_tf_dict(params)
        fn = model_fn_builder(config, store=store, dist=dp, device=dev, seed=3, vit_grad_buckets=2)
        data, _ = micro_batches(CFG, world * A)  # replica v = rank * A + j
        feats = [{"images": im.to(dev).bfloat16(), "input_ids": ids.to(dev), "shuffled_idx_img": sh.to(dev),
                  "video_src_ids": vid.to(dev)} for im, ids, sh, vid in data[rank * A:(rank + 1) * A]]
        seen = capture_applied(fn, store)
        spec = fn(feats)
        mk = torch.cat([torch.cat([m["masked_ids"].reshape(-1), m["masked_idx"].reshape(-1)]) for m in spec.mask_info]).int()
        all_mk = [torch.empty_like(mk) for _ in range(world)]
        dp.dist.all_gather(all_mk, mk)
        B, Lj = 2 * NC // CFG["num_chunks_in_group"], LC * CFG["num_chunks_in_group"]
        masks = []
        for v in range(world * A):
            flat = all_mk[v // A].cpu().view(A, -1)[v % A]
            masks.append({"masked_ids": flat[:B * Lj], "masked_idx": flat[B * Lj:]})
        gs, _ = oracle_replica_gradients(CFG, params, data, masks)  # every rank computes the same oracle
        norms = [norm_of(g) for g in gs]
        c = choose_clip(norms, "some")
        fn.optimizer.clip_norm = c
        spec.train_op()
        torch.cuda.synchronize()
        out = {"rank": rank}
        got_norm = torch.tensor([float(spec.metrics["gradnorms/_overall"])], device=dev)
        all_norm = [torch.empty_like(got_norm) for _ in range(world)]
        dp.dist.all_gather(all_norm, got_norm)
        if rank == 0:
            want = clipped_mean(gs, norms, c)
            worst = {k: rel(seen[k], v) for k, v in want.items() if float(v.norm()) >= 1e-7}
            out.update(grad_max=max(worst.values()), grad_worst=sorted(worst.items(), key=lambda kv: -kv[1])[:5],
                       norms=[float(t) for t in all_norm], ref_norms=[sum(norms[r * A:(r + 1) * A]) / A for r in range(world)],
                       clipped=sum(n > c for n in norms))
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
def test_two_ranks_two_clipped_micro_batches_against_four_replicas():
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
    assert 0 < r0["clipped"] < 4
    assert r0["grad_max"] < 4e-2, r0["grad_worst"]
    for got, ref in zip(r0["norms"], r0["ref_norms"]):
        assert abs(got - ref) <= 2e-2 * ref
    assert all(res[r]["params_identical"] and res[r]["step"] == 3 for r in range(world))
