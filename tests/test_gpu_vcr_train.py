"""VCR fine-tuning on the GPU (pytest -m gpu): the answer / rationale classifier towers (merlot_b200/vcr.py cls_head and its
backward) and the VCR training step (vcr_model_fn_builder) against the fp32 oracle restatement of downstream/vcr/modeling.py
(tests/vcr_oracle.py) on bf16-rounded weights, with the oracle drawing the very dropout masks the kernels draw.
Bars: losses 1e-3 relative, activations 1e-2 and gradients 4e-2 relative-Frobenius."""
import math
import os
import socket

import pytest
import torch

from oracle import merlot_oracle as O
from tests import vcr_oracle as V

pytestmark = pytest.mark.gpu
DEV = "cuda"
OCFG = dict(type="adam_optimizer", learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=0, weight_decay_rate=0.01,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"], {"weight_decay_rate": 0}]])


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def vcr_cfg(tiny_cfg, **kw):
    return dict(tiny_cfg, num_texts=4, num_chunks_in_group=1, hidden_dropout_prob=0.1, **kw)


def build(cfg, seed=1, tower_scale=3.0, encoder_scale=5.0, device=DEV, ocfg=OCFG):
    """Oracle-initialised VCR variables, GEMM operands rounded to bf16, loaded into a ParamStore(task="vcr").  Two scalings
    keep the comparison meaningful.  The joint encoder's kernels are scaled so that a sequence's first token depends on its
    text: at the initialisers the four candidates' first tokens agree to a cosine of 0.9999, the tower gradients are then
    sums of nearly cancelling terms, and any bf16 rounding looks like a 30 % error (a fine-tuned model tells its candidates
    apart; here the cosine is 0.90).  The tower kernels are scaled so that the logits depend on the hidden state and on the
    dropout masks, not only on the output bias."""
    from merlot_b200.params import ParamStore
    params = V.init_params(cfg, seed=seed, perturb=0.05)
    for k in params:
        if k.split("/")[0] in V.TOWERS and k.endswith("kernel"):
            params[k] = params[k] * tower_scale
        elif k.startswith("encoder/layer") and k.endswith("kernel"):
            params[k] = params[k] * encoder_scale
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    store = ParamStore(cfg, device=device, optimizer_cfg=ocfg, task="vcr")
    store.load_tf_dict(params)
    return params, store


def batch(cfg, questions, L=16, hw=(64, 96), seed=0):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(2 * questions, *hw, 3, generator=g).bfloat16().float()
    ids = torch.randint(100, cfg["vocab_size"], (2 * questions * 4, L), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(L // 2, L + 1, (2 * questions * 4,), generator=g)
    ids = (ids * (torch.arange(L)[None] < lens[:, None])).int()
    target = torch.randint(0, 4, (2 * questions,), generator=g).int()
    return image, ids, target


def neat(cfg, mode="answer", **opt):
    from merlot_b200.config import NeatConfig
    return NeatConfig.from_dict({"data": {}, "model": dict(cfg, image_size=[64, 96]), "optimizer": dict(OCFG, **opt),
                                 "device": {"use_tpu": False, "output_dir": "/tmp/merlot_vcr"},
                                 "downstream": {"task": "vcr", "mode": mode}})


class _Hidden:
    """What the oracle's head reads of a model: encoder_hidden_states['lang'] as an autograd leaf."""

    def __init__(self, lang):
        self.encoder_hidden_states = {"lang": lang}


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_head_against_autograd(tiny_cfg, p):
    """cls_head + cls_loss + cls_head_backward on a fixed hidden state: logits, loss, every tower gradient and the gradient
    of the hidden state against fp32 autograd (training: the oracle applies the kernels' masks of the same seed).  The hidden
    state's gradient sits at row P of each sequence only; answer_cls is fed by even images and rationale_cls by odd ones (an
    oracle loss with one tower's logits detached gives exactly those rows); an oracle with another seed misses the bar."""
    from merlot_b200 import vcr
    from merlot_b200.modeling import MerlotModel
    cfg = vcr_cfg(tiny_cfg)
    params, store = build(cfg, tower_scale=10.0)
    image, ids, target = batch(cfg, 2)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), params=store)
    B, Sj, H, P = m.B, m._dims["Sj"], cfg["hidden_size"], m.P
    seed = 2 ** 32 + 41
    logits = vcr.cls_head(m, store, dropout=(p, seed))
    loss, acc = vcr.cls_loss(logits, target.to(DEV))
    hidden = m.encoder_info["hidden_state"].float().cpu()
    lang = hidden[:, P:].clone().requires_grad_(True)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items() if k.split("/")[0] in V.TOWERS}
    hook = V.dropout_hook(seed, p) if p > 0 else None
    ref = V.vcr_cls_head_train(_Hidden(lang), leaf, dropout=hook)
    ref_loss, _ = V.vcr_loss(ref, target)
    assert tuple(logits.shape) == (4, 4) and rel(logits, ref) < 1e-2
    assert abs(float(loss) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    # accuracy is the argmax metric of the logits the head computed (a near-tie may flip an argmax within the logits bar)
    assert float(acc) == pytest.approx(float((logits.argmax(-1).cpu() == target.long()).float().mean()), abs=1e-6)
    if p > 0:  # negative control: the masks of another seed
        other = V.vcr_cls_head_train(_Hidden(lang.detach()), leaf, dropout=V.dropout_hook(seed + 1, p))
        assert rel(logits, other) > 1e-2
    store.g.zero_()
    d_hidden = vcr.cls_head_backward(m, store, target.to(DEV)).float().cpu().reshape(B, Sj, H)
    ref_loss.backward()
    grads = store.to_tf_dict("g")
    for k, v in leaf.items():
        if k.endswith("classifier_mlp1/bias"):  # softmax is shift invariant: the output bias's gradient is zero
            assert abs(float(grads[k])) < 1e-6 and abs(float(v.grad)) < 1e-6
            continue
        assert rel(grads[k], v.grad) < 4e-2, k
    assert rel(d_hidden[:, P], lang.grad[:, 0]) < 4e-2
    keep = torch.zeros(Sj, dtype=torch.bool)
    keep[P] = True
    assert float(d_hidden[:, ~keep].abs().max()) == 0.0 and float(d_hidden[:, P].abs().max()) > 0
    # tower routing: the answer tower's loss reaches the even images' sequences only, the rationale tower's the odd ones
    img = torch.arange(B) // 4
    for t, tower in enumerate(V.TOWERS):
        lang_t = lang.detach().clone().requires_grad_(True)
        leaf_t = {k: v.detach().clone().requires_grad_(True) for k, v in leaf.items()}
        lg = V.vcr_cls_head_train(_Hidden(lang_t), leaf_t, dropout=hook)
        mine = (torch.arange(lg.shape[0]) % 2 == t)[:, None]
        V.vcr_loss(torch.where(mine, lg, lg.detach()), target)[0].backward()  # the other tower's upstream gradient zeroed
        other_tower = V.TOWERS[1 - t]
        assert all(leaf_t[k].grad is None or float(leaf_t[k].grad.abs().max()) == 0 for k in leaf_t if k.startswith(other_tower))
        for k in leaf_t:
            if k.startswith(tower):
                assert rel(leaf_t[k].grad, leaf[k].grad) < 1e-6, k
        mine_rows = img % 2 == t
        assert float(lang_t.grad[~mine_rows].abs().max()) == 0.0
        assert rel(d_hidden[mine_rows, P], lang_t.grad[mine_rows, 0]) < 4e-2


def _step_parity(cfg, monkeypatch, hw=(64, 96), seed=2 ** 32 + 5):
    """One VCR training step (2 questions: 4 images, 16 texts) against the oracle: loss, accuracy, every parameter gradient;
    then AdamW against AdamOracle fed the same gradients.  With the hybrid stem the oracle's lite_resnet50 is replaced by a leaf
    holding the GPU's stem output, as tests/test_gpu_stem.py's training step does, and that test's bars apply: the stem's
    own gradients are checked there, the gradient handed to the stem here."""
    from merlot_b200 import vcr
    params, store = build(cfg)
    image, ids, target = batch(cfg, 2, hw=hw, seed=3)
    fn = vcr.vcr_model_fn_builder(neat(cfg), store=store, seed=seed)
    feats = {"images": image.to(DEV).bfloat16(), "lm_input": ids.to(DEV)}
    spec = fn(feats, {"lm_targets": target.to(DEV)}, "train")
    assert spec.metrics["learning_rate"] == pytest.approx(3e-4) and store.global_step == 0
    hybrid = bool(cfg.get("resnet_layers"))
    if hybrid:
        rc = spec.model._stem.tape[-1][1]["y"]
        N, hs, ws = image.shape[0], hw[0] // 16, hw[1] // 16
        leaf_rc = rc.float().cpu().reshape(N, hs, ws, rc.shape[1]).clone().requires_grad_(True)
        monkeypatch.setattr(O, "lite_resnet50", lambda x, p, scope, layers, width=64, rnd=O._ident: leaf_rc)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    hook = V.dropout_hook(seed, 0.1)
    om = O.MerlotOracle(cfg, leaf, image, ids, dropout=hook, log_attention_probs=False)
    assert rel(spec.model.encoder_hidden_states["lang"], om.encoder_hidden_states["lang"]) < 1e-2
    ref_logits = V.vcr_cls_head_train(om, leaf, dropout=hook)
    ref_loss, _ = V.vcr_loss(ref_logits, target)
    assert abs(float(spec.metrics["loss"]) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    gpu_logits = spec.model._vcr_cls[0][:, :4]
    assert rel(gpu_logits, ref_logits) < 1e-2
    assert float(spec.metrics["accuracy"]) == pytest.approx(float((gpu_logits.argmax(-1).cpu() == target.long()).float().mean()),
                                                            abs=1e-6)
    assert spec.loss == pytest.approx(float(spec.metrics["loss"]))
    # the gradients train_op hands to the optimizer: the head backward, then the model backward from its d_hidden_state
    store.g.zero_()
    d_hidden = vcr.cls_head_backward(spec.model, store, target.to(DEV))
    spec.model.backward(d_hidden_state=d_hidden)
    ref_loss.backward()
    grads = store.to_tf_dict("g")
    assert set(grads) == set(leaf)
    worst = {}
    for k, v in leaf.items():
        if "resnet50lite" in k or v.grad is None or float(v.grad.norm()) < 1e-7:  # key biases: exactly zero gradient
            continue
        worst[k] = rel(grads[k], v.grad)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    if hybrid:
        vals = sorted(worst.values())
        assert len(worst) > 40 and max(vals) < 6e-2 and vals[len(vals) // 2] < 2.5e-2, top
        assert rel(spec.model.d_rc, leaf_rc.grad.reshape(N * hs * ws, -1)) < 4e-2
    else:
        assert len(worst) > 40 and max(worst.values()) < 4e-2, top
    for tower in V.TOWERS:
        assert f"{tower}/classifier_mlp1/kernel" in worst and f"{tower}/classifier_mlp0/bias" in worst
    p_before = {k: v.clone() for k, v in store.to_tf_dict("p").items()}
    adam = O.AdamOracle(p_before, OCFG)
    adam.apply_gradients(p_before, grads)
    fn.optimizer.apply_gradients()
    after = store.to_tf_dict("p")
    for k in after:
        assert (after[k] - p_before[k]).abs().max().item() < 2e-6, k
    for tower in V.TOWERS:  # padding columns of classifier_mlp1 stay zero through the update
        assert float(store.P(f"{tower}/classifier_mlp1/kernel")[:, 1:].abs().max()) == 0.0
        assert float(store.P(f"{tower}/classifier_mlp1/bias")[1:].abs().max()) == 0.0
    assert float(store.g.abs().max()) == 0.0 and store.global_step == 1


def test_vcr_step_parity_patch_embed_saved_head(tiny_cfg, monkeypatch):
    _step_parity(vcr_cfg(tiny_cfg), monkeypatch)


def test_vcr_step_parity_hybrid_stem_saved_head(tiny_cfg, monkeypatch):
    _step_parity(vcr_cfg(tiny_cfg, resnet_layers=[1, 2, 1]), monkeypatch)


def test_train_then_evaluate_on_the_trained_tower(tiny_cfg):
    """Two train_op steps, then the eval step (mode 'rationale'): cls_head_val on head_from_store(store, 'rationale') equals
    the oracle's vcr_cls_head_val on the updated weights."""
    from merlot_b200 import vcr
    cfg = vcr_cfg(tiny_cfg)
    _, store = build(cfg)
    image, ids, target = batch(cfg, 2, seed=4)
    fn = vcr.vcr_model_fn_builder(neat(cfg, mode="rationale"), store=store, seed=3)
    before = store.P("rationale_cls/classifier_mlp0/kernel").clone()
    for _ in range(2):
        fn({"images": image.to(DEV).bfloat16(), "lm_input": ids.to(DEV), "lm_targets": target.to(DEV)}).train_op()
    assert store.global_step == 2 and not torch.equal(before, store.P("rationale_cls/classifier_mlp0/kernel"))
    ev_image, ev_ids, ev_target = batch(cfg, 1, seed=6)  # 2 validation images, each with its 4 candidates
    ev_ids = ev_ids.reshape(2, 4, -1)
    spec = fn({"images": ev_image.to(DEV).bfloat16(), "lm_input": ev_ids.to(DEV)}, {"lm_targets": ev_target.to(DEV)}, "eval")
    assert spec.train_op is None
    trained = {k: v.clone() for k, v in store.to_tf_dict("p").items()}
    trained = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in trained.items()}
    om = O.MerlotOracle(cfg, trained, ev_image, ev_ids.reshape(8, -1), log_attention_probs=False)
    ref = O.vcr_cls_head_val(om, trained, "rationale")
    assert tuple(spec.metrics["logits"].shape) == (2, 4) and rel(spec.metrics["logits"], ref) < 1e-2
    ref_loss = torch.nn.functional.cross_entropy(ref, ev_target.long(), reduction="sum") / 2
    assert abs(float(spec.metrics["loss"]) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    assert torch.equal(spec.metrics["predictions"].cpu(), spec.metrics["logits"].argmax(-1).cpu())
    head = vcr.head_from_store(store, "rationale")
    assert tuple(head["rationale_cls/classifier_mlp1/kernel"].shape) == (cfg["hidden_size"] // 2, 1)
    assert tuple(head["rationale_cls/classifier_mlp1/bias"].shape) == (1,)


def test_seeds_of_the_saved_head(tiny_cfg):
    """One seed twice: the same logits and loss, gradients within the fp32-atomics spread; another seed: other logits."""
    from merlot_b200 import vcr
    cfg = vcr_cfg(tiny_cfg)
    image, ids, target = batch(cfg, 2, seed=5)
    out = []
    for seed in (11, 11, 12):
        _, store = build(cfg, tower_scale=10.0)
        fn = vcr.vcr_model_fn_builder(neat(cfg), store=store, seed=seed)
        spec = fn({"images": image.to(DEV).bfloat16(), "lm_input": ids.to(DEV), "lm_targets": target.to(DEV)})
        logits = spec.model._vcr_cls[0][:, :4].clone()
        store.g.zero_()
        spec.model.backward(d_hidden_state=vcr.cls_head_backward(spec.model, store, target.to(DEV)))
        out.append((logits, float(spec.metrics["loss"]), store.g.clone()))
    assert torch.equal(out[0][0], out[1][0]) and out[0][1] == out[1][1]
    assert rel(out[1][2], out[0][2]) < 1e-2
    assert rel(out[2][0], out[0][0]) > 1e-2


def test_full_size_vcr_step():
    """merlot_vcr.yaml per-GPU sizes (8 questions: 16 images of 384x704 through the hybrid stem, 64 texts of 184 tokens), as
    the CLI builds it: finite loss near log 4 at initialisation (output bias -log 3 on every candidate), one full train_op,
    and the peak memory of the step."""
    from merlot_b200 import train, vcr
    from merlot_b200.config import NeatConfig
    model = dict(init_checkpoint=None, transpose_input=True, num_texts=4, image_size=[384, 704], patch_size=16, spatial_pool_size=2,
                 use_bfloat16=True, vocab_size=50370, hidden_size=768, resnet_layers=[3, 4, 9], attention_probs_dropout_prob=0.0,
                 hidden_dropout_prob=0.1, hidden_act="gelu", initializer_range=0.02, intermediate_size=3072,
                 max_position_embeddings=1024, num_attention_heads=12, num_hidden_layers=12,
                 num_vision_transformer_hidden_layers=12, num_lang_transformer_hidden_layers=12, share_params=True)
    optimizer = dict(type="adam_optimizer", learning_rate=0.000012, num_train_steps=60000, num_warmup_steps=6000,
                     weight_decay_rate=0.01, beta_2=0.98, clip_norm=0.0, adafactor=False, use_bfloat16_adam=True, verbose=False,
                     param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias", "batch_normalization"], {"weight_decay_rate": 0}]])
    cfg = NeatConfig.from_dict({"data": {}, "model": model, "optimizer": optimizer,
                                "device": {"use_tpu": False, "output_dir": "/tmp/merlot_vcr", "train_batch_size": 8},
                                "downstream": {"task": "vcr", "mode": "answer"}})
    torch.cuda.reset_peak_memory_stats()
    fn = vcr.vcr_model_fn_builder(cfg)
    feats = train.synthetic_vcr_batch(cfg, 8, seed=0)
    spec = fn(feats)
    loss = float(spec.metrics["loss"])
    assert math.isfinite(loss) and abs(loss - math.log(4.0)) < 0.1, loss
    spec.train_op()
    torch.cuda.synchronize()
    assert fn.store.global_step == 1 and torch.isfinite(fn.store.p).all()
    peak = torch.cuda.max_memory_allocated()
    print(f"VCR step at merlot_vcr.yaml per-GPU sizes on {torch.cuda.get_device_name()}: loss {loss:.4f}, "
          f"peak memory {peak / 2 ** 30:.1f} GiB")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        from merlot_b200 import vcr
        from merlot_b200.train import DataParallel
        dp = DataParallel("nccl")
        tiny = dict(use_bfloat16=True, hidden_size=128, vocab_size=1000, patch_size=16, spatial_pool_size=2, num_attention_heads=2,
                    num_hidden_layers=2, num_vision_transformer_hidden_layers=4, num_lang_transformer_hidden_layers=2,
                    intermediate_size=256, initializer_range=0.02, attention_probs_dropout_prob=0.0, max_position_embeddings=64,
                    resnet_layers=[])
        cfg = vcr_cfg(tiny)
        _, store = build(cfg, device=dev)
        image, ids, target = batch(cfg, 2, seed=20 + rank)
        feats = {"images": image.to(dev).bfloat16(), "lm_input": ids.to(dev), "lm_targets": target.to(dev)}
        fn = vcr.vcr_model_fn_builder(neat(cfg), store=store, dist=dp, device=dev, vit_grad_buckets=2)
        # this rank's gradient, then the replica mean of it
        spec = fn(feats)
        store.g.zero_()
        spec.model.backward(d_hidden_state=vcr.cls_head_backward(spec.model, store, feats["lm_targets"]))
        mean = store.g.clone()
        dp.dist.all_reduce(mean)
        mean /= world
        store.g.zero_()
        # the gradient the optimizer sees in train_op: captured range by range as AdamW is called on it
        seen = torch.zeros_like(store.g)
        apply = fn.optimizer.apply_gradients

        def capture(*a, only=None, **kw):
            for lo, hi in (only if only is not None else [(0, store.total)]):
                seen[lo:hi] = store.g[lo:hi]
            return apply(*a, only=only, **kw)

        fn.optimizer.apply_gradients = capture
        fn(feats).train_op()
        fn.optimizer.apply_gradients = apply
        fn(feats).train_op()
        torch.cuda.synchronize()
        pl = [torch.empty_like(store.p) for _ in range(world)]
        dp.dist.all_gather(pl, store.p)
        q.put({"rank": rank, "grad_rel": rel(seen / world, mean), "params_identical": all(torch.equal(pl[0], x) for x in pl[1:]),
               "step": store.global_step})
        dp.barrier()
    except Exception:
        import traceback
        q.put({"rank": rank, "error": traceback.format_exc()})
        raise


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_vcr_step():
    """Two NCCL ranks on different batches: the gradient train_op hands to AdamW is the replica mean of the ranks' own
    gradients, and the parameters are bit-identical on both ranks after two steps."""
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in ps:
        p.join(timeout=120)
    for r in res:
        assert "error" not in r, r.get("error")
    for r in res:
        assert r["grad_rel"] < 1e-2 and r["params_identical"] and r["step"] == 2, r
