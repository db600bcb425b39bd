"""Several training steps in a row against float64/fp32 oracles (pytest -m gpu), each step teacher-forced: the oracle is
rebuilt at the weights, moments and global_step the GPU's earlier steps left, so an error in state that crosses a step
boundary shows at the step where it first matters.  State covered: non-zero Adam moments and bias corrections with t > 1,
the learning-rate schedule across the warm-up boundary, the bf16 compute copy `pb` K10 writes, the zeroing of store.g
(padding and skipped entries included), the per-step dropout and masking seed, the buffers _Buffers reuses and the hybrid
stem's cached WsPlan.

At every step k of a run of K steps on one store, with a new batch per step:
  * `pb` equals bf16(p) (round to nearest even) bit for bit over the whole arena;
  * the oracle at the GPU's current weights (bf16-rounded GEMM operands), the step's masks and, with dropout, the hook of
    the step's seed: losses (1e-3 total, 2e-3 per part), hidden states (1e-2) and every gradient AdamW applies (4e-2 per
    tensor; the hybrid stem and clipped accumulation keep the bars of their own tests);
  * AdamOracle.from_state(pre-step p, m, v, global_step) fed the applied gradient: parameters within 2e-6, m and v bit for
    bit; global_step k + 1, store.g all zero, metrics["learning_rate"] = float32(lr * lr_scale(k));
  * at step 0 of the warm-up the learning rate is 0: p is bitwise unchanged while m and v have moved.
Every check can fail: wrong references -- the oracle at the previous step's weights, the previous step's dropout seed,
AdamOracle at global_step k - 1 or from zero moments -- must each miss one of those bars by 2x or more, and from step 1 on
the parameters move by at least 100x the update bar.

Every measured error goes into a JSON report: $MERLOT_TRAJECTORY_REPORT if set, else a fresh file under the temporary
directory (its path is printed)."""
import json
import os
import tempfile
import time

import numpy as np
import pytest
import torch

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O
from tests import share_params_oracle as SO
from tests import test_gpu_clip_accumulation as CA
from tests import test_gpu_model as TM
from tests import test_gpu_vcr_train as VT
from tests import vcr_oracle as V

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 2 ** 32 + 91  # model_fn's run seed; its high word is not zero
# learning-rate scales 0, 0.5, 0.8, 0.6, 0.4: warm-up, then the decay.  Measured on an H100 80GB HBM3 (700 W): at 1.5e-3
# every true reference stays within its bars (worst 0.85 of a bar) and every wrong reference misses by 15x or more (the
# stem output alone at the previous weights misses its bar by 4.3x).
LR, WARMUP, TRAIN_STEPS = 1.5e-3, 2, 6
OCFG = dict(type="adam_optimizer", learning_rate=LR, num_train_steps=TRAIN_STEPS, num_warmup_steps=WARMUP, weight_decay_rate=0.1,
            beta_2=0.98, clip_norm=0.0, use_bfloat16_adam=True,
            param_overrides=[[["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]])
VARIANTS = {
    # patch stem, bf16 moments, hidden dropout in the text stacks and another probability in the ViT
    "headline": dict(steps=5, model=dict(hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2)),
    # the reference's defaults: fp32 moments; no image shuffling, so viz_viz_temporal/ gets no gradient and AdamW skips it
    "reference_default": dict(steps=5, model=dict(hidden_dropout_prob=0.0, vit_hidden_dropout_prob=0.0, image_shuffle_prob=0.0),
                              optimizer=dict(use_bfloat16_adam=False)),
    # three steps: from the fourth on, the gradient of one ViT query bias (a sum of dQ rows that nearly cancel) varies run
    # to run between 0.5x and 1.5x the 6e-2 bar of test_gpu_stem.py at this learning rate, and reaches 4.4x at 3e-3
    "hybrid_stem": dict(steps=3, model=dict(resnet_layers=[1, 2, 1], hidden_dropout_prob=0.0), hw=(128, 192), nc=2),
    "clipped_accumulation": dict(steps=3, accum=2, model=dict(hidden_dropout_prob=0.1), optimizer=dict(clip_norm=1.0)),
    "separate_encoder": dict(steps=3, model=dict(share_params=False, num_lang_transformer_hidden_layers=3,
                                                 hidden_dropout_prob=0.1)),
    "vcr": dict(steps=3, optimizer=dict(num_warmup_steps=0)),
}
BARS = dict(total=1e-3, lang=2e-3, contr=2e-3, temporal=2e-3, hidden_viz=1e-2, hidden_lang=1e-2, logits=1e-2, grad=4e-2,
            gradnorm=2e-2, update=2e-6)
STEM_BARS = dict(grad=6e-2, grad_median=2.5e-2, d_rc=4e-2)  # test_gpu_stem.py::test_training_step_through_the_hybrid_stem
MISS = 2.0
_report = {"path": None, "data": {}}


def record(section, payload):
    if _report["path"] is None:
        _report["path"] = os.environ.get("MERLOT_TRAJECTORY_REPORT") or os.path.join(
            tempfile.mkdtemp(prefix="merlot_trajectory_"), "trajectory.json")
        print(f"trajectory report: {_report['path']}")
    _report["data"][section] = payload
    with open(_report["path"], "w") as f:
        json.dump(_report["data"], f, indent=1, sort_keys=True)


def optimizer_cfg(name):
    base = VT.OCFG if name == "vcr" else OCFG
    return dict(dict(base, learning_rate=LR, num_train_steps=TRAIN_STEPS, num_warmup_steps=WARMUP), **VARIANTS[name].get("optimizer", {}))


def model_cfg(name, tiny_cfg):
    if name == "vcr":
        return VT.vcr_cfg(tiny_cfg)
    return dict(tiny_cfg, **VARIANTS[name].get("model", {}))


def step_seeds(name, k):
    """The dropout and masking seed of each micro-batch of step k on one GPU: SEED + k A + j."""
    A = VARIANTS[name].get("accum", 1)
    return [SEED + k * A + j for j in range(A)]


def lr_scales(name):
    c = optimizer_cfg(name)
    return [float(O.lr_scale(k, c["num_train_steps"], c["num_warmup_steps"])) for k in range(VARIANTS[name]["steps"])]


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def relerr(a, b):
    return abs(float(a) - float(b)) / abs(float(b))


def miss(errs, bars):
    """The largest error-to-bar ratio over the metrics that have a bar."""
    return max(v / bars[k] for k, v in errs.items() if k in bars)


def _moments(store, buf):
    return {nm: t.detach().cpu().contiguous() for _, nm, t in store.tf_views(buf)}


# ---- one step of each kind: (errors of the true reference, {wrong reference: its errors}, bars, applied gradient) ----
class _Pretrain:
    """model_fn over one batch: the oracle's losses, hidden states and gradients at the step's weights and seed."""

    def __init__(self, name, cfg, ocfg):
        from merlot_b200.config import NeatConfig
        from merlot_b200.train import model_fn_builder, variables_without_gradient
        var = VARIANTS[name]
        self.cfg, self.hw, self.nc = cfg, var.get("hw", (64, 96)), var.get("nc", 4)
        self.hybrid = bool(cfg.get("resnet_layers"))
        self.p, self.p_vit = cfg.get("hidden_dropout_prob", 0.0), cfg.get("vit_hidden_dropout_prob", cfg.get("hidden_dropout_prob", 0.0))
        self.params0, self.store, _ = TM.build(cfg, ocfg=ocfg)
        config = NeatConfig.from_dict({"data": {"num_chunks": self.nc, "chunk_text_len": 16},
                                       "model": dict(cfg, image_size=list(self.hw)), "optimizer": ocfg,
                                       "device": {"use_tpu": False, "output_dir": "/tmp/unused"}})
        self.fn = model_fn_builder(config, store=self.store, device=DEV, seed=SEED)
        self.skip = variables_without_gradient(cfg, self.store)
        self.seen = CA.capture_applied(self.fn, self.store)
        self.real_stem = O.lite_resnet50

    def hook(self, seed):
        return DM.dropout_hook(seed, self.p, self.p_vit) if max(self.p, self.p_vit) > 0 else None

    def step(self, k, params, prev, monkeypatch):
        cfg, store = self.cfg, self.store
        image, ids, shuf, vid = TM.synth(cfg, 2, self.nc, 16, *self.hw, seed=k)
        feats = {"images": image.to(DEV).bfloat16(), "input_ids": ids.to(DEV), "shuffled_idx_img": shuf.to(DEV),
                 "video_src_ids": vid.to(DEV)}
        spec = self.fn(feats)
        m = spec.model
        B, Lj = 2 * self.nc // cfg["num_chunks_in_group"], 16 * cfg["num_chunks_in_group"]
        gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj),
              "masked_idx": m.lang_mask_info["masked_idx"].cpu().reshape(B, -1)}
        gpu = [float(x) for x in spec.loss_parts]
        hidden = {n: m.encoder_hidden_states[n].float().cpu() for n in ("viz", "lang")}
        out, bars = {"lr_metric": spec.metrics["learning_rate"]}, dict(BARS)
        if self.hybrid:  # the GPU's stem output against lite_resnet50 at the fp32 weights, bars of test_gpu_stem's forward test
            rc = m._stem.tape[-1][1]["y"].float().cpu()
            N, hs, ws = image.shape[0], self.hw[0] // 16, self.hw[1] // 16
            scope, layers = "vision_backbone/vision_transformer/resnet50lite", cfg["resnet_layers"]
            fp32 = {kk: v for kk, v in prev["p32"].items() if "resnet50lite" in kk}
            ref = self.real_stem(image - 0.5, fp32, scope, layers).reshape(N * hs * ws, -1)
            ref16 = self.real_stem(image - 0.5, fp32, scope, layers, rnd=O.bf16_round).reshape(N * hs * ws, -1)
            bars["stem"] = 1.5 * rel(ref16, ref) + 1e-2
            stem_errs = {"stem": max(rel(rc, ref), rel(rc, ref16))}
            leaf_rc = rc.reshape(N, hs, ws, -1).clone().requires_grad_(True)
            monkeypatch.setattr(O, "lite_resnet50", lambda x, p, scope, layers, width=64, rnd=O._ident: leaf_rc)

        def oracle(p, seed, grad):
            leaf = {kk: v.clone().requires_grad_(grad) for kk, v in p.items()}
            om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm, dropout=self.hook(seed))
            total, info = O.pretrain_losses(om, shuf, vid)
            e = {"total": relerr(sum(gpu), total), "lang": relerr(gpu[0], info["lang"]["loss"]),
                 "contr": relerr(gpu[1], info["contr"]["loss_all"]), "temporal": relerr(gpu[2], info["temporal"]["loss"])}
            if not self.hybrid:
                e.update({f"hidden_{n}": rel(hidden[n], om.encoder_hidden_states[n]) for n in ("viz", "lang")})
            return leaf, total, e

        leaf, total, errs = oracle(params, step_seeds(self.name, k)[0], True)
        wrong = {}
        if prev["moved"] is not None:
            wrong["previous_weights"] = oracle(prev["moved"], step_seeds(self.name, k)[0], False)[2]
            if self.hybrid:
                old = {kk: v for kk, v in prev["p32_before"].items() if "resnet50lite" in kk}
                r_old = self.real_stem(image - 0.5, old, scope, layers).reshape(N * hs * ws, -1)
                wrong["previous_weights"]["stem"] = rel(rc, r_old)
        if k > 0 and self.hook(0) is not None:
            wrong["previous_seed"] = oracle(params, step_seeds(self.name, k - 1)[0], False)[2]
        if self.hybrid:
            errs.update(stem_errs)
        for e in self.skip:  # a gradient sitting in a skipped entry must be neither applied nor left behind
            ent = store.entries[e]
            store.g[ent.offset:ent.offset + ent.padded] = 1.0
        self.seen.clear()
        spec.train_op()
        torch.cuda.synchronize()
        total.backward()
        g = {}
        for kk, v in leaf.items():
            if v.grad is None or float(v.grad.norm()) < 1e-7 or (self.hybrid and "resnet50lite" in kk):
                continue
            g[kk] = rel(self.seen[kk], v.grad)
        vals = sorted(g.values())
        errs["grad"] = vals[-1]
        out["grad_worst"] = max(g, key=g.get)
        norms = torch.stack([v.grad.norm() for v in leaf.values() if v.grad is not None])
        out["grad_worst_norm_and_median"] = [float(leaf[out["grad_worst"]].grad.norm()), float(norms.median())]
        if self.hybrid:
            errs["grad_median"] = vals[len(vals) // 2]
            errs["d_rc"] = rel(m.d_rc, leaf_rc.grad.reshape(N * hs * ws, -1))
            bars.update(STEM_BARS)
        skip_tf = {nm for e_, nm, _ in store.tf_views(store.g) if e_.name in self.skip}
        out["skipped"] = sorted(skip_tf)
        applied = {kk: v.float() for kk, v in self.seen.items() if kk not in skip_tf}
        return errs, wrong, bars, applied, out


class _Clipped:
    """model_fn over A = 2 micro-batches with clip_norm > 0: the replica oracle, each micro-batch's gradient clipped alone
    (test_gpu_clip_accumulation.clipped_step) at a clip_norm below every micro-batch's norm."""

    def __init__(self, name, cfg, ocfg):
        from merlot_b200.config import NeatConfig
        from merlot_b200.train import model_fn_builder
        self.cfg, self.A, self.p = cfg, VARIANTS[name]["accum"], cfg["hidden_dropout_prob"]
        self.params0, self.store, _ = TM.build(cfg, ocfg=ocfg)
        config = NeatConfig.from_dict({"data": {"num_chunks": CA.NC, "chunk_text_len": CA.LC},
                                       "model": dict(cfg, image_size=[64, 96]), "optimizer": ocfg,
                                       "device": {"use_tpu": False, "output_dir": "/tmp/unused"}})
        self.fn = model_fn_builder(config, store=self.store, device=DEV, seed=SEED)
        self.skip = []
        self.seen = CA.capture_applied(self.fn, self.store)

    def step(self, k, params, prev, monkeypatch):
        data, feats = CA.micro_batches(self.cfg, self.A, seed=100 + self.A * k)
        hooks = lambda kk: [DM.dropout_hook(s, self.p) for s in step_seeds(self.name, kk)]
        self.seen.clear()
        r = CA.clipped_step(self.fn, self.cfg, params, data, feats, "all", hooks(k))
        spec, c = r["spec"], r["c"]

        def errors(gs, norms, loss):
            want = CA.clipped_mean(gs, norms, c)
            g = {kk: rel(self.seen[kk], v) for kk, v in want.items() if float(v.norm()) >= 1e-7}
            return {"total": relerr(spec.loss, loss), "grad": max(g.values())}, g

        errs, g = errors(r["gs"], r["norms"], r["ref_loss"])
        errs["gradnorm"] = relerr(spec.metrics["gradnorms/_overall"], sum(r["norms"]) / self.A)
        wrong = {}
        if prev["moved"] is not None:
            gs, loss = CA.oracle_replica_gradients(self.cfg, prev["moved"], data, spec.mask_info, hooks(k))
            wrong["previous_weights"] = errors(gs, [CA.norm_of(x) for x in gs], loss)[0]
        if k > 0:
            gs, loss = CA.oracle_replica_gradients(self.cfg, params, data, spec.mask_info, hooks(k - 1))
            wrong["previous_seed"] = errors(gs, [CA.norm_of(x) for x in gs], loss)[0]
        out = {"lr_metric": spec.metrics["learning_rate"], "grad_worst": max(g, key=g.get), "clip_norm": c, "norms": r["norms"]}
        assert all(n > c for n in r["norms"])
        return errs, wrong, dict(BARS), {kk: v.float() for kk, v in self.seen.items()}, out


class _Vcr:
    """vcr_model_fn_builder: the VCR oracle (tests/vcr_oracle.py) on test_gpu_vcr_train.build's scaled weights."""

    def __init__(self, name, cfg, ocfg):
        from merlot_b200 import vcr
        self.cfg = cfg
        self.params0, self.store = VT.build(cfg, ocfg=ocfg)
        self.fn = vcr.vcr_model_fn_builder(VT.neat(cfg, **{kk: v for kk, v in ocfg.items() if kk != "type"}), store=self.store,
                                           seed=SEED)
        self.skip = []
        self.seen = CA.capture_applied(self.fn, self.store)

    def step(self, k, params, prev, monkeypatch):
        cfg, store = self.cfg, self.store
        image, ids, target = VT.batch(cfg, 2, seed=k)
        spec = self.fn({"images": image.to(DEV).bfloat16(), "lm_input": ids.to(DEV)}, {"lm_targets": target.to(DEV)}, "train")
        gpu_loss, gpu_logits = float(spec.metrics["loss"]), spec.model._vcr_cls[0][:, :4].float().cpu()
        hidden = spec.model.encoder_hidden_states["lang"].float().cpu()

        def oracle(p, seed, grad):
            leaf = {kk: v.clone().requires_grad_(grad) for kk, v in p.items()}
            hook = V.dropout_hook(seed, cfg["hidden_dropout_prob"])
            om = O.MerlotOracle(cfg, leaf, image, ids, dropout=hook, log_attention_probs=False)
            logits = V.vcr_cls_head_train(om, leaf, dropout=hook)
            loss, _ = V.vcr_loss(logits, target)
            return leaf, loss, {"total": relerr(gpu_loss, loss), "logits": rel(gpu_logits, logits),
                                "hidden_lang": rel(hidden, om.encoder_hidden_states["lang"])}

        leaf, loss, errs = oracle(params, step_seeds(self.name, k)[0], True)
        wrong = {}
        if prev["moved"] is not None:
            wrong["previous_weights"] = oracle(prev["moved"], step_seeds(self.name, k)[0], False)[2]
        if k > 0:
            wrong["previous_seed"] = oracle(params, step_seeds(self.name, k - 1)[0], False)[2]
        self.seen.clear()
        spec.train_op()
        torch.cuda.synchronize()
        loss.backward()
        g = {kk: rel(self.seen[kk], v.grad) for kk, v in leaf.items() if v.grad is not None and float(v.grad.norm()) >= 1e-7}
        errs["grad"] = max(g.values())
        for tower in V.TOWERS:  # the classifier's padding columns stay zero through every update
            assert float(store.P(f"{tower}/classifier_mlp1/kernel")[:, 1:].abs().max()) == 0.0, (k, tower)
            assert float(store.P(f"{tower}/classifier_mlp1/bias")[1:].abs().max()) == 0.0, (k, tower)
        out = {"lr_metric": spec.metrics["learning_rate"], "grad_worst": max(g, key=g.get)}
        return errs, wrong, dict(BARS), {kk: v.float() for kk, v in self.seen.items()}, out


def _runner(name, cfg, ocfg):
    kind = _Vcr if name == "vcr" else _Clipped if "accum" in VARIANTS[name] else _Pretrain
    r = kind(name, cfg, ocfg)
    r.name = name
    return r


@pytest.mark.parametrize("name", list(VARIANTS))
def test_trajectory(name, tiny_cfg, monkeypatch):
    t0 = time.time()
    if name == "separate_encoder":
        SO.use_separate_oracle(monkeypatch)
    cfg, ocfg = model_cfg(name, tiny_cfg), optimizer_cfg(name)
    run = _runner(name, cfg, ocfg)
    store, K = run.store, VARIANTS[name]["steps"]
    scales = lr_scales(name)
    steps, before = [], None
    for k in range(K):
        assert store.global_step == k
        pb_ok = torch.equal(TM.bits(store.pb), TM.bits(store.p.bfloat16()))
        p32 = store.to_tf_dict("p")
        pre = dict(p=p32, m=_moments(store, store.m), v=_moments(store, store.v), arena=store.p.clone())
        params = TM.bf16_operands(p32)
        prev = {"p32": p32, "p32_before": before, "moved": None}
        if before is not None and any(not torch.equal(before[kk], p32[kk]) for kk in p32):
            prev["moved"] = TM.bf16_operands(before)
        errs, wrong, bars, applied, out = run.step(k, params, prev, monkeypatch)
        torch.cuda.synchronize()
        # the update against AdamOracle started from the GPU's pre-step state
        post = store.to_tf_dict("p")
        post_m, post_v = _moments(store, store.m), _moments(store, store.v)

        def adam(step, zero_moments=False):
            p = {kk: v.clone() for kk, v in pre["p"].items()}
            m, v = (({kk: torch.zeros_like(t) for kk, t in d.items()} for d in (pre["m"], pre["v"])) if zero_moments
                    else (pre["m"], pre["v"]))
            opt = O.AdamOracle.from_state(p, ocfg, m, v, step)
            opt.apply_gradients(p, applied)
            return p, opt

        def update_err(p):
            return max((post[kk] - p[kk]).abs().max().item() for kk in post)

        ref_p, opt = adam(k)
        errs["update"] = update_err(ref_p)
        moments_exact = all(torch.equal(TM.bits(post_m[kk]), TM.bits(opt.m[kk])) and torch.equal(TM.bits(post_v[kk]), TM.bits(opt.v[kk]))
                            for kk in post_m)
        if k > 0:
            wrong["adam_previous_step"] = {"update": update_err(adam(k - 1)[0])}
            wrong["adam_zero_moments"] = {"update": update_err(adam(k, zero_moments=True)[0])}
        dp = max((post[kk] - pre["p"][kk]).abs().max().item() for kk in post)
        lr_want = float(np.float32(np.float32(ocfg["learning_rate"]) * O.lr_scale(k, ocfg["num_train_steps"], ocfg["num_warmup_steps"])))
        info = dict(step=k, lr_scale=scales[k], pb_equals_bf16_p=pb_ok, errors=errs, bars={kk: bars[kk] for kk in errs},
                    true_miss=miss(errs, bars), max_abs_dp=dp, moments_bitwise=moments_exact,
                    wrong_miss={w: miss(e, bars) for w, e in wrong.items()}, wrong_errors=wrong, lr_metric=float(out.pop("lr_metric")),
                    lr_want=lr_want, global_step_after=store.global_step, g_zero=float(store.g.abs().max()) == 0.0, **out)
        if scales[k] == 0.0:
            info["warmup_p_unchanged"] = torch.equal(TM.bits(store.p), TM.bits(pre["arena"]))
            info["warmup_moments_moved"] = float(store.m.float().abs().max()) > 0 and float(store.v.float().abs().max()) > 0
        info["p_finite"] = bool(torch.isfinite(store.p).all())
        steps.append(info)
        print(f"{name} step {k}: " + json.dumps({kk: info[kk] for kk in ("true_miss", "wrong_miss", "max_abs_dp")}))
        before = p32
        if not info["p_finite"]:  # nothing after a non-finite update is worth comparing
            break
    final_pb = torch.equal(TM.bits(store.pb), TM.bits(store.p.bfloat16()))
    record(name, dict(steps=steps, final_pb_equals_bf16_p=final_pb, wall_s=time.time() - t0, learning_rate=LR))
    for s in steps:
        k = s["step"]
        assert s["p_finite"], f"step {k}: the update left non-finite parameters"
        assert s["pb_equals_bf16_p"], f"step {k}: pb is not bf16(p): the compute copy was not refreshed"
        assert s["true_miss"] < 1.0, (k, s["errors"], s["bars"])
        assert s["moments_bitwise"], f"step {k}: Adam moments differ from AdamOracle"
        assert s["lr_metric"] == s["lr_want"], (k, s["lr_metric"], s["lr_want"])
        assert s["global_step_after"] == k + 1 and s["g_zero"], (k, s["global_step_after"], s["g_zero"])
        if s["lr_scale"] == 0.0:
            assert s["warmup_p_unchanged"] and s["warmup_moments_moved"], k
        else:
            assert s["max_abs_dp"] >= 100 * BARS["update"], (k, s["max_abs_dp"])
        for w, f in s["wrong_miss"].items():
            assert f >= MISS, f"step {k}: the wrong reference {w} misses the bars by only {f:.2f}x: {s['wrong_errors'][w]}"
        if k >= 1:
            assert {"adam_previous_step", "adam_zero_moments"} <= set(s["wrong_miss"]), k
        if k >= 2 or (k >= 1 and s["lr_scale"] > 0 and steps[k - 1]["lr_scale"] > 0):
            assert "previous_weights" in s["wrong_miss"], k
    assert final_pb
