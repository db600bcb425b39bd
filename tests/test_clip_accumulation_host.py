"""Per-micro-batch gradient clipping on the host (no GPU): the VCR training step over A micro-batches with float64 stand-ins
for the kernels it launches (K10's AdamW, the clip kernels, the metric axpby), a model whose backward adds a known gradient
and a tower backward that adds another.  Checked: every backward writes store.g, each micro-batch is clipped alone into the
store's accumulator, the learning-rate-0 variables stay out of every norm, AdamW applies (1/A) sum_j clip(g_j) from the
accumulator, gradnorms/_overall is the mean of the micro-batches' norms, and with clip_norm 0 (or A = 1) no accumulator is
allocated and no new kernel runs."""
import pytest
import torch

from merlot_b200 import ops
from merlot_b200.modeling import _Buffers

FROZEN = "word_embeddings/word_embeddings"  # learning rate 0 through param_overrides: removed from tvars before clipping


def _config(tiny_cfg, clip_norm):
    from merlot_b200.config import NeatConfig
    ocfg = dict(type="adam_optimizer", learning_rate=1e-4, num_train_steps=100, num_warmup_steps=0, weight_decay_rate=0.01,
                beta_2=0.98, clip_norm=clip_norm, use_bfloat16_adam=True,
                param_overrides=[[["LayerNorm", "layer_norm", "bias"], {"weight_decay_rate": 0}],
                                 [["word_embeddings"], {"learning_rate": 0}]])
    m = dict(tiny_cfg, num_texts=4, image_size=[64, 96], hidden_dropout_prob=0.0, num_chunks_in_group=1)
    return NeatConfig.from_dict({"data": {}, "model": m, "optimizer": ocfg,
                                 "device": {"use_tpu": False, "output_dir": "/tmp/unused"},
                                 "downstream": {"task": "vcr", "mode": "answer"}})


class _Kernels:
    """float64 stand-ins for the kernels of the optimizer step; every call is recorded with the arena it touched."""

    def __init__(self, store):
        self.store, self.calls = store, []

    def arena(self, t):
        """('g' | 'g_acc', element offset) of a view into one of the store's gradient arenas."""
        for name in ("g", "g_acc"):
            base = getattr(self.store, name)
            if base is not None and 0 <= t.data_ptr() - base.data_ptr() < 4 * self.store.total:
                return name, (t.data_ptr() - base.data_ptr()) // 4
        raise AssertionError("not a gradient arena")

    def clip_accumulate(self, acc, g, clip_norm, scratch, norm_out):
        norm = float(g.double().norm())
        self.calls.append(("clip_accumulate", self.arena(acc)[0], self.arena(g)[0], norm))
        acc += (g.double() * (clip_norm / max(norm, clip_norm))).float()
        g.zero_()
        norm_out[0] = norm

    def clip_by_global_norm(self, g, clip_norm, scratch, norm_out):
        norm = float(g.double().norm())
        self.calls.append(("clip_by_global_norm", self.arena(g)[0], norm))
        g.copy_((g.double() * (clip_norm / max(norm, clip_norm))).float())
        norm_out[0] = norm

    def adamw_step(self, p, g, m, v, pb, n, *hyper):
        grad_scale, zero_grad = hyper[-2], hyper[-1]
        self.calls.append(("adamw_step", *self.arena(g), g.double() * grad_scale))
        if zero_grad:
            g.zero_()

    def axpby(self, x, y, a=1.0, b=1.0):
        self.calls.append(("axpby",))
        y.view(-1)[:] = a * x.reshape(-1).double() + (b * y.reshape(-1).double() if b else 0.0)

    def applied(self):
        """The gradient AdamW applied, as one flat arena, and the set of arenas it read."""
        out, arenas = torch.zeros(self.store.total, dtype=torch.float64), set()
        for c in self.calls:
            if c[0] == "adamw_step":
                _, name, off, val = c
                out[off:off + val.numel()] = val
                arenas.add(name)
        return out, arenas


def _step(monkeypatch, tiny_cfg, clip_norm, A, seed=0):
    """One VCR training step over A micro-batches (A = 1: the single-batch step) on a CPU store.  Micro-batch j's model
    gradient has scale 0.5 + j and carries 1e3 in every element of the learning-rate-0 word embeddings; its tower gradient
    (cls_head_backward's writes) is separate.  Returns the store, the recorded kernels, the step, the gradient each micro-batch
    should contribute to its norm (frozen variables zeroed), and (arena, sum |g|) that each backward found when it began."""
    from merlot_b200 import vcr
    from merlot_b200.params import ParamStore
    config = _config(tiny_cfg, clip_norm)
    store = ParamStore(config.model, device="cpu", optimizer_cfg=config.optimizer, task="vcr")
    k = _Kernels(store)
    for name in ("clip_accumulate", "clip_by_global_norm", "adamw_step", "axpby"):
        monkeypatch.setattr(ops, name, getattr(k, name))
    g = torch.Generator().manual_seed(seed)
    fe = store.entries[FROZEN]
    model_g, tower_g = [], []
    for j in range(A):
        t = torch.randn(store.total, generator=g) * (0.5 + j)
        t[fe.offset:fe.offset + fe.numel] = 1e3
        tw = torch.zeros(store.total)
        for e in store.entries.values():
            if e.name.startswith("answer_cls/"):
                tw[e.offset:e.offset + e.numel] = torch.randn(e.numel, generator=g)
        model_g.append(t)
        tower_g.append(tw)
    seen = []

    class Model:
        def __init__(self, params=None, **kw):
            self.store, self._bufs = params, _Buffers(params)

        def backward(self, d_hidden_state=None, **kw):
            self.store.g += model_g[len(seen) - 1]

    def cls_head_backward(model, st, target):  # the first gradient writer of a micro-batch
        seen.append((k.arena(st.g)[0], float(st.g.abs().sum())))
        st.g += tower_g[len(seen) - 1]

    monkeypatch.setattr(vcr, "MerlotModel", Model)
    monkeypatch.setattr(vcr, "cls_head", lambda model, st, dropout=None: None)
    monkeypatch.setattr(vcr, "cls_loss", lambda logits, target: (torch.tensor(1.0), torch.tensor(0.5)))
    monkeypatch.setattr(vcr, "cls_head_backward", cls_head_backward)
    fn = vcr.vcr_model_fn_builder(config, store=store, device="cpu")
    feats = [{"images": torch.zeros(2, 64, 96, 3), "lm_input": torch.zeros(8, 16, dtype=torch.int32),
              "lm_targets": torch.zeros(2, dtype=torch.int32)} for _ in range(A)]
    spec = fn(feats if A > 1 else feats[0])
    spec.train_op()
    frozen = torch.zeros(store.total, dtype=torch.bool)
    for h, off, cnt in store.groups:
        frozen[off:off + cnt] = h[0] == 0
    assert frozen[fe.offset]
    per = [(a + b).double().masked_fill(frozen, 0.0) for a, b in zip(model_g, tower_g)]
    return store, k, spec, per, seen


@pytest.mark.parametrize("A", [2, 3])
@pytest.mark.parametrize("which", ["all clip", "some clip"])
def test_each_micro_batch_is_clipped_alone_into_the_accumulator(monkeypatch, tiny_cfg, A, which):
    norms = sorted(float(p.norm()) for p in _step(monkeypatch, tiny_cfg, 0.0, A)[3])
    c = 0.5 * norms[0] if which == "all clip" else (norms[0] + norms[1]) / 2
    store, k, spec, per, seen = _step(monkeypatch, tiny_cfg, c, A)
    norms = [float(p.norm()) for p in per]
    assert store.g_acc is not None and store.g_acc.shape == store.g.shape and store.g_acc.dtype == torch.float32
    # every micro-batch's backward starts on an empty store.g: the previous one was moved into the accumulator
    assert seen == [("g", 0.0)] * A
    clips = [c_ for c_ in k.calls if c_[0].startswith("clip")]
    assert [c_[:3] for c_ in clips] == [("clip_accumulate", "g_acc", "g")] * A
    # each norm is the micro-batch's own, without the learning-rate-0 variables (1e3 per element would dominate it)
    assert [c_[3] for c_ in clips] == pytest.approx(norms, rel=1e-6)
    assert sum(n > c for n in norms) == (A if which == "all clip" else A - 1)
    applied, arenas = k.applied()
    assert arenas == {"g_acc"}
    want = sum(p * min(1.0, c / n) for p, n in zip(per, norms)) / A
    assert torch.allclose(applied, want, rtol=1e-5, atol=1e-7)
    assert float(spec.metrics["gradnorms/_overall"]) == pytest.approx(sum(norms) / A, rel=1e-6)
    # both arenas are empty again for the next step
    assert float(store.g.abs().sum()) == 0.0 and float(store.g_acc.abs().sum()) == 0.0
    assert store.global_step == 1


@pytest.mark.parametrize("clip_norm,A", [(0.0, 1), (0.0, 3), (1.0, 1)])
def test_no_accumulator_and_no_new_kernel_without_clipped_accumulation(monkeypatch, tiny_cfg, clip_norm, A):
    store, k, spec, per, seen = _step(monkeypatch, tiny_cfg, clip_norm, A)
    assert store.g_acc is None
    assert not any(c[0] == "clip_accumulate" for c in k.calls)
    assert sum(c[0] == "clip_by_global_norm" for c in k.calls) == (1 if clip_norm > 0 else 0)
    assert sum(c[0] == "axpby" for c in k.calls) == (2 * A if A > 1 else 0)  # the loss and accuracy means only
    assert [a for a, _ in seen] == ["g"] * A
    applied, arenas = k.applied()
    assert arenas == {"g"}
    total = sum(per)
    if clip_norm > 0:
        n = float(total.norm())
        total = total * min(1.0, clip_norm / n)
        assert float(spec.metrics["gradnorms/_overall"]) == pytest.approx(n, rel=1e-6)
    else:
        assert "gradnorms/_overall" not in spec.metrics
    assert torch.allclose(applied, total / A, rtol=1e-5, atol=1e-7)
