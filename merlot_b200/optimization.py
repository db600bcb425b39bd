"""Mirror of utils/optimization.py: LR schedule, regex parameter groups, fused AdamW step (K10) on the flat arena.

`build_optimizer_from_config` keeps the reference's name, kwargs (YAML `optimizer:` + `device:` sections) and error
behaviour (utils/optimization.py:11-30,137-141,178-179); instead of a TF `train_op` it returns a callable that runs
backward + all-reduce + AdamW.
"""
from __future__ import annotations

from copy import deepcopy
from typing import Iterable, Optional

import numpy as np
import torch

from . import ops
from .params import ParamStore


def learning_rate_scale(step: int, num_train_steps: int, num_warmup_steps: int) -> np.float32:
    """utils/optimization.py:94-115: warmup step/W while step < W, else base*(1 - min(step,T)/T) with
    base = T/(T-W+1) (tf.train.polynomial_decay, power 1, end 0).  fp32 arithmetic like the TF graph."""
    T, W = np.float32(num_train_steps), np.float32(num_warmup_steps)
    base = np.float32(float(num_train_steps) / (float(num_train_steps) - float(num_warmup_steps) + 1.0)) \
        if num_warmup_steps else np.float32(1.0)
    if num_warmup_steps and step < num_warmup_steps:
        return np.float32(np.float32(step) / W)
    gs = np.float32(min(step, num_train_steps))
    return np.float32(base * (np.float32(1.0) - gs / T))


class AdamOptimizer:
    """AdamOptimizer.apply_gradients (utils/optimization.py:339-416) as one fused launch per hyper-parameter group."""

    def __init__(self, store: ParamStore, learning_rate, num_train_steps, num_warmup_steps, use_bfloat16_adam=False,
                 clip_norm=1.0, adafactor=False, **kwargs):
        if adafactor:
            raise ValueError("Adafactor not supported rn")  # optimization.py:178-179
        # The moments' storage was fixed when the ParamStore was built: fp32 for use_bfloat16_adam False (the reference's
        # default), bf16 m and sign-packed bf16 v for True (utils/optimization.py:371-411).
        want_dt = torch.bfloat16 if use_bfloat16_adam else torch.float32
        if store.moment_dtype != want_dt:
            raise ValueError(f"ParamStore keeps {store.moment_dtype} Adam moments but this config sets use_bfloat16_adam: "
                             f"{bool(use_bfloat16_adam)}; build ParamStore(cfg, optimizer_cfg=...) from the same config")
        self.clip_norm = float(clip_norm or 0.0)
        self.store = store
        self.learning_rate = learning_rate
        self.num_train_steps, self.num_warmup_steps = num_train_steps, num_warmup_steps
        # The arena's hyper-parameter groups were fixed when the ParamStore was built; they must be the ones THIS optimizer
        # config implies (utils/optimization.py:125-156), otherwise the update would silently use other rates (e.g. a store
        # built without optimizer_cfg has learning_rate 0 everywhere and would train nothing).
        from .params import hyper_for
        ocfg = dict(kwargs, learning_rate=learning_rate)
        for e in store.entries.values():
            want = {hyper_for(t, ocfg) for t in e.tf_names}
            if want != {tuple(e.hyper)}:
                raise ValueError(f"ParamStore was grouped with other optimizer hyper-parameters than this config gives for "
                                 f"{e.name}: store {tuple(e.hyper)} vs config {sorted(want)}; build ParamStore(cfg, optimizer_cfg=...)")
        if all(h[0] == 0 for h, _, _ in store.groups):
            raise ValueError("every parameter group has learning_rate 0: nothing would be trained")
        self._frozen = [(off, off + cnt) for h, off, cnt in store.groups if h[0] == 0]

    def zero_frozen_grads(self, g: Optional[torch.Tensor] = None):
        """Variables with learning_rate 0 are removed from tvars before tf.gradients / clipping in the reference
        (utils/optimization.py:149-156): their accumulated gradients are discarded here so they neither enter the global norm
        nor grow step after step.  `g`: the gradient arena (default store.g)."""
        g = self.store.g if g is None else g
        for a, b in self._frozen:
            g[a:b].zero_()

    def scalars(self, hyper, step):
        lr, wd, b1, b2, eps = hyper
        b1, b2 = np.float32(b1), np.float32(b2)
        scale = learning_rate_scale(step, self.num_train_steps, self.num_warmup_steps)
        t = np.float32(step) + np.float32(1.0)  # :355
        bc1 = np.float32(1.0) - np.power(b1, t, dtype=np.float32)
        bc2 = np.float32(1.0) - np.power(b2, t, dtype=np.float32)
        lr_t = np.float32(np.float32(np.float32(lr) * scale) * np.sqrt(bc2, dtype=np.float32) / bc1)  # :352-358
        return dict(beta1=float(b1), omb1=float(np.float32(1.0) - b1), beta2=float(b2), omb2=float(np.float32(1.0) - b2),
                    eps=float(np.float32(eps)), lr_t=float(lr_t), wd=float(np.float32(wd)), lr=float(np.float32(lr) * scale))

    def apply_gradients(self, grad_scale: float = 1.0, skip: Iterable[str] = (), zero_grad=True, only=None, advance=True,
                        grads: Optional[torch.Tensor] = None):
        """One optimizer step on every parameter that received a gradient; `skip` lists parameters whose gradient is
        None in the reference (optimization.py:343-344 leaves those untouched).  `only` = [(a, b), ...] restricts the update
        to those arena ranges (data-parallel training updates the already all-reduced part while the rest is in flight);
        pass advance=False for all but the last partial call of a step.  `grads` is the gradient arena to apply, in store.g's
        layout (default store.g; a clipped accumulated step applies store.grad_accumulator())."""
        st = self.store
        g = st.g if grads is None else grads
        step = st.global_step
        if zero_grad:
            self.zero_frozen_grads(g)
        skip_ranges = sorted((st.entries[n].offset, st.entries[n].offset + st.entries[n].padded) for n in skip)
        if only is not None:  # complement of `only` is skipped in this call
            cur, extra = 0, []
            for a, b in sorted(only):
                if a > cur:
                    extra.append((cur, a))
                cur = max(cur, b)
            if cur < st.total:
                extra.append((cur, st.total))
            zero_ranges = [r for r in skip_ranges]
            skip_ranges = sorted(skip_ranges + extra)
        else:
            zero_ranges = skip_ranges
        for hyper, off, cnt in st.groups:
            if hyper[0] == 0:  # learning_rate 0 => not trainable (:149-156)
                continue
            s = self.scalars(hyper, step)
            segs, cur = [], off
            for a, b in skip_ranges:
                if b <= off or a >= off + cnt:
                    continue
                if a > cur:
                    segs.append((cur, a))
                cur = max(cur, b)
            if cur < off + cnt:
                segs.append((cur, off + cnt))
            for a, b in segs:
                ops.adamw_step(st.p[a:b], g[a:b], st.m[a:b], st.v[a:b], st.pb[a:b], b - a, s["beta1"], s["omb1"], s["beta2"],
                               s["omb2"], s["eps"], s["lr_t"], s["wd"], grad_scale, zero_grad)
        if zero_grad and zero_ranges and advance:
            for a, b in zero_ranges:
                g[a:b].zero_()
        if advance:
            st.global_step += 1  # :251-253

    def clip_gradients(self):
        """tf.clip_by_global_norm on the LOCAL gradients -- the reference clips before CrossShardOptimizer averages
        (utils/optimization.py:233-245).  Returns the pre-clip global norm (0-d CUDA tensor) or None when clip_norm == 0."""
        if self.clip_norm <= 0.0:
            return None
        st = self.store
        self.zero_frozen_grads()
        self._clip_buffers()
        ops.clip_by_global_norm(st.g, self.clip_norm, st._clip_scratch, st._clip_norm)
        return st._clip_norm[0]

    def clip_accumulate(self):
        """One micro-batch of a step over A > 1 micro-batches with clip_norm > 0.  The reference clips every replica's own
        gradient before CrossShardOptimizer averages them (utils/optimization.py:233-245), so each micro-batch is clipped
        alone: the learning-rate-0 variables' gradients in store.g are zeroed, then store.grad_accumulator() += clipped
        store.g and store.g = 0 (one K10c call).  Returns the micro-batch's pre-clip norm (0-d CUDA tensor, overwritten by
        the next call)."""
        st = self.store
        self.zero_frozen_grads()
        self._clip_buffers()
        ops.clip_accumulate(st.grad_accumulator(), st.g, self.clip_norm, st._clip_scratch, st._clip_norm)
        return st._clip_norm[0]

    def _clip_buffers(self):
        st = self.store
        if not hasattr(st, "_clip_scratch"):
            st._clip_scratch = torch.zeros(1, dtype=torch.float64, device=st.device)
            st._clip_norm = torch.zeros(1, dtype=torch.float32, device=st.device)

    def current_lr(self):
        return float(np.float32(self.learning_rate) * learning_rate_scale(self.store.global_step, self.num_train_steps,
                                                                          self.num_warmup_steps))


def build_optimizer_from_config(loss, optimizer_config, device_config=None, *, store: ParamStore):
    """utils/optimization.py:11-30.  `loss` is accepted for signature parity (the gradient comes from model.backward())."""
    optimizer_types = {"adam_optimizer": AdamOptimizer}
    if optimizer_config["type"] not in optimizer_types:
        raise ValueError("The optimizer type {} isn't supported".format(optimizer_config["type"]))
    kwargs = deepcopy(optimizer_config)
    if device_config is not None:
        kwargs.update(deepcopy(device_config))
    del kwargs["type"]
    opt = optimizer_types[optimizer_config["type"]](store, **kwargs)
    train_metrics = {"learning_rate": opt.current_lr(), "minibatch_loss": loss}
    return opt, train_metrics
