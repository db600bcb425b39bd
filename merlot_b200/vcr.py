"""VCR downstream pieces (SURVEY 8(f)-3): downstream/vcr/modeling.py over MerlotModel(num_texts=4).

`MerlotModel(config with num_texts: 4, image=[b, h, w, 3], input_ids=[b*4, L])` tiles every image's tokens to its four
candidate texts (model/modeling.py:111-119; merlot_b200/modeling.py does that with four LayerNorm row remaps).  This module adds
  * `cls_head_val` (downstream/vcr/modeling.py:57-77): first language token -> dense(H/2)+gelu -> dense(1) -> [img_batch, 4]
    logits, on a dict of variables keyed by the reference's names (`<mode>_cls/classifier_mlp{0,1}/{kernel,bias}`), from
    `init_head`, a checkpoint, or `head_from_store` (a store trained by the VCR step);
  * `cls_loss` (:133-143): softmax cross entropy over the four candidates, summed over images / img_batch_size;
  * `cls_head` / `cls_head_backward` (:77-127): the TRAINING head, one answer_cls and one rationale_cls tower of
    dropout -> dense(H/2)+gelu -> dropout -> dense(1), with variables in a ParamStore(task="vcr"); its backward writes the
    towers' gradients into store.g and returns the gradient that enters the model through MerlotModel.backward(d_hidden_state=...);
  * `vcr_model_fn_builder` (:23-219): the fine-tuning step (train) and the validation forward (eval).
All arithmetic runs in libmerlot_b200.so (K1 GEMM with its fused epilogues, the row gather / scatter, dropout, the CE kernel,
the strided fp32 small GEMM).
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from . import ops
from .modeling import (MerlotModel, _SITE_VCR_ANS_HID, _SITE_VCR_ANS_IN, _SITE_VCR_RAT_HID, _SITE_VCR_RAT_IN, _SoftmaxCE)
from .params import VCR_TOWERS

# (variable scope, input-dropout site, hidden-dropout site); image 2i of a question feeds tower 0, image 2i+1 tower 1 (:79-84)
_TOWERS = ((VCR_TOWERS[0], _SITE_VCR_ANS_IN, _SITE_VCR_ANS_HID), (VCR_TOWERS[1], _SITE_VCR_RAT_IN, _SITE_VCR_RAT_HID))


def init_head(hidden_size: int, mode: str = "answer", initializer_range: float = 0.02, bias_pi: float = 0.25, seed: int = 0,
              device="cuda") -> Dict[str, torch.Tensor]:
    """Reference initialisers (downstream/vcr/modeling.py:63-74): truncated normal kernels, bias1 = -log((1-pi)/pi)."""
    g = torch.Generator().manual_seed(seed)
    k0 = torch.empty(hidden_size, hidden_size // 2)
    k1 = torch.empty(hidden_size // 2, 1)
    for t in (k0, k1):
        torch.nn.init.trunc_normal_(t, 0.0, initializer_range, -2 * initializer_range, 2 * initializer_range, generator=g)
    p = {f"{mode}_cls/classifier_mlp0/kernel": k0, f"{mode}_cls/classifier_mlp0/bias": torch.zeros(hidden_size // 2),
         f"{mode}_cls/classifier_mlp1/kernel": k1, f"{mode}_cls/classifier_mlp1/bias": torch.full((1,), -math.log((1 - bias_pi) / bias_pi))}
    return {k: v.to(device) for k, v in p.items()}


def cls_head_val(model, head: Dict[str, torch.Tensor], mode: str = "answer") -> torch.Tensor:
    """downstream/vcr/modeling.py:57-77 on model.encoder_hidden_states['lang'] -> fp32 logits [img_batch_size, 4]."""
    y = model.encoder_info["hidden_state"]  # bf16 [B, P+L, H]; encoder_hidden_states['lang'][:, 0] is its row P (cast to fp32 there)
    B, Sj, H = y.shape
    lang0 = model.encoder_pieces[1]["start"]  # P * num_imgs: the language piece follows every image's viz tokens
    if B % 4 != 0:
        raise ValueError(f"VCR heads score 4 candidates per image: batch {B} is not a multiple of 4")
    dev = y.device
    first = torch.empty((B, H), dtype=torch.bfloat16, device=dev)
    idx = (torch.arange(B, device=dev, dtype=torch.int32) * Sj + lang0).contiguous()
    ops.gather_rows(y.reshape(B * Sj, H), idx, first)  # hidden_state[:, 0, :] of the language piece
    k0 = head[f"{mode}_cls/classifier_mlp0/kernel"].to(torch.bfloat16).contiguous()
    pre = ops.gemm(first, k0, b_mn_major=True, bias=head[f"{mode}_cls/classifier_mlp0/bias"].float().contiguous(), out_dtype=torch.float32)
    act = torch.empty_like(pre)
    ops.gelu_f32(pre, act)
    actb = torch.empty(pre.shape, dtype=torch.bfloat16, device=dev)
    ops.cast_f32_to_bf16(act, actb)
    k1 = torch.zeros((H // 2, 8), dtype=torch.bfloat16, device=dev)  # N = 1 padded to a TMA-legal row of 8
    k1[:, :1] = head[f"{mode}_cls/classifier_mlp1/kernel"].to(torch.bfloat16)
    b1 = torch.zeros(8, dtype=torch.float32, device=dev)
    b1[:1] = head[f"{mode}_cls/classifier_mlp1/bias"].float()
    logits = ops.gemm(actb, k1, b_mn_major=True, bias=b1, out_dtype=torch.float32)  # [B, 8], column 0 is the logit
    return logits[:, 0].reshape(B // 4, 4)


def cls_loss(logits_flat: torch.Tensor, target: torch.Tensor):
    """downstream/vcr/modeling.py:133-150: mean softmax cross entropy over the 4 candidates + accuracy (0-d CUDA tensors)."""
    n = logits_flat.shape[0]
    dev = logits_flat.device
    padded = torch.zeros((n, 8), dtype=torch.float32, device=dev)
    padded[:, :4] = logits_flat
    per, lse, corr = (torch.empty(n, dtype=torch.float32, device=dev) for _ in range(3))
    ops.softmax_ce_fwd(padded, target.to(torch.int32).contiguous(), 4, per, lse, corr)
    out2 = torch.empty(2, dtype=torch.float32, device=dev)
    coeff = torch.empty(n, dtype=torch.float32, device=dev)
    ops.weighted_loss(per, corr, None, None, 0, 1.0, out2, coeff)
    return out2[0], out2[1]


def head_from_store(store, mode: str = "answer") -> Dict[str, torch.Tensor]:
    """The `<mode>_cls` variables of a ParamStore(task="vcr") as the dict `cls_head_val` takes: views of the fp32 master arena
    at the reference's shapes (classifier_mlp1 [H/2, 1] and [1], without the padding columns).  EVAL / PREDICT use the
    training tower of the same name (downstream/vcr/modeling.py:59, `{downstream.mode}_cls`)."""
    sc = f"{mode}_cls"
    if f"{sc}/classifier_mlp0/kernel" not in store.entries:
        raise KeyError(f"the store has no {sc} tower (build it with ParamStore(..., task='vcr'); mode is 'answer' or 'rationale')")
    return {f"{sc}/classifier_mlp0/kernel": store.P(f"{sc}/classifier_mlp0/kernel"),
            f"{sc}/classifier_mlp0/bias": store.P(f"{sc}/classifier_mlp0/bias"),
            f"{sc}/classifier_mlp1/kernel": store.P(f"{sc}/classifier_mlp1/kernel")[:, :1],
            f"{sc}/classifier_mlp1/bias": store.P(f"{sc}/classifier_mlp1/bias")[:1]}


def _head_index(model, b: int, Sj: int):
    """Per tower: int32 [4b] rows of the joint hidden state (the first language row, P * num_imgs, of every sequence of Sj
    rows) that the tower reads,
    question-major (row 4q + c = candidate text c of question q); plus the constant E fp32 [32, 4], E[8c, c] = 1, that moves
    logits between a tower's padded dense(1) output and the [2b, 4] logits (see cls_head)."""
    bf, dev = model._bufs, model.store.device
    P = model.encoder_pieces[1]["start"]  # P * num_imgs
    key = ("_vcr_idx", b, Sj, P)
    if key not in bf.d:
        q = torch.arange(b, device=dev)[:, None]
        c = torch.arange(4, device=dev)[None]
        idx = [(((2 * q + t) * 4 + c) * Sj + P).reshape(-1).to(torch.int32).contiguous() for t in (0, 1)]
        sel = torch.zeros((32, 4), dtype=torch.float32, device=dev)
        sel[torch.arange(4) * 8, torch.arange(4)] = 1.0
        bf.d[key] = (idx, sel)
    return bf.d[key]


def cls_head(model, store, dropout=(0.0, 0)) -> torch.Tensor:
    """downstream/vcr/modeling.py:77-127 on model.encoder_info['hidden_state'] -> fp32 logits [img_batch_size, 4]: row 2i holds
    question i's answer logits, row 2i+1 its rationale logits.  dropout = (p, seed): the reference's hidden_dropout_prob and the
    step's dropout seed (the sites are _SITE_VCR_* of modeling.py).  The tower variables are store's
    `{answer,rationale}_cls/classifier_mlp{0,1}/{kernel,bias}` (classifier_mlp1 zero-padded to 8 output columns)."""
    y = model.encoder_info["hidden_state"]  # bf16 [B, P+L, H]; row P of a sequence is encoder_hidden_states['lang'][:, 0]
    B, Sj, H = y.shape
    if B % 8 != 0 or model.num_texts != 4:
        raise ValueError(f"the VCR training head scores 2 images (answer, rationale) x 4 texts per question: batch {B}, "
                         f"num_texts {model.num_texts}")
    b, H2 = B // 8, H // 2
    p, seed = float(dropout[0]), int(dropout[1])
    bf = model._bufs
    idx, sel = _head_index(model, b, Sj)
    logits = bf.get("vcr.logits", (2 * b, 8), torch.float32)  # CE reads columns [0, 4)
    saved = []
    for t, (sc, site_in, site_hid) in enumerate(_TOWERS):
        x = bf.get(f"vcr.{t}.x", (4 * b, H), torch.bfloat16)
        ops.gather_rows(y.reshape(B * Sj, H), idx[t], x)
        xd = x
        if p > 0.0:  # :87 / :106
            xd = bf.get(f"vcr.{t}.xd", (4 * b, H), torch.bfloat16)
            ops.dropout_apply(x, xd, p, seed, site_in)
        # dense(H/2) + erf-GeLU (:88-94), dropout (:95): h <- drop(gelu(pre)); gp <- gelu'(pre) for the backward
        h = bf.get(f"vcr.{t}.h", (4 * b, H2), torch.bfloat16)
        gp = bf.get(f"vcr.{t}.gp", (4 * b, H2), torch.bfloat16)
        ops.gemm(xd, store.W(f"{sc}/classifier_mlp0/kernel"), b_mn_major=True, bias=store.P(f"{sc}/classifier_mlp0/bias"),
                 gelu=True, out_pre=gp, gelu_grad_out=True, out=h, dropout_p=p, dropout_seed=seed, dropout_site=site_hid)
        # dense(1) (:96-102) with N = 1 padded to 8: z[4q + c, 0] is the logit of question q, candidate c
        z = bf.get(f"vcr.{t}.z", (4 * b, 8), torch.float32)
        ops.gemm(h, store.W(f"{sc}/classifier_mlp1/kernel"), b_mn_major=True, bias=store.P(f"{sc}/classifier_mlp1/bias"), out=z)
        # concat + reshape (:124-125): logits[2q + t, c] = sum_k z[q, k] E[k, c] over z viewed as [b, 32] -- an exact
        # strided copy of column 0 (one product by 1.0, the rest by 0.0)
        ops.small_gemm(z, 32, 1, sel, 1, 4, logits[t::2], b, 4, 32)
        saved.append((xd, h, gp))
    model._vcr_cls = (logits, saved, p, seed)  # what cls_head_backward reads
    return logits[:, :4]


def cls_head_backward(model, store, target: torch.Tensor) -> torch.Tensor:
    """Gradient of cls_loss(cls_head(...), target) (:133-143 over :77-127).  ACCUMULATES the towers' parameter gradients into
    store.g and returns the bf16 d_hidden_state [B*(P+L), H] for model.backward(d_hidden_state=...): non-zero only at row P of
    each sequence."""
    if getattr(model, "_vcr_cls", None) is None:
        raise RuntimeError("cls_head_backward needs cls_head(model, store, ...) first")
    logits, saved, p, seed = model._vcr_cls
    y = model.encoder_info["hidden_state"]
    B, Sj, H = y.shape
    b, H2 = logits.shape[0] // 2, H // 2
    bf = model._bufs
    idx, sel = _head_index(model, b, Sj)
    ce = _SoftmaxCE(bf, "vcr", logits, target.to(torch.int32).contiguous(), 4)  # coeff = 1 / img_batch_size (:142)
    dlog = ce.backward(bf.get("vcr.dlogits", (2 * b, 8), torch.float32))
    d_hidden = bf.get("vcr.d_hidden", (B * Sj, H), torch.bfloat16, zero=True)
    for t, ((sc, site_in, site_hid), (x, h, gp)) in enumerate(zip(_TOWERS, saved)):
        # dz[4q + c, 0] = dlogits[2q + t, c], columns 1..7 zero: dz viewed as [b, 32] = dlogits[t::2, :4] E^T
        dz = bf.get(f"vcr.{t}.dz", (4 * b, 8), torch.float32)
        ops.small_gemm(dlog[t::2], 16, 1, sel, 4, 1, dz.view(b, 32), b, 32, 4)
        ops.bias_grad(dz, store.G(f"{sc}/classifier_mlp1/bias"), rows=4 * b, N=8)
        dzb = bf.get(f"vcr.{t}.dzb", (4 * b, 8), torch.bfloat16)
        ops.cast_f32_to_bf16(dz, dzb)
        ops.gemm(h, dzb, a_mn_major=True, b_mn_major=True, out=store.G(f"{sc}/classifier_mlp1/kernel"), atomic=True,
                 M=H2, N=8, K=4 * b)
        # d pre = (dz W1^T) * keep/(1-p) * gelu'(pre): the hidden dropout and the GeLU backward in the dgrad epilogue
        dpre = bf.get(f"vcr.{t}.dpre", (4 * b, H2), torch.bfloat16)
        ops.gemm(dzb, store.W(f"{sc}/classifier_mlp1/kernel"), out=dpre, mul_aux=gp, dropout_p=p, dropout_seed=seed,
                 dropout_site=site_hid, M=4 * b, N=H2, K=8)
        ops.bias_grad(dpre, store.G(f"{sc}/classifier_mlp0/bias"), rows=4 * b, N=H2)
        ops.gemm(x, dpre, a_mn_major=True, b_mn_major=True, out=store.G(f"{sc}/classifier_mlp0/kernel"), atomic=True,
                 M=H, N=H2, K=4 * b)
        # d first-token = (dpre W0^T) * keep/(1-p): the input dropout in the dgrad epilogue
        dx = bf.get(f"vcr.{t}.dx", (4 * b, H), torch.float32)
        ops.gemm(dpre, store.W(f"{sc}/classifier_mlp0/kernel"), out=dx, dropout_p=p, dropout_seed=seed, dropout_site=site_in,
                 M=4 * b, N=H, K=H2)
        ops.scatter_add_rows(dx, idx[t], d_hidden)
    return d_hidden


def vcr_model_fn_builder(config, *, store=None, dist=None, seed: int = 0, device="cuda", vit_grad_buckets: int = 4):
    """downstream/vcr/modeling.py:23-219 with the call shape of train.model_fn_builder.  Returns model_fn(features, labels, mode):
      * features: 'images' [2b, h, w, 3] (or [h, w, 3, 2b] with transpose_input), 'lm_input' [2b*4, L] in training and
        [b', 4, L] in eval; labels: {'lm_targets': [2b]} (or features['lm_targets']), images ordered
        [q0 answer, q0 rationale, q1 answer, ...] in training (dataloader_joint.py:163-189,257-271);
      * mode "train": MerlotModel(is_training=True, mask_input=False), cls_head + cls_loss; metrics loss / accuracy /
        learning_rate; train_op = the head backward, model.backward(d_hidden_state=...), gradient mean over replicas, AdamW;
      * mode "eval": MerlotModel(is_training=False), cls_head_val on the `{downstream.mode}_cls` tower; metrics loss, accuracy,
        logits and predictions, no train_op;
      * mode "predict": as "eval" without lm_targets, loss or accuracy (metrics logits and predictions), for unlabelled
        records: the CE kernel is not run.
    `store=None` builds ParamStore(task="vcr"), applies the reference initialisers and then `model.init_checkpoint` if set
    (restore by name, model/modeling.py:724-740: the towers keep their initial values; a missing checkpoint raises).  The
    dropout seed of a step follows the pretraining rule: seed + step * world + rank.

    Gradient accumulation: model_fn([f_0, ..., f_{A-1}]) in training, A feature dicts of one micro-batch each, returns a
    step whose train_op runs forward, head and backward of every micro-batch in turn (the VCR loss has no term across
    questions), with dropout seed seed + step*world*A + rank*A + j, then one AdamW step over the mean of the world * A
    micro-batch gradients.  Its metrics, the means over the rank's micro-batches, are complete after train_op()."""
    from .config import replica_seed
    from .optimization import build_optimizer_from_config
    from .params import ParamStore
    from .train import StepSpec, accumulate_mean, backward_and_apply, backward_micro_batch
    m_cfg = config.model
    if store is None:
        store = ParamStore(m_cfg, device=device, optimizer_cfg=config.optimizer, task="vcr")
        store.init_reference(seed=0)
        ckpt = m_cfg.get("init_checkpoint")
        if ckpt:
            missing = store.load_checkpoint(ckpt)
            print(f"init_checkpoint {ckpt}: {len(missing)} variables not in the checkpoint keep their initial values: "
                  f"{', '.join(missing)}", flush=True)
    elif store.task != "vcr":
        raise ValueError(f"the VCR step trains a ParamStore(task='vcr'), got task={store.task!r}")
    optimizer, _ = build_optimizer_from_config(loss=None, optimizer_config=config.optimizer, device_config=config.device,
                                               store=store)
    eval_mode = config.downstream.get("mode", "answer")

    def accumulated_step(micro, labels):
        A = len(micro)
        world, rank = (dist.world, dist.rank) if dist is not None else (1, 0)
        p = float(m_cfg.get("hidden_dropout_prob", 0.0) or 0.0)
        metrics = {"learning_rate": optimizer.current_lr()}
        loss_parts = []

        def train_op():
            acc = {}
            for j, f in enumerate(micro):
                imgs = f["images"]
                if m_cfg.get("transpose_input", False) and imgs.shape[-1] != 3:
                    imgs = imgs.permute(3, 0, 1, 2).contiguous()
                target = (labels[j] if labels else f)["lm_targets"]
                step_seed = replica_seed(seed, store.global_step, world, A, rank, j)
                model = MerlotModel(config=m_cfg, is_training=True, use_tpu=config.device.get("use_tpu", False), image=imgs,
                                    input_ids=f["lm_input"], mask_input=False, params=store, dropout_seed=step_seed, dist=dist,
                                    log_attention_probs=False)
                logits = cls_head(model, store, dropout=(p, step_seed))
                loss, accuracy = cls_loss(logits, target)
                accumulate_mean(model._bufs, acc, {"loss": loss, "accuracy": accuracy}, j, A)
                d_hidden = cls_head_backward(model, store, target)
                if j + 1 < A:
                    norm = backward_micro_batch(model, optimizer, d_hidden_state=d_hidden)
                else:
                    norm = backward_and_apply(model, optimizer, dist, metrics=metrics, vit_grad_buckets=vit_grad_buckets,
                                              d_hidden_state=d_hidden, accum=A)
                if norm is not None and A > 1:
                    accumulate_mean(model._bufs, acc, {"gradnorms/_overall": norm}, j, A)
            metrics.update(acc)
            loss_parts[:] = [acc["loss"]]

        return StepSpec(None, loss_parts, metrics, train_op)

    def model_fn(features, labels=None, mode="train", params=None):
        if isinstance(features, (list, tuple)):
            if mode != "train":
                raise ValueError("a list of micro-batches is a training step (mode 'train')")
            return accumulated_step(list(features), labels)
        is_training = mode == "train"
        imgs, ids = features["images"], features["lm_input"]
        target = None if mode == "predict" else (labels or features)["lm_targets"]
        if is_training and m_cfg.get("transpose_input", False) and imgs.shape[-1] != 3:
            imgs = imgs.permute(3, 0, 1, 2).contiguous()  # :35-37
        if not is_training:  # [b, 4, L] -> [4b, L] (:39-44)
            ids = ids.reshape(-1, ids.shape[-1])
        world, rank = (dist.world, dist.rank) if dist is not None else (1, 0)
        step_seed = seed + store.global_step * world + rank
        model = MerlotModel(config=m_cfg, is_training=is_training, use_tpu=config.device.get("use_tpu", False), image=imgs,
                            input_ids=ids, mask_input=False, params=store, dropout_seed=step_seed, dist=dist,
                            log_attention_probs=False)
        if not is_training:
            logits = cls_head_val(model, head_from_store(store, eval_mode), eval_mode)
            metrics = {"logits": logits, "predictions": logits.argmax(-1)}
            if target is None:
                return StepSpec(model, (), metrics, None)
            loss, acc = cls_loss(logits, target)
            metrics.update(loss=loss, accuracy=acc)
            return StepSpec(model, (loss,), metrics, None)
        p = float(m_cfg.get("hidden_dropout_prob", 0.0) or 0.0)
        logits = cls_head(model, store, dropout=(p, step_seed))
        loss, acc = cls_loss(logits, target)
        metrics = {"loss": loss, "accuracy": acc, "learning_rate": optimizer.current_lr()}

        def train_op():
            d_hidden = cls_head_backward(model, store, target)
            backward_and_apply(model, optimizer, dist, metrics=metrics, vit_grad_buckets=vit_grad_buckets, d_hidden_state=d_hidden)

        return StepSpec(model, (loss,), metrics, train_op)

    model_fn.store = store
    model_fn.optimizer = optimizer
    return model_fn
