"""Multiple-choice video QA fine-tuning (downstream.task: video_mc): F = model.num_imgs frames and C = model.num_texts
candidate texts per question, one softmax over the candidates.

The reference describes this adaptation (a MerlotModel over several frames, an output layer, fine-tuning) without code for
it; its worked example is VCR (downstream/vcr/modeling.py, merlot_b200/vcr.py).  This module is VCR's training head with one
tower instead of two and C candidates instead of 4:
  * `mc_head` / `mc_loss` / `mc_head_backward`: the first language row (P * F) of every sequence -> dropout -> dense(H/2)
    + gelu -> dropout -> dense(1) -> logits [b, C] -> softmax cross entropy over the C candidates, on the `mc_cls` tower of a
    ParamStore(task="video_mc"); the backward writes the tower's gradients into store.g and returns the gradient that
    enters the model through MerlotModel.backward(d_hidden_state=...);
  * `video_mc_model_fn_builder`: the fine-tuning step (train), the validation forward (eval) and the scoring forward
    (predict), with the call shape of vcr.vcr_model_fn_builder;
  * `tower_forward` / `tower_backward`: the tower's kernel sequence on given rows of the hidden state, which the open-ended
    video QA head (video_qa.py) runs as well.
All arithmetic runs in libmerlot_b200.so: the row gather / scatter, dropout, the K1 GEMM with its fused epilogues, the
strided fp32 small GEMM, the CE kernel and the bias-gradient kernel -- the kernels of VCR's head.  C <= 8 because the tower's
dense(1) output is padded to 8 columns, and the logits of a question are a row of those 8 columns.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import ops
from .modeling import _SITE_MC_HID, _SITE_MC_IN, MerlotModel
from .params import VIDEO_MC_TOWERS

TOWER = VIDEO_MC_TOWERS[0]
MIN_CHOICES, MAX_CHOICES = 2, 8  # a softmax needs two candidates; the logits row holds eight


def check_config(model_cfg) -> Tuple[int, int]:
    """(F, C) = (model.num_imgs, model.num_texts) of a video_mc model config; ValueError outside F >= 1, 2 <= C <= 8."""
    F, C = int(model_cfg.get("num_imgs", 1)), int(model_cfg.get("num_texts", 1))
    if F < 1:
        raise ValueError(f"video_mc: model.num_imgs (frames per question) must be >= 1, got {F}")
    if not MIN_CHOICES <= C <= MAX_CHOICES:
        raise ValueError(f"video_mc: model.num_texts (candidate answers per question) must be in [{MIN_CHOICES}, "
                         f"{MAX_CHOICES}], got {C}")
    return F, C


def _head_index(model, b: int, C: int, Sj: int):
    """int32 [C*b] rows of the joint hidden state the tower reads (row P * F, the first language row, of every sequence of
    Sj rows; question-major, row q*C + c = candidate c of question q), and the constant E fp32 [8C, C], E[8c, c] = 1, that
    moves logits between the tower's padded dense(1) output [C*b, 8] and the logits [b, 8] (see mc_head)."""
    bf, dev = model._bufs, model.store.device
    P = model.encoder_pieces[1]["start"]  # P * num_imgs: the language piece follows every frame's viz tokens
    key = ("_mc_idx", b, C, Sj, P)
    if key not in bf.d:
        idx = (torch.arange(b * C, device=dev) * Sj + P).to(torch.int32).contiguous()
        sel = torch.zeros((8 * C, C), dtype=torch.float32, device=dev)
        sel[torch.arange(C) * 8, torch.arange(C)] = 1.0
        bf.d[key] = (idx, sel)
    return bf.d[key]


def mc_head(model, store, dropout=(0.0, 0)) -> torch.Tensor:
    """The tower on model.encoder_info['hidden_state'] -> fp32 logits [b, C] (a view of a fresh [b, 8] buffer whose first C
    columns are the logits).  dropout = (p, seed): hidden_dropout_prob and the step's dropout seed, at sites _SITE_MC_IN
    (the tower's input) and _SITE_MC_HID (its hidden layer); p = 0 in evaluation."""
    y = model.encoder_info["hidden_state"]  # bf16 [B, P*F + L, H]
    B, Sj, H = y.shape
    C = model.num_texts
    if not MIN_CHOICES <= C <= MAX_CHOICES or B % C != 0:
        raise ValueError(f"the video_mc head scores {MIN_CHOICES}..{MAX_CHOICES} candidates per question: batch {B}, "
                         f"num_texts {C}")
    b = B // C
    p, seed = float(dropout[0]), int(dropout[1])
    bf = model._bufs
    idx, sel = _head_index(model, b, C, Sj)
    # dense(1) with N = 1 padded to 8: z[q*C + c, 0] is the logit of question q, candidate c
    z = bf.get("mc.z", (B, 8), torch.float32)
    xd, h, gp = tower_forward(bf, store, TOWER, y, idx, z, (p, seed, _SITE_MC_IN, _SITE_MC_HID), "mc")
    # logits[q, c] = sum_k z[q, k] E[k, c] over z viewed as [b, 8C]: an exact strided copy of column 0
    logits = torch.empty((b, 8), dtype=torch.float32, device=y.device)
    ops.small_gemm(z, 8 * C, 1, sel, 1, C, logits, b, C, 8 * C)
    model._mc = {"logits": logits, "x": xd, "h": h, "gp": gp, "p": p, "seed": seed, "C": C}  # what the backward reads
    return logits[:, :C]


def mc_loss(model, target: torch.Tensor):
    """Mean softmax cross entropy over the C candidates of the logits mc_head computed last, and the accuracy (0-d fp32
    CUDA tensors).  `target` int [b] must hold labels in [0, C): the CE kernel reads the label's logit unchecked, so the
    input pipeline checks labels on the host."""
    st = getattr(model, "_mc", None)
    if st is None:
        raise RuntimeError("mc_loss needs mc_head(model, store, ...) first")
    logits, C = st["logits"], st["C"]
    b, dev = logits.shape[0], logits.device
    tgt = target.to(torch.int32).contiguous()
    per, lse, corr, coeff = (torch.empty(b, dtype=torch.float32, device=dev) for _ in range(4))
    out2 = torch.empty(2, dtype=torch.float32, device=dev)
    ops.softmax_ce_fwd(logits, tgt, C, per, lse, corr)
    ops.weighted_loss(per, corr, None, None, 0, 1.0, out2, coeff)  # coeff = 1 / b
    st.update(target=tgt, lse=lse, coeff=coeff)
    return out2[0], out2[1]


def mc_head_backward(model, store) -> torch.Tensor:
    """Gradient of mc_loss(mc_head(...)).  ACCUMULATES the tower's parameter gradients into store.g and returns the bf16
    d_hidden_state [B*(P*F+L), H] for model.backward(d_hidden_state=...): non-zero only at row P*F of each sequence."""
    st = getattr(model, "_mc", None)
    if st is None or "lse" not in st:
        raise RuntimeError("mc_head_backward needs mc_head(model, store, ...) and mc_loss(model, target) first")
    logits, x, h, gp, p, seed, C = (st[k] for k in ("logits", "x", "h", "gp", "p", "seed", "C"))
    y = model.encoder_info["hidden_state"]
    B = y.shape[0]
    b = B // C
    bf = model._bufs
    idx, sel = _head_index(model, b, C, y.shape[1])
    dlog = bf.get("mc.dlogits", (b, 8), torch.float32)
    ops.softmax_ce_bwd(logits, st["target"], C, st["lse"], st["coeff"], dlog)
    # dz[q*C + c, 0] = dlogits[q, c], columns 1..7 zero: dz viewed as [b, 8C] = dlogits[:, :C] E^T
    dz = bf.get("mc.dz", (B, 8), torch.float32)
    ops.small_gemm(dlog, 8, 1, sel, C, 1, dz.view(b, 8 * C), b, 8 * C, C)
    return tower_backward(bf, store, TOWER, y, idx, dz, x, h, gp, (p, seed, _SITE_MC_IN, _SITE_MC_HID), "mc")


def tower_forward(bf, store, tower: str, y, idx, z, dropout, key: str):
    """The classifier tower `tower` of a ParamStore on rows `idx` (int32 [n]) of the bf16 hidden state y [B, Sj, H]:
    gather -> dropout -> dense(H/2) + erf-GeLU -> dropout -> dense(N) into the fp32 z [n, N] (N = the stored columns of
    classifier_mlp1, a multiple of 8).  dropout = (p, seed, input site, hidden site); buffers are named `key`.*.  Returns
    what tower_backward reads: the tower's (dropped) input, its hidden layer and gelu'(pre)."""
    B, Sj, H = y.shape
    n, H2 = idx.numel(), H // 2
    p, seed, site_in, site_hid = dropout
    x = bf.get(f"{key}.x", (n, H), torch.bfloat16)
    ops.gather_rows(y.reshape(B * Sj, H), idx, x)
    xd = x
    if p > 0.0:
        xd = bf.get(f"{key}.xd", (n, H), torch.bfloat16)
        ops.dropout_apply(x, xd, p, seed, site_in)
    # dense(H/2) + erf-GeLU, dropout: h <- drop(gelu(pre)); gp <- gelu'(pre) for the backward
    h = bf.get(f"{key}.h", (n, H2), torch.bfloat16)
    gp = bf.get(f"{key}.gp", (n, H2), torch.bfloat16)
    ops.gemm(xd, store.W(f"{tower}/classifier_mlp0/kernel"), b_mn_major=True, bias=store.P(f"{tower}/classifier_mlp0/bias"),
             gelu=True, out_pre=gp, gelu_grad_out=True, out=h, dropout_p=p, dropout_seed=seed, dropout_site=site_hid)
    ops.gemm(h, store.W(f"{tower}/classifier_mlp1/kernel"), b_mn_major=True, bias=store.P(f"{tower}/classifier_mlp1/bias"), out=z)
    return xd, h, gp


def tower_backward(bf, store, tower: str, y, idx, dz, x, h, gp, dropout, key: str):
    """Backward of tower_forward from dz fp32 [n, N], the gradient of its output z.  ACCUMULATES the tower's parameter
    gradients into store.g and returns the bf16 d_hidden_state [B*Sj, H], non-zero only at the rows `idx`."""
    B, Sj, H = y.shape
    n, N = dz.shape
    H2 = H // 2
    p, seed, site_in, site_hid = dropout
    ops.bias_grad(dz, store.G(f"{tower}/classifier_mlp1/bias"), rows=n, N=N)
    dzb = bf.get(f"{key}.dzb", (n, N), torch.bfloat16)
    ops.cast_f32_to_bf16(dz, dzb)
    ops.gemm(h, dzb, a_mn_major=True, b_mn_major=True, out=store.G(f"{tower}/classifier_mlp1/kernel"), atomic=True,
             M=H2, N=N, K=n)
    # d pre = (dz W1^T) * keep/(1-p) * gelu'(pre): the hidden dropout and the GeLU backward in the dgrad epilogue
    dpre = bf.get(f"{key}.dpre", (n, H2), torch.bfloat16)
    ops.gemm(dzb, store.W(f"{tower}/classifier_mlp1/kernel"), out=dpre, mul_aux=gp, dropout_p=p, dropout_seed=seed,
             dropout_site=site_hid, M=n, N=H2, K=N)
    ops.bias_grad(dpre, store.G(f"{tower}/classifier_mlp0/bias"), rows=n, N=H2)
    ops.gemm(x, dpre, a_mn_major=True, b_mn_major=True, out=store.G(f"{tower}/classifier_mlp0/kernel"), atomic=True,
             M=H, N=H2, K=n)
    # d first-token = (dpre W0^T) * keep/(1-p): the input dropout in the dgrad epilogue
    dx = bf.get(f"{key}.dx", (n, H), torch.float32)
    ops.gemm(dpre, store.W(f"{tower}/classifier_mlp0/kernel"), out=dx, dropout_p=p, dropout_seed=seed, dropout_site=site_in,
             M=n, N=H, K=H2)
    d_hidden = bf.get(f"{key}.d_hidden", (B * Sj, H), torch.bfloat16, zero=True)
    ops.scatter_add_rows(dx, idx, d_hidden)
    return d_hidden


def video_mc_model_fn_builder(config, *, store=None, dist=None, seed: int = 0, device="cuda", vit_grad_buckets: int = 4):
    """The video_mc step with the call shape of vcr.vcr_model_fn_builder.  Returns model_fn(features, labels, mode):
      * features: 'images' [b*F, h, w, 3] (or [h, w, 3, b*F] with transpose_input; question-major, frame-minor),
        'img_mask' [b, F] bool (False: the frame slot is empty; absent: every slot holds a frame), 'lm_input' [b*C, L] or
        [b, C, L] (question-major); labels: {'lm_targets': [b]} (or features['lm_targets']) in [0, C);
      * mode "train": MerlotModel(is_training=True, mask_input=False, img_mask=...), mc_head + mc_loss; metrics loss /
        accuracy / learning_rate; train_op = the head backward, model.backward(d_hidden_state=...), gradient mean over
        replicas, AdamW;
      * mode "eval": MerlotModel(is_training=False) and the head without dropout; metrics loss, accuracy, logits [b, C] and
        predictions, no train_op;
      * mode "predict": as "eval" without lm_targets, loss or accuracy, for unlabelled records: the CE kernel is not run.
    `store=None` builds ParamStore(task="video_mc"), applies the reference initialisers and then `model.init_checkpoint` if
    set (restore by name: a pretraining checkpoint leaves the mc_cls tower at its initial values; a missing checkpoint
    raises).  The dropout seed of a step follows the pretraining rule: seed + step * world + rank.

    Gradient accumulation: model_fn([f_0, ..., f_{A-1}]) in training, A feature dicts of one micro-batch each, returns a
    step whose train_op runs forward, head and backward of every micro-batch in turn (the loss has no term across
    questions), with dropout seed seed + step*world*A + rank*A + j, then one AdamW step over the mean of the world * A
    micro-batch gradients (clipped one by one with clip_norm > 0).  Its metrics, the means over the rank's micro-batches,
    are complete after train_op()."""
    from .config import replica_seed
    from .optimization import build_optimizer_from_config
    from .params import ParamStore
    from .train import StepSpec, accumulate_mean, backward_and_apply, backward_micro_batch
    m_cfg = config.model
    check_config(m_cfg)
    if store is None:
        store = ParamStore(m_cfg, device=device, optimizer_cfg=config.optimizer, task="video_mc")
        store.init_reference(seed=0)
        ckpt = m_cfg.get("init_checkpoint")
        if ckpt:
            missing = store.load_checkpoint(ckpt)
            print(f"init_checkpoint {ckpt}: {len(missing)} variables not in the checkpoint keep their initial values: "
                  f"{', '.join(missing)}", flush=True)
    elif store.task != "video_mc":
        raise ValueError(f"the video_mc step trains a ParamStore(task='video_mc'), got task={store.task!r}")
    optimizer, _ = build_optimizer_from_config(loss=None, optimizer_config=config.optimizer, device_config=config.device,
                                               store=store)

    def forward(f, is_training: bool, step_seed: int):
        imgs, ids = f["images"], f["lm_input"]
        if m_cfg.get("transpose_input", False) and imgs.shape[-1] != 3:
            imgs = imgs.permute(3, 0, 1, 2).contiguous()
        ids = ids.reshape(-1, ids.shape[-1])  # [b, C, L] -> [b*C, L]
        return MerlotModel(config=m_cfg, is_training=is_training, use_tpu=config.device.get("use_tpu", False), image=imgs,
                           input_ids=ids, mask_input=False, img_mask=f.get("img_mask"), params=store, dropout_seed=step_seed,
                           dist=dist, log_attention_probs=False)

    def hidden_p():
        return float(m_cfg.get("hidden_dropout_prob", 0.0) or 0.0)

    def accumulated_step(micro, labels):
        A = len(micro)
        world, rank = (dist.world, dist.rank) if dist is not None else (1, 0)
        metrics = {"learning_rate": optimizer.current_lr()}
        loss_parts = []

        def train_op():
            acc = {}
            for j, f in enumerate(micro):
                target = (labels[j] if labels else f)["lm_targets"]
                step_seed = replica_seed(seed, store.global_step, world, A, rank, j)
                model = forward(f, True, step_seed)
                mc_head(model, store, dropout=(hidden_p(), step_seed))
                loss, accuracy = mc_loss(model, target)
                accumulate_mean(model._bufs, acc, {"loss": loss, "accuracy": accuracy}, j, A)
                d_hidden = mc_head_backward(model, store)
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
        if mode not in ("train", "eval", "predict"):
            raise ValueError(f"mode must be 'train', 'eval' or 'predict', got {mode!r}")
        if isinstance(features, (list, tuple)):
            if mode != "train":
                raise ValueError("a list of micro-batches is a training step (mode 'train')")
            return accumulated_step(list(features), labels)
        is_training = mode == "train"
        target = None if mode == "predict" else (labels or features)["lm_targets"]
        world, rank = (dist.world, dist.rank) if dist is not None else (1, 0)
        step_seed = seed + store.global_step * world + rank
        model = forward(features, is_training, step_seed)
        logits = mc_head(model, store, dropout=(hidden_p() if is_training else 0.0, step_seed))
        if not is_training:
            metrics = {"logits": logits, "predictions": logits.argmax(-1)}
            if target is None:
                return StepSpec(model, (), metrics, None)
            loss, acc = mc_loss(model, target)
            metrics.update(loss=loss, accuracy=acc)
            return StepSpec(model, (loss,), metrics, None)
        loss, acc = mc_loss(model, target)
        metrics = {"loss": loss, "accuracy": acc, "learning_rate": optimizer.current_lr()}

        def train_op():
            d_hidden = mc_head_backward(model, store)
            backward_and_apply(model, optimizer, dist, metrics=metrics, vit_grad_buckets=vit_grad_buckets, d_hidden_state=d_hidden)

        return StepSpec(model, (loss,), metrics, train_op)

    model_fn.store = store
    model_fn.optimizer = optimizer
    return model_fn
