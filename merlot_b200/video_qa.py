"""Open-ended video QA fine-tuning (downstream.task: video_qa): F = model.num_imgs frames and one question text per
example, a softmax over a fixed vocabulary of A = downstream.num_answers answers (MSRVTT-QA, TGIF-FrameQA, ActivityNet-QA).

The reference describes this adaptation without code for it; like video_mc.py it is VCR's training head
(downstream/vcr/modeling.py) with one tower, here over A answer classes instead of candidate texts:
  * `qa_head` / `qa_loss` / `qa_head_backward`: the first language row (P * F) of every sequence -> dropout -> dense(H/2)
    + gelu -> dropout -> dense(A) -> logits [b, A] -> softmax cross entropy over the A answers, on the `qa_cls` tower of a
    ParamStore(task="video_qa").  The output layer is stored as A8 = ceil(A/8)*8 columns whose padding stays zero, so the
    logits are the first A columns of the tower's fp32 [b, A8] output and the CE kernel reads them with row stride A8;
  * `video_qa_model_fn_builder`: the fine-tuning step (train), the validation forward (eval) and the scoring forward
    (predict), with the call shape of video_mc.video_mc_model_fn_builder.
A label of -1 marks a question whose answer is not in the vocabulary (out of vocabulary, OOV).  The CE kernel reads the
label's logit unchecked, so such a row gets the stand-in label 0 and weight 0: it adds nothing to the loss or to any
gradient, and it counts as answered wrong.  The training input skips OOV questions; evaluation keeps them.
All arithmetic of the head runs in libmerlot_b200.so (video_mc.tower_forward / tower_backward, the CE kernel, the weighted
mean); no kernel is this module's own.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import ops
from .modeling import _SITE_QA_HID, _SITE_QA_IN, MerlotModel
from .params import VIDEO_QA_TOWER, padded_answers
from .video_mc import tower_backward, tower_forward

TOWER = VIDEO_QA_TOWER
MIN_ANSWERS = 2


def check_config(model_cfg, downstream_cfg) -> Tuple[int, int]:
    """(F, A) = (model.num_imgs, downstream.num_answers) of a video_qa config; ValueError for F < 1, model.num_texts other
    than 1, or num_answers missing or < 2."""
    F = int(model_cfg.get("num_imgs", 1))
    if F < 1:
        raise ValueError(f"video_qa: model.num_imgs (frames per question) must be >= 1, got {F}")
    T = model_cfg.get("num_texts")
    if T is not None and int(T) != 1:
        raise ValueError(f"video_qa: model.num_texts must be 1 (one question text per example), got {T}")
    A = downstream_cfg.get("num_answers")
    if A is None:
        raise ValueError("video_qa: downstream.num_answers (the size of the answer vocabulary) is missing, got None")
    if int(A) < MIN_ANSWERS:
        raise ValueError(f"video_qa: downstream.num_answers must be >= {MIN_ANSWERS}, got {A}")
    return F, int(A)


def _head_index(model, b: int, Sj: int):
    """int32 [b]: row P * F of every sequence of Sj rows, the first language row (START), which the tower reads."""
    bf, dev = model._bufs, model.store.device
    P = model.encoder_pieces[1]["start"]  # P * num_imgs: the language piece follows every frame's viz tokens
    key = ("_qa_idx", b, Sj, P)
    if key not in bf.d:
        bf.d[key] = (torch.arange(b, device=dev) * Sj + P).to(torch.int32).contiguous()
    return bf.d[key]


def qa_head(model, store, dropout=(0.0, 0)) -> torch.Tensor:
    """The tower on model.encoder_info['hidden_state'] -> fp32 logits [b, A]: a view of the first A columns of a fresh
    [b, A8] buffer.  dropout = (p, seed): hidden_dropout_prob and the step's dropout seed, at sites _SITE_QA_IN (the
    tower's input) and _SITE_QA_HID (its hidden layer); p = 0 in evaluation."""
    y = model.encoder_info["hidden_state"]  # bf16 [b, P*F + L, H]
    if model.num_texts != 1 or store.num_answers is None:
        raise ValueError(f"the video_qa head reads one text per question from a ParamStore(task='video_qa'): num_texts "
                         f"{model.num_texts}, store task {store.task!r}")
    b, Sj, _ = y.shape
    A = store.num_answers
    p, seed = float(dropout[0]), int(dropout[1])
    idx = _head_index(model, b, Sj)
    logits = torch.empty((b, padded_answers(A)), dtype=torch.float32, device=y.device)
    xd, h, gp = tower_forward(model._bufs, store, TOWER, y, idx, logits, (p, seed, _SITE_QA_IN, _SITE_QA_HID), "qa")
    model._qa = {"logits": logits, "x": xd, "h": h, "gp": gp, "p": p, "seed": seed, "A": A}  # what the backward reads
    return logits[:, :A]


def qa_loss(model, target: torch.Tensor):
    """Softmax cross entropy over the A answers of the logits qa_head computed last.  `target` int [b] holds answers in
    [0, A) or -1 (OOV).  Returns (loss, accuracy, counts), 0-d fp32 CUDA tensors: loss = the mean over the in-vocabulary
    rows (weighted_loss's sum w + 1e-5 denominator), accuracy = correct rows / b with OOV rows wrong, and counts = {loss_sum:
    the CE summed over the in-vocabulary rows, in_vocab: their number, correct: the rows answered right}."""
    st = getattr(model, "_qa", None)
    if st is None:
        raise RuntimeError("qa_loss needs qa_head(model, store, ...) first")
    logits, A = st["logits"], st["A"]
    b, dev = logits.shape[0], logits.device
    tgt = target.to(torch.int32)
    weight = (tgt >= 0).to(torch.float32).contiguous()
    safe = tgt.clamp(min=0).contiguous()  # the stand-in label of an OOV row, whose weight is 0
    per, lse, corr, coeff = (torch.empty(b, dtype=torch.float32, device=dev) for _ in range(4))
    out2 = torch.empty(2, dtype=torch.float32, device=dev)
    acc2 = torch.empty(2, dtype=torch.float32, device=dev)
    ops.softmax_ce_fwd(logits, safe, A, per, lse, corr)
    ops.weighted_loss(per, corr, weight, None, 1, 1.0, out2, coeff)  # coeff = w / (sum w + 1e-5): OOV rows get 0
    ops.weighted_loss(corr, None, weight, None, 0, 1.0, acc2, None)  # sum(correct * w) / b
    st.update(target=safe, lse=lse, coeff=coeff)
    counts = {"loss_sum": (per * weight).sum(), "in_vocab": weight.sum(), "correct": (corr * weight).sum()}
    return out2[0], acc2[0], counts


def qa_head_backward(model, store) -> torch.Tensor:
    """Gradient of qa_loss(qa_head(...)).  ACCUMULATES the tower's parameter gradients into store.g and returns the bf16
    d_hidden_state [b*(P*F+L), H] for model.backward(d_hidden_state=...): non-zero only at row P*F of each sequence."""
    st = getattr(model, "_qa", None)
    if st is None or "lse" not in st:
        raise RuntimeError("qa_head_backward needs qa_head(model, store, ...) and qa_loss(model, target) first")
    logits, x, h, gp, p, seed, A = (st[k] for k in ("logits", "x", "h", "gp", "p", "seed", "A"))
    y = model.encoder_info["hidden_state"]
    b, Sj, _ = y.shape
    bf = model._bufs
    idx = _head_index(model, b, Sj)
    # the CE kernel writes columns [0, A); the padding columns stay zero, so the padded weights get no gradient
    dlog = bf.get("qa.dlogits", tuple(logits.shape), torch.float32, zero=True)
    ops.softmax_ce_bwd(logits, st["target"], A, st["lse"], st["coeff"], dlog)
    return tower_backward(bf, store, TOWER, y, idx, dlog, x, h, gp, (p, seed, _SITE_QA_IN, _SITE_QA_HID), "qa")


def video_qa_model_fn_builder(config, *, store=None, dist=None, seed: int = 0, device="cuda", vit_grad_buckets: int = 4):
    """The video_qa step with the call shape of video_mc.video_mc_model_fn_builder.  Returns model_fn(features, labels,
    mode):
      * features: 'images' [b*F, h, w, 3] (or [h, w, 3, b*F] with transpose_input; question-major, frame-minor),
        'img_mask' [b, F] bool (absent: every slot holds a frame), 'lm_input' [b, L]; labels: {'lm_targets': [b]} (or
        features['lm_targets']) in [0, A), or -1 for an OOV answer;
      * mode "train": MerlotModel(is_training=True, mask_input=False, img_mask=...), qa_head + qa_loss; metrics loss /
        accuracy / learning_rate; train_op = the head backward, model.backward(d_hidden_state=...), gradient mean over
        replicas, AdamW;
      * mode "eval": MerlotModel(is_training=False) and the head without dropout; metrics loss (over the in-vocabulary
        questions), accuracy (over all, OOV wrong), logits [b, A], predictions, and loss_sum / in_vocab / correct (the
        counts a validator sums over batches); no train_op;
      * mode "predict": as "eval" without lm_targets, loss or accuracy: the CE kernel is not run.
    `store=None` builds ParamStore(task="video_qa", num_answers=A), applies the reference initialisers and then
    `model.init_checkpoint` if set (restore by name: a pretraining checkpoint leaves the qa_cls tower at its initial
    values).  Dropout seeds and gradient accumulation (a list of micro-batch feature dicts in "train") follow
    video_mc_model_fn_builder: seed + step*world*A + rank*A + j, one AdamW step over the mean of the world * A
    micro-batch gradients (clipped one by one with clip_norm > 0)."""
    from .config import replica_seed
    from .optimization import build_optimizer_from_config
    from .params import ParamStore
    from .train import StepSpec, accumulate_mean, backward_and_apply, backward_micro_batch
    m_cfg = config.model
    _, A = check_config(m_cfg, config.downstream)
    if store is None:
        store = ParamStore(m_cfg, device=device, optimizer_cfg=config.optimizer, task="video_qa", num_answers=A)
        store.init_reference(seed=0)
        ckpt = m_cfg.get("init_checkpoint")
        if ckpt:
            missing = store.load_checkpoint(ckpt)
            print(f"init_checkpoint {ckpt}: {len(missing)} variables not in the checkpoint keep their initial values: "
                  f"{', '.join(missing)}", flush=True)
    elif store.task != "video_qa":
        raise ValueError(f"the video_qa step trains a ParamStore(task='video_qa'), got task={store.task!r}")
    elif store.num_answers != A:
        raise ValueError(f"the ParamStore holds {store.num_answers} answers, downstream.num_answers is {A}")
    optimizer, _ = build_optimizer_from_config(loss=None, optimizer_config=config.optimizer, device_config=config.device,
                                               store=store)
    m_cfg = dict(m_cfg, num_texts=1)

    def forward(f, is_training: bool, step_seed: int):
        imgs, ids = f["images"], f["lm_input"]
        if config.model.get("transpose_input", False) and imgs.shape[-1] != 3:
            imgs = imgs.permute(3, 0, 1, 2).contiguous()
        return MerlotModel(config=m_cfg, is_training=is_training, use_tpu=config.device.get("use_tpu", False), image=imgs,
                           input_ids=ids, mask_input=False, img_mask=f.get("img_mask"), params=store, dropout_seed=step_seed,
                           dist=dist, log_attention_probs=False)

    def hidden_p():
        return float(m_cfg.get("hidden_dropout_prob", 0.0) or 0.0)

    def accumulated_step(micro, labels):
        n_micro = len(micro)
        world, rank = (dist.world, dist.rank) if dist is not None else (1, 0)
        metrics = {"learning_rate": optimizer.current_lr()}
        loss_parts = []

        def train_op():
            acc = {}
            for j, f in enumerate(micro):
                target = (labels[j] if labels else f)["lm_targets"]
                step_seed = replica_seed(seed, store.global_step, world, n_micro, rank, j)
                model = forward(f, True, step_seed)
                qa_head(model, store, dropout=(hidden_p(), step_seed))
                loss, accuracy, _ = qa_loss(model, target)
                accumulate_mean(model._bufs, acc, {"loss": loss, "accuracy": accuracy}, j, n_micro)
                d_hidden = qa_head_backward(model, store)
                if j + 1 < n_micro:
                    norm = backward_micro_batch(model, optimizer, d_hidden_state=d_hidden)
                else:
                    norm = backward_and_apply(model, optimizer, dist, metrics=metrics, vit_grad_buckets=vit_grad_buckets,
                                              d_hidden_state=d_hidden, accum=n_micro)
                if norm is not None and n_micro > 1:
                    accumulate_mean(model._bufs, acc, {"gradnorms/_overall": norm}, j, n_micro)
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
        logits = qa_head(model, store, dropout=(hidden_p() if is_training else 0.0, step_seed))
        if not is_training:
            metrics = {"logits": logits, "predictions": logits.argmax(-1)}
            if target is None:
                return StepSpec(model, (), metrics, None)
            loss, acc, counts = qa_loss(model, target)
            metrics.update(loss=loss, accuracy=acc, **counts)
            return StepSpec(model, (loss,), metrics, None)
        loss, acc, _ = qa_loss(model, target)
        metrics = {"loss": loss, "accuracy": acc, "learning_rate": optimizer.current_lr()}

        def train_op():
            d_hidden = qa_head_backward(model, store)
            backward_and_apply(model, optimizer, dist, metrics=metrics, vit_grad_buckets=vit_grad_buckets, d_hidden_state=d_hidden)

        return StepSpec(model, (loss,), metrics, train_op)

    model_fn.store = store
    model_fn.optimizer = optimizer
    return model_fn
