"""Fill-in-the-blank video QA fine-tuning (downstream.task: video_fib): F = model.num_imgs frames and one sentence with one
word blanked out per example; the model names the word, one of A answers of a fixed vocabulary (LSMDC-FiB).

The reference ships no code for this form.  It is the MLM objective of pretraining (model/modeling.py mask_loss, :528-551)
restricted to an answer vocabulary, so the head reuses the pretrained MLM head:
  * the blank is one MASK token (id 1) in the text; the head reads the joint encoder's hidden state at that row, row
    P * F + (the MASK's position in lm_input).  The encoder runs with mask_input=False, so the MASK is only an input id,
    one per blank whatever the answer's length;
  * `fib_head` / `fib_loss` / `fib_head_backward`: that row -> lm_head/projection dense(H) + gelu -> lm_head/LayerNorm
    (with model.do_projection, exactly as MerlotModel._lm_head runs them; no dropout, as the reference's lm_head has none)
    -> the fib_cls/answers dense(A) -> logits [b, A] -> softmax cross entropy over the A answers.  The answer layer is
    stored as A8 = ceil(A/8)*8 columns whose padding stays zero, as video_qa's output layer;
  * `init_answer_layer`: the answer layer's initial value.  Column a is the mean of the word-embedding rows of answer a's
    tokens and bias[a] the mean of lm_head/output_bias at them (params.derive_fib_answers), so for a one-token answer the
    logit is that token's MLM logit: a pretraining checkpoint answers zero-shot, and fine-tuning starts from a working head;
  * `video_fib_model_fn_builder`: the fine-tuning step (train), the validation forward (eval) and the scoring forward
    (predict), with the call shape and seeds of video_qa.video_qa_model_fn_builder.
A label of -1 marks an answer outside the vocabulary (OOV), handled as video_qa handles it: weight 0 in the loss, counted
wrong, skipped by the training input.  All arithmetic of the step runs in libmerlot_b200.so (the row gather / scatter, the
K1 GEMM, gelu, LayerNorm, the CE kernel and the weighted mean); the only torch ops build row indices.  The derivation runs
once, when a store is set up.
"""
from __future__ import annotations

import json
from typing import List, Optional, Tuple

import torch

from . import ops
from .modeling import MASK, MerlotModel, _Dense, _MlpLn
from .params import VIDEO_FIB_ANSWERS, derive_fib_answers, padded_answers

MIN_ANSWERS = 2
FIRST_WORD_ID = 7  # ids 0..6 are PADDING, MASK, START, END and the NEXTCAPTION markers (utils/encode/encoder.py:16-22)


def load_answer_tokens(path: str, vocab_size: int) -> List[List[int]]:
    """The answer vocabulary of downstream.answer_tokens: a JSON list of A lists of token ids, answer a's BPE encoding.
    ValueError unless A >= 2, every list is non-empty and every id lies in [7, vocab_size) (no special id)."""
    with open(path, encoding="utf-8") as f:
        answers = json.load(f)
    if not isinstance(answers, list) or len(answers) < MIN_ANSWERS:
        n = len(answers) if isinstance(answers, list) else type(answers).__name__
        raise ValueError(f"video_fib: downstream.answer_tokens {path!r} must hold a list of >= {MIN_ANSWERS} answers, got {n}")
    out = []
    for a, toks in enumerate(answers):
        if not isinstance(toks, list) or not toks:
            raise ValueError(f"video_fib: answer {a} of {path!r} must be a non-empty list of token ids, got {toks!r}")
        for t in toks:
            if isinstance(t, bool) or not isinstance(t, int) or not FIRST_WORD_ID <= t < vocab_size:
                raise ValueError(f"video_fib: answer {a} of {path!r} holds token id {t!r} outside [{FIRST_WORD_ID}, "
                                 f"{vocab_size}) (ids below {FIRST_WORD_ID} are special)")
        out.append([int(t) for t in toks])
    return out


def check_config(model_cfg, downstream_cfg) -> Tuple[int, List[List[int]]]:
    """(F, answers) of a video_fib config: model.num_imgs and the answer vocabulary of downstream.answer_tokens
    (load_answer_tokens).  ValueError for F < 1, model.num_texts other than 1, answer_tokens missing, or a
    downstream.num_answers that is given and differs from the number of answers A."""
    F = int(model_cfg.get("num_imgs", 1))
    if F < 1:
        raise ValueError(f"video_fib: model.num_imgs (frames per question) must be >= 1, got {F}")
    T = model_cfg.get("num_texts")
    if T is not None and int(T) != 1:
        raise ValueError(f"video_fib: model.num_texts must be 1 (one sentence per example), got {T}")
    path = downstream_cfg.get("answer_tokens")
    if not path:
        raise ValueError("video_fib: downstream.answer_tokens (a JSON file of the answers' token ids) is missing")
    answers = load_answer_tokens(str(path), int(model_cfg["vocab_size"]))
    A = downstream_cfg.get("num_answers")
    if A is not None and int(A) != len(answers):
        raise ValueError(f"video_fib: downstream.num_answers is {A}, downstream.answer_tokens holds {len(answers)} answers")
    return F, answers


def blank_positions(ids: torch.Tensor) -> torch.Tensor:
    """int32 [b]: the position of the MASK in every row of lm_input [b, L] on the device.  ValueError unless every row
    holds exactly one (this reads a count back to the host; the input pipeline gives blank_pos instead)."""
    is_mask = ids == MASK
    if not bool((is_mask.sum(1) == 1).all()):
        raise ValueError("video_fib: every lm_input row must hold exactly one MASK (id 1), the blank")
    return is_mask.to(torch.int32).argmax(1).to(torch.int32)


def _head_index(model, blank_pos: torch.Tensor, b: int, Sj: int) -> torch.Tensor:
    """int32 [b]: row P * F + blank_pos[q] of sequence q of Sj rows, the joint hidden state's row at the blank."""
    bf, dev = model._bufs, model.store.device
    P = model.encoder_pieces[1]["start"]  # P * num_imgs: the language piece follows every frame's viz tokens
    key = ("_fib_base", b, Sj, P)
    if key not in bf.d:
        bf.d[key] = (torch.arange(b, device=dev, dtype=torch.int32) * Sj + P).contiguous()
    return (bf.d[key] + blank_pos.to(device=dev, dtype=torch.int32)).contiguous()


def fib_head(model, store, blank_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The head on model.encoder_info['hidden_state'] -> fp32 logits [b, A]: a view of the first A columns of a fresh
    [b, A8] buffer.  blank_pos int [b] is the MASK's position in every text (None: found on the device from the model's
    input ids)."""
    y = model.encoder_info["hidden_state"]  # bf16 [b, P*F + L, H]
    if model.num_texts != 1 or store.task != "video_fib":
        raise ValueError(f"the video_fib head reads one text per question from a ParamStore(task='video_fib'): num_texts "
                         f"{model.num_texts}, store task {store.task!r}")
    b, Sj, H = y.shape
    A = store.num_answers
    if blank_pos is None:
        blank_pos = blank_positions(model.input_ids.reshape(b, -1))
    bf = model._bufs
    idx = _head_index(model, blank_pos, b, Sj)
    x = bf.get("fib.x", (b, H), torch.bfloat16)
    ops.gather_rows(y.reshape(b * Sj, H), idx, x)
    proj = None
    if store.cfg.get("do_projection", False):
        proj = _MlpLn(store, bf, "fib.proj", x, "lm_head/projection", "lm_head/LayerNorm", H)
    dense = _Dense(store, bf, "fib", VIDEO_FIB_ANSWERS, proj.out if proj else x)
    logits = torch.empty((b, padded_answers(A)), dtype=torch.float32, device=y.device)
    dense.forward(logits)
    model._fib = {"logits": logits, "idx": idx, "proj": proj, "dense": dense, "A": A}  # what the backward reads
    return logits[:, :A]


def fib_loss(model, target: torch.Tensor):
    """Softmax cross entropy over the A answers of the logits fib_head computed last, with video_qa.qa_loss's arithmetic:
    `target` int [b] holds answers in [0, A) or -1 (OOV).  Returns (loss, accuracy, counts), 0-d fp32 CUDA tensors: loss =
    the mean over the in-vocabulary rows, accuracy = correct rows / b with OOV rows wrong, counts = {loss_sum, in_vocab,
    correct}."""
    st = getattr(model, "_fib", None)
    if st is None:
        raise RuntimeError("fib_loss needs fib_head(model, store, ...) first")
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


def fib_head_backward(model, store) -> torch.Tensor:
    """Gradient of fib_loss(fib_head(...)).  ACCUMULATES the head's parameter gradients (fib_cls/answers, and
    lm_head/projection and lm_head/LayerNorm with do_projection) into store.g and returns the bf16 d_hidden_state
    [b*(P*F+L), H] for model.backward(d_hidden_state=...): non-zero only at the blank rows."""
    st = getattr(model, "_fib", None)
    if st is None or "lse" not in st:
        raise RuntimeError("fib_head_backward needs fib_head(model, store, ...) and fib_loss(model, target) first")
    logits, A, proj, dense = st["logits"], st["A"], st["proj"], st["dense"]
    y = model.encoder_info["hidden_state"]
    b, Sj, H = y.shape
    bf = model._bufs
    # the CE kernel writes columns [0, A); the padding columns stay zero, so the padded weights get no gradient
    dlog = bf.get("fib.dlogits", tuple(logits.shape), torch.float32, zero=True)
    ops.softmax_ce_bwd(logits, st["target"], A, st["lse"], st["coeff"], dlog)
    dx = dense.backward(dlog)
    if proj is not None:
        dx = proj.backward(dx)
    d_hidden = bf.get("fib.d_hidden", (b * Sj, H), torch.bfloat16, zero=True)
    ops.scatter_add_rows(dx, st["idx"], d_hidden)
    return d_hidden


def init_answer_layer(store, answers, prefix: Optional[str] = None, restored=None) -> bool:
    """Set up a fresh ParamStore(task='video_fib') after its initialisers: restore `prefix` by name (init_checkpoint,
    ParamStore.load_checkpoint) if given, then derive the answer layer (params.derive_fib_answers) from the store's word
    embeddings and the checkpoint's lm_head/output_bias (zero without one) unless fib_cls/answers came from the checkpoint.
    `restored` (a list) receives the names load_checkpoint found missing.  Returns whether the layer was derived.
    Resuming a video_fib run (ParamStore.restore_checkpoint) restores the layer instead and never derives it."""
    from .tf_checkpoint import load_checkpoint
    missing = list(store.entries) if prefix is None else store.load_checkpoint(prefix)
    if restored is not None:
        restored[:] = missing
    names = (f"{VIDEO_FIB_ANSWERS}/kernel", f"{VIDEO_FIB_ANSWERS}/bias")
    if not any(n in missing for n in names):
        return False
    bias = None
    if prefix is not None and store.cfg.get("do_bias", False):
        bias = load_checkpoint(prefix, names=["lm_head/output_bias"]).get("lm_head/output_bias")
    derive_fib_answers(store, answers, bias)
    return True


def video_fib_model_fn_builder(config, *, store=None, dist=None, seed: int = 0, device="cuda", vit_grad_buckets: int = 4):
    """The video_fib step with the call shape of video_qa.video_qa_model_fn_builder.  Returns model_fn(features, labels,
    mode):
      * features: 'images' [b*F, h, w, 3] (or [h, w, 3, b*F] with transpose_input; question-major, frame-minor),
        'img_mask' [b, F] bool (absent: every slot holds a frame), 'lm_input' [b, L] with one MASK per row, 'blank_pos'
        [b] int (absent: found on the device); labels: {'lm_targets': [b]} (or features['lm_targets']) in [0, A), or -1
        for an OOV answer;
      * mode "train": MerlotModel(is_training=True, mask_input=False, img_mask=...), fib_head + fib_loss; metrics loss /
        accuracy / learning_rate; train_op = the head backward, model.backward(d_hidden_state=...), gradient mean over
        replicas, AdamW;
      * mode "eval": MerlotModel(is_training=False); metrics loss (over the in-vocabulary questions), accuracy (over all,
        OOV wrong), logits [b, A], predictions, and loss_sum / in_vocab / correct; no train_op;
      * mode "predict": as "eval" without lm_targets, loss or accuracy: the CE kernel is not run.
    `store=None` builds ParamStore(task="video_fib", num_answers=A), applies the reference initialisers, then
    init_answer_layer with `model.init_checkpoint` if set: a pretraining checkpoint restores the encoder and lm_head by
    name and the answer layer is derived from its embeddings and output bias.  Seeds and gradient accumulation (a list of
    micro-batch feature dicts in "train") follow video_qa_model_fn_builder."""
    from .config import replica_seed
    from .optimization import build_optimizer_from_config
    from .params import ParamStore
    from .train import StepSpec, accumulate_mean, backward_and_apply, backward_micro_batch
    m_cfg = config.model
    _, answers = check_config(m_cfg, config.downstream)
    A = len(answers)
    if store is None:
        store = ParamStore(m_cfg, device=device, optimizer_cfg=config.optimizer, task="video_fib", num_answers=A)
        store.init_reference(seed=0)
        ckpt = m_cfg.get("init_checkpoint")
        missing = []
        derived = init_answer_layer(store, answers, ckpt or None, missing)
        if ckpt:
            print(f"init_checkpoint {ckpt}: {len(missing)} variables not in the checkpoint keep their initial values: "
                  f"{', '.join(missing)}", flush=True)
        if derived:
            print(f"{VIDEO_FIB_ANSWERS}: derived from the word embeddings for {A} answers", flush=True)
    elif store.task != "video_fib":
        raise ValueError(f"the video_fib step trains a ParamStore(task='video_fib'), got task={store.task!r}")
    elif store.num_answers != A:
        raise ValueError(f"the ParamStore holds {store.num_answers} answers, downstream.answer_tokens holds {A}")
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
                fib_head(model, store, f.get("blank_pos"))
                loss, accuracy, _ = fib_loss(model, target)
                accumulate_mean(model._bufs, acc, {"loss": loss, "accuracy": accuracy}, j, n_micro)
                d_hidden = fib_head_backward(model, store)
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
        logits = fib_head(model, store, features.get("blank_pos"))
        if not is_training:
            metrics = {"logits": logits, "predictions": logits.argmax(-1)}
            if target is None:
                return StepSpec(model, (), metrics, None)
            loss, acc, counts = fib_loss(model, target)
            metrics.update(loss=loss, accuracy=acc, **counts)
            return StepSpec(model, (loss,), metrics, None)
        loss, acc, _ = fib_loss(model, target)
        metrics = {"loss": loss, "accuracy": acc, "learning_rate": optimizer.current_lr()}

        def train_op():
            d_hidden = fib_head_backward(model, store)
            backward_and_apply(model, optimizer, dist, metrics=metrics, vit_grad_buckets=vit_grad_buckets, d_hidden_state=d_hidden)

        return StepSpec(model, (loss,), metrics, train_op)

    model_fn.store = store
    model_fn.optimizer = optimizer
    model_fn.answers = answers
    return model_fn
