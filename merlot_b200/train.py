"""Driver-loop role of model/train.py + model_fn (model/modeling.py:671-810), re-provided without TPUEstimator.

  * `synthetic_batch`  -- features with the dataloader's output contract (model/dataloader.py:56-126,210-272):
                          images [b*n,H,W,3] bf16, input_ids [b,n,Lc] int32 (START first, zero padded),
                          shuffled_idx_img [B*g] int32, video_src_ids [b,n] int32.
  * `synthetic_vcr_batch` -- the same for VCR fine-tuning (downstream/vcr/dataloader_joint.py:135-189,257-271).
  * `synthetic_video_mc_batch` -- the same for multiple-choice video QA (video_mc_input.py's training batches).
  * `synthetic_video_qa_batch` -- the same for open-ended video QA (video_qa_input.py's training batches).
  * `synthetic_video_fib_batch` -- the same for fill-in-the-blank video QA (video_fib_input.py's training batches).
  * `model_fn_builder` -- same name and call shape as the reference; returns a model_fn(features, labels, mode, params)
                          that builds MerlotModel(is_training=True, mask_input=True), sums lang + contr + temp losses
                          (modeling.py:700-713) and exposes `train_op()` = backward + gradient all-reduce + AdamW.
  * `DataParallel`     -- the two collectives of the reference (SURVEY 2.3): gradient mean over replicas
                          (CrossShardOptimizer, utils/optimization.py:241-245) as ONE NCCL all-reduce over the flat
                          gradient arena, and the contrastive feature all-gather / reduce-scatter
                          (tpu_cross_replica_stack, utils/model_utils.py:673-707).
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch

from .config import NeatConfig, micro_batching, replica_seed
from .dataloader import input_fn_builder, train_files
from .modeling import MASK, MerlotModel, START, _Buffers, contrastive_head, contrastive_head_bwd
from .optimization import build_optimizer_from_config
from .params import ParamStore


class DataParallel:
    """One process per GPU; torch.distributed (NCCL over NVLink/NVSwitch, or gloo for the CPU tests) is the plumbing."""

    def __init__(self, backend: Optional[str] = None):
        import torch.distributed as dist
        self.dist = dist
        # The gradient all-reduce runs under the backward pass: bound the SMs NCCL may take (one collective CTA owns a whole SM)
        # and keep the persistent GEMM / attention grids off those SMs (merlot_set_sm_reserve) -- otherwise every persistent
        # kernel launched while a collective is in flight has CTAs queueing behind NCCL's and runs up to twice as long.
        self.comm_ctas = int(os.environ.get("MERLOT_DP_COMM_CTAS", "24"))
        if self.comm_ctas > 0:
            os.environ.setdefault("NCCL_MAX_CTAS", str(self.comm_ctas))
            os.environ.setdefault("NCCL_MIN_CTAS", str(min(4, self.comm_ctas)))
        if not dist.is_initialized():
            dist.init_process_group(backend=backend or ("nccl" if torch.cuda.is_available() else "gloo"))
        self.world = dist.get_world_size()
        self.rank = dist.get_rank()
        self._lib = None
        if self.world > 1 and self.comm_ctas > 0 and torch.cuda.is_available():
            from . import _lib
            self._lib = _lib.lib()

    def reserve_sms(self, on: bool):
        """Kernels ENQUEUED while this is on leave `comm_ctas` SMs to the collective (train_op switches it on for the part of
        the backward pass that runs under the gradient all-reduce)."""
        if self._lib is not None:
            self._lib.merlot_set_sm_reserve(self.comm_ctas if on else 0)

    def all_reduce_grads(self, g: torch.Tensor):
        """Sum over replicas; the 1/world of the MEAN reduction is folded into the AdamW kernel (grad_scale)."""
        if self.world > 1:
            self.dist.all_reduce(g, op=self.dist.ReduceOp.SUM)

    skip_grad_allreduce = False  # diagnostics only (bench.py: step time without the gradient collective = its exposed cost)

    def all_reduce_ranges_async(self, g: torch.Tensor, ranges):
        """Start summing g[a:b] for every range on the NCCL stream, ordered after the work already queued on the current
        stream; returns handles for wait_all().  Lets the collective overlap the rest of the backward pass."""
        if self.world <= 1 or self.skip_grad_allreduce:
            return []
        return [self.dist.all_reduce(g[a:b], op=self.dist.ReduceOp.SUM, async_op=True) for a, b in ranges if b > a]

    @staticmethod
    def wait_all(handles):
        for h in handles:
            h.wait()  # the current stream waits for the collective; no host sync

    def all_gather_rows(self, x: torch.Tensor) -> torch.Tensor:
        out = torch.empty((self.world * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        self.dist.all_gather_into_tensor(out, x.contiguous())
        return out

    def reduce_scatter_rows(self, x_all: torch.Tensor) -> torch.Tensor:
        n = x_all.shape[0] // self.world
        out = torch.empty((n,) + tuple(x_all.shape[1:]), dtype=x_all.dtype, device=x_all.device)
        self.dist.reduce_scatter_tensor(out, x_all.contiguous(), op=self.dist.ReduceOp.SUM)
        return out

    def barrier(self):
        self.dist.barrier()


def synthetic_batch(config: NeatConfig, batch_size: int, seed: int = 0, device="cuda", num_chunks: Optional[int] = None,
                    chunk_text_len: Optional[int] = None, pin: bool = False) -> Dict[str, torch.Tensor]:
    """Synthetic features of the dataloader's shapes (SURVEY 8(d)): images uniform [0,1) bf16; ids uniform in
    [100, 50357) with START at position 0 and a zero-padded tail of random length; one shuffled group per batch."""
    m, d = config.model, config.data
    n = num_chunks or m.get("num_chunks_in_group", d.get("num_chunks", 4))
    Lc = chunk_text_len or d.get("chunk_text_len", 32)
    Hh, Ww = m["image_size"]
    g = torch.Generator().manual_seed(seed)
    images = torch.rand(batch_size * n, Hh, Ww, 3, generator=g).to(torch.bfloat16)
    ids = torch.randint(100, 50357, (batch_size, n, Lc), generator=g, dtype=torch.int32)
    ids[:, :, 0] = START
    lens = torch.randint(min(8, Lc), Lc + 1, (batch_size, n), generator=g)
    ids = ids * (torch.arange(Lc)[None, None] < lens[..., None]).int()
    ncg = m.get("num_chunks_in_group", n)
    B = batch_size * n // ncg
    shuf = torch.arange(ncg, dtype=torch.int32).repeat(B)
    if m.get("image_shuffle_prob", 0) > 0:  # dataloader offset 16 (model/dataloader.py:226,254)
        shuf[:ncg] = 16 + torch.randperm(ncg, generator=g).int()
    vid = torch.zeros(batch_size, n, dtype=torch.int32)
    feats = {"images": images, "input_ids": ids, "shuffled_idx_img": shuf, "video_src_ids": vid}
    if pin:
        return {k: v.pin_memory() for k, v in feats.items()}
    return {k: v.to(device) for k, v in feats.items()}


VCR_MAX_NUM_TOKENS = 184  # downstream/vcr/dataloader_joint.py:135


def synthetic_vcr_batch(config: NeatConfig, questions: int, seed: int = 0, device="cuda") -> Dict[str, torch.Tensor]:
    """Training features of `questions` VCR questions with the joint dataloader's shapes: images [2q, H, W, 3] bf16 uniform
    [0,1) ordered [q0 answer, q0 rationale, q1 answer, ...]; lm_input [2q*4, 184] int32, every text START followed by ids in
    [100, vocab) and a zero-padded tail; lm_targets [2q] int32 in [0, 4).  Synthetic ids stand in for the prompts, contexts
    and answer choices (dataloader_joint.py:167-181)."""
    m = config.model
    Hh, Ww = m["image_size"]
    L = VCR_MAX_NUM_TOKENS
    g = torch.Generator().manual_seed(seed)
    images = torch.rand(2 * questions, Hh, Ww, 3, generator=g).to(torch.bfloat16)
    ids = torch.randint(100, m["vocab_size"], (2 * questions * 4, L), generator=g, dtype=torch.int32)
    ids[:, 0] = START
    lens = torch.randint(16, L + 1, (2 * questions * 4,), generator=g)
    ids = ids * (torch.arange(L)[None] < lens[:, None]).int()
    targets = torch.randint(0, 4, (2 * questions,), generator=g, dtype=torch.int32)
    feats = {"images": images, "lm_input": ids, "lm_targets": targets}
    return {k: v.to(device) for k, v in feats.items()}


def synthetic_video_mc_batch(config: NeatConfig, questions: int, seed: int = 0, device="cuda") -> Dict[str, torch.Tensor]:
    """Training features of `questions` multiple-choice video questions with video_mc_input's shapes (F = model.num_imgs
    frames, C = model.num_texts candidates, L = downstream.max_text_len, default 128): images [q*F, H, W, 3] bf16 uniform
    [0,1) with zeros in the empty slots, img_mask [q, F] bool (question i holds 1 + i % F frames), lm_input [q*C, L] int32,
    every text START followed by ids in [100, vocab) and a zero-padded tail, lm_targets [q] int32 in [0, C)."""
    m = config.model
    Hh, Ww = m["image_size"]
    F, C = int(m.get("num_imgs", 1)), int(m.get("num_texts", 1))
    L = int(config.downstream.get("max_text_len", 128))
    g = torch.Generator().manual_seed(seed)
    img_mask = torch.arange(F)[None] < (1 + torch.arange(questions) % F)[:, None]
    images = torch.rand(questions * F, Hh, Ww, 3, generator=g) * img_mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, m["vocab_size"], (questions * C, L), generator=g, dtype=torch.int32)
    ids[:, 0] = START
    lens = torch.randint(min(16, L), L + 1, (questions * C,), generator=g)
    ids = ids * (torch.arange(L)[None] < lens[:, None]).int()
    targets = torch.randint(0, C, (questions,), generator=g, dtype=torch.int32)
    feats = {"images": images.to(torch.bfloat16), "img_mask": img_mask, "lm_input": ids, "lm_targets": targets}
    return {k: v.to(device) for k, v in feats.items()}


def synthetic_video_qa_batch(config: NeatConfig, questions: int, seed: int = 0, device="cuda") -> Dict[str, torch.Tensor]:
    """Training features of `questions` open-ended video questions with video_qa_input's shapes (F = model.num_imgs frames,
    L = downstream.max_text_len, default 128, A = downstream.num_answers): images and img_mask as
    synthetic_video_mc_batch's, lm_input [q, L] int32, every text START followed by ids in [100, vocab) and a zero-padded
    tail, lm_targets [q] int32 in [0, A)."""
    m = config.model
    Hh, Ww = m["image_size"]
    F, A = int(m.get("num_imgs", 1)), int(config.downstream["num_answers"])
    L = int(config.downstream.get("max_text_len", 128))
    g = torch.Generator().manual_seed(seed)
    img_mask = torch.arange(F)[None] < (1 + torch.arange(questions) % F)[:, None]
    images = torch.rand(questions * F, Hh, Ww, 3, generator=g) * img_mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, m["vocab_size"], (questions, L), generator=g, dtype=torch.int32)
    ids[:, 0] = START
    lens = torch.randint(min(16, L), L + 1, (questions,), generator=g)
    ids = ids * (torch.arange(L)[None] < lens[:, None]).int()
    targets = torch.randint(0, A, (questions,), generator=g, dtype=torch.int32)
    feats = {"images": images.to(torch.bfloat16), "img_mask": img_mask, "lm_input": ids, "lm_targets": targets}
    return {k: v.to(device) for k, v in feats.items()}


def synthetic_video_fib_batch(config: NeatConfig, questions: int, seed: int = 0, device="cuda") -> Dict[str, torch.Tensor]:
    """Training features of `questions` fill-in-the-blank video questions with video_fib_input's shapes: images, img_mask
    and lm_input drawn as synthetic_video_qa_batch's, then one MASK at a random position of every text's words,
    blank_pos [q] int32 its position, and lm_targets [q] int32 in [0, A) (A = the answers of downstream.answer_tokens)."""
    from .video_fib import check_config
    m = config.model
    Hh, Ww = m["image_size"]
    F, answers = check_config(m, config.downstream)
    L = int(config.downstream.get("max_text_len", 128))
    g = torch.Generator().manual_seed(seed)
    img_mask = torch.arange(F)[None] < (1 + torch.arange(questions) % F)[:, None]
    images = torch.rand(questions * F, Hh, Ww, 3, generator=g) * img_mask.reshape(-1, 1, 1, 1)
    ids = torch.randint(100, m["vocab_size"], (questions, L), generator=g, dtype=torch.int32)
    ids[:, 0] = START
    lens = torch.randint(min(16, L), L + 1, (questions,), generator=g)
    ids = ids * (torch.arange(L)[None] < lens[:, None]).int()
    blank = 1 + (torch.rand(questions, generator=g) * (lens - 1)).long()  # one of the words after START
    ids[torch.arange(questions), blank] = MASK
    targets = torch.randint(0, len(answers), (questions,), generator=g, dtype=torch.int32)
    feats = {"images": images.to(torch.bfloat16), "img_mask": img_mask, "lm_input": ids, "lm_targets": targets,
             "blank_pos": blank.to(torch.int32)}
    return {k: v.to(device) for k, v in feats.items()}


class StepSpec:
    """What TPUEstimatorSpec carries in the reference: loss, metrics and the train op."""

    def __init__(self, model, loss_parts, metrics, train_op):
        self.model, self.loss_parts, self.metrics, self.train_op = model, loss_parts, metrics, train_op

    @property
    def loss(self):
        return sum(float(x) for x in self.loss_parts)


def backward_and_apply(model, optimizer, dist: Optional[DataParallel], *, metrics: dict, skip=(), vit_grad_buckets: int = 4,
                       d_hidden_state=None, d_contrastive_features=None, accum: int = 1):
    """The train op of every training step: model.backward (with an external head's gradient `d_hidden_state`, if any, whose
    parameter gradients are already in store.g, and the injected contrastive gradient `d_contrastive_features`), the gradient
    mean over replicas and AdamW.  With clip_norm > 0 the pre-clip global norm goes into metrics['gradnorms/_overall'] and is
    returned (None without clipping).
    `accum` = A > 1: this is the last of A micro-batches, whose earlier backward passes ran through backward_micro_batch,
    and AdamW applies the mean over the world * A virtual replicas.  With clip_norm > 0 every micro-batch's gradient is
    clipped alone (the reference's per-replica clip) into store.grad_accumulator(), which is then all-reduced and applied."""
    store = optimizer.store
    world = dist.world if dist is not None else 1
    grad_scale = 1.0 / (world * accum)
    bwd = dict(d_hidden_state=d_hidden_state, d_contrastive_features=d_contrastive_features)
    pending = []
    if optimizer.clip_norm > 0.0:  # local clip needs the complete local gradient first: no bucket overlap
        model.backward(**bwd)
        if accum > 1:
            norm, grads = optimizer.clip_accumulate(), store.grad_accumulator()
        else:
            norm, grads = optimizer.clip_gradients(), store.g
        metrics["gradnorms/_overall"] = norm
        if world > 1:
            dist.all_reduce_grads(grads)
        optimizer.apply_gradients(grad_scale=grad_scale, skip=skip, zero_grad=True, grads=grads)
        return norm
    elif world > 1:
        # Bucketed, overlapped gradient all-reduce (CrossShardOptimizer's mean, utils/optimization.py:241-245; the 1/world
        # is folded into AdamW).  Bucket 0 = everything outside the ViT, reduced while the ViT backward runs; the ViT is
        # walked in layer groups top-down and each group's kernels are reduced as soon as that group has run, so only
        # the last group's bucket is exposed.  AdamW updates every bucket as its reduction lands.
        groups, vit_ranges = store.vit_buckets(vit_grad_buckets)
        vit_pending = []

        def on_group(k):
            if k + 1 < len(groups):
                vit_pending.append(dist.all_reduce_ranges_async(store.g, vit_ranges[k]))

        def on_rest():
            pending.extend(dist.all_reduce_ranges_async(store.g, store.rest_ranges))
            dist.reserve_sms(True)  # the ViT backward is enqueued (and runs) under the collectives

        model.backward(on_non_vit_grads_ready=on_rest, vit_layer_groups=groups, on_vit_group_done=on_group, **bwd)
        dist.reserve_sms(False)
        vit_pending.append(dist.all_reduce_ranges_async(store.g, vit_ranges[-1]))
        dist.wait_all(pending)
        optimizer.apply_gradients(grad_scale=grad_scale, skip=skip, zero_grad=True, only=store.rest_ranges, advance=False)
        for k, hs in enumerate(vit_pending):
            dist.wait_all(hs)
            optimizer.apply_gradients(grad_scale=grad_scale, skip=skip, zero_grad=True, only=vit_ranges[k],
                                      advance=(k + 1 == len(vit_pending)))
    else:
        model.backward(**bwd)
        optimizer.apply_gradients(grad_scale=grad_scale, skip=skip, zero_grad=True)
    return None


def backward_micro_batch(model, optimizer, *, d_hidden_state=None, d_contrastive_features=None):
    """model.backward of a micro-batch before the step's last.  Without clipping store.g accumulates (every gradient writer
    adds).  With clip_norm > 0 the micro-batch's gradient, complete in store.g, is clipped into store.grad_accumulator() and
    store.g is zeroed for the next micro-batch; returns its pre-clip norm (None without clipping)."""
    model.backward(d_hidden_state=d_hidden_state, d_contrastive_features=d_contrastive_features)
    return optimizer.clip_accumulate() if optimizer.clip_norm > 0.0 else None


def accumulate_mean(bufs, acc: dict, metrics: dict, j: int, accum: int):
    """acc[k] <- the running mean over micro-batches 0..j of accum of every tensor metric (0-d fp32 CUDA tensors, which the
    next micro-batch's buffers overwrite); other values are copied."""
    from . import ops
    for k, v in metrics.items():
        if not torch.is_tensor(v):
            acc[k] = v
            continue
        t = bufs.get(f"accum.metric.{k}", (1,), torch.float32)
        ops.axpby(v.float(), t, 1.0 / accum, 1.0 if j else 0.0)
        acc[k] = t[0]


def model_fn_builder(config: NeatConfig, *, store: Optional[ParamStore] = None, dist: Optional[DataParallel] = None,
                     device="cuda", seed: int = 0, log_attention_probs: bool = True, vit_grad_buckets: int = 4):
    """model/modeling.py:671-810.  `seed` is the run seed of every random draw of the step (dropout masks, Gumbel noise,
    span lengths, 10/80/10 options, replacement ids): replica r at step t uses seed + t*world + r, so replicas draw
    independently like the reference's per-core tf.random ops and two runs with different seeds differ.
    `log_attention_probs` defaults to the reference's model_fn (modeling.py:691-709 computes attn/* every step).
    Modes: "train" (the default), "eval" (eval_step) and "predict" (predict_step), the last two with params
    {"eval_batch": k} and, for "predict", the reference's params["batch_size"].

    Gradient accumulation: model_fn([f_0, ..., f_{A-1}]) with A feature dicts of one micro-batch each is the step of the
    world * A virtual replicas v = rank * A + j, with seed + t*world*A + v (config.replica_seed).  The contrastive loss of
    each replica is taken against the features of all world * A replicas, exactly, in two passes: model_fn runs a
    features-only forward of every micro-batch, the contrastive head over all their features and its backward (the
    contrastive metrics are known on return); train_op then runs, per micro-batch, the training forward again with the same
    seed and masks, mask_loss, temporal_loss and the backward from the injected contrastive gradient.  Only the last
    micro-batch's backward runs the bucketed all-reduce; AdamW applies the mean over the world * A replicas.  The lang/,
    temporal/ and attn/ metrics (means over the rank's micro-batches) and the loss are complete after train_op()."""
    if store is None:
        store = ParamStore(config.model, device=device, optimizer_cfg=config.optimizer)
        store.init_reference(seed=0)
    optimizer, _ = build_optimizer_from_config(loss=None, optimizer_config=config.optimizer, device_config=config.device,
                                               store=store)
    skip = variables_without_gradient(config.model, store)
    world, rank = (dist.world, dist.rank) if dist is not None else (1, 0)

    def build_model(features, dropout_seed, transpose=True, replicas=dist, **kw):
        imgs = features["images"]
        if transpose and config.model.get("transpose_input", False) and imgs.shape[-1] != 3:
            imgs = imgs.permute(3, 0, 1, 2).contiguous()  # [H,W,3,N] -> [N,H,W,3], modeling.py:683-685
        return MerlotModel(config=config.model, is_training=True,  # the reference hard-codes True (:693, SURVEY quirk 3)
                           image=imgs, input_ids=features["input_ids"], use_tpu=config.device.get("use_tpu", False),
                           shuffled_idx_img=features.get("shuffled_idx_img", None), mask_input=True, params=store,
                           dropout_seed=dropout_seed, dist=replicas, **kw)

    def temporal_loss(model, features):
        if config.model.get("temporal_coef", 1.0) > 0.0:
            return model.temporal_loss(features["shuffled_idx_img"], video_src_ids=features["video_src_ids"])
        return torch.zeros((), device=store.device), {}

    def metrics_of(model, lang_losses, contr_losses, temp_losses, learning_rate=True):
        losses = {f"lang/{k}": v for k, v in lang_losses.items()}
        losses.update({f"contr/{k}": v for k, v in contr_losses.items()})
        losses.update({f"temporal/{k}": v for k, v in temp_losses.items()})
        if learning_rate:  # a train metric (modeling.py:720-725); eval_metrics take `losses` alone (:708-711, :788-798)
            losses["learning_rate"] = optimizer.current_lr()
        if log_attention_probs:  # modeling.py:709  losses.update(model.attention_log)
            losses.update({f"attn/{k}": v for k, v in model.attention_log.items()})
        return losses

    def model_fn(features, labels=None, mode="train", params=None):
        if mode == "eval":
            return eval_step(features, int((params or {}).get("eval_batch", 0)))
        if mode == "predict":
            params = params or {}
            return predict_step(features, int(params.get("eval_batch", 0)),
                                int(params.get("batch_size", features["input_ids"].shape[0])))
        if isinstance(features, (list, tuple)):
            return accumulated_step(list(features))
        model = build_model(features, seed + store.global_step * world + rank, transpose=mode == "train",
                            log_attention_probs=log_attention_probs)
        lang_loss, lang_losses = model.mask_loss()
        contr_loss, contr_losses = model.contrastive_loss()
        temp_loss, temp_losses = temporal_loss(model, features)
        losses = metrics_of(model, lang_losses, contr_losses, temp_losses)

        def train_op():
            backward_and_apply(model, optimizer, dist, metrics=losses, skip=skip, vit_grad_buckets=vit_grad_buckets)

        return StepSpec(model, (lang_loss, contr_loss, temp_loss), losses, train_op)

    def eval_step(features, k, **kw):
        """EVAL mode (modeling.py:691-711, :788-798) on evaluation batch k: the training forward as the reference builds it
        (is_training=True, mask_input=True), keeping nothing for a backward, with no collective (one batch is one replica:
        its contrastive negatives are its own videos) and with the dropout and masking seed eval_seed(seed, k).  Returns a
        StepSpec whose metrics are the `losses` dict without learning_rate, whose `total_loss` is lang + contr + temporal
        (device scalars, which the next model on this store overwrites) and whose train_op is None."""
        kw.setdefault("log_attention_probs", log_attention_probs)
        model = build_model(features, eval_seed(seed, k), transpose=False, replicas=None, save_for_backward=False, **kw)
        lang_loss, lang_losses = model.mask_loss()
        contr_loss, contr_losses = model.contrastive_loss()
        temp_loss, temp_losses = temporal_loss(model, features)
        spec = StepSpec(model, (lang_loss, contr_loss, temp_loss),
                        metrics_of(model, lang_losses, contr_losses, temp_losses, learning_rate=False), None)
        spec.total_loss = lang_loss + contr_loss + temp_loss
        return spec

    def predict_step(features, k, bsz):
        """PREDICT mode (modeling.py:760-787) on evaluation batch k of bsz videos: eval_step's forward (same seed, dropout
        and masks, no backward, no collective) with the joint encoder's attention maps exported as their layer mean.
        Returns the reference's predictions dict on the host (predictions()): self_attn_probs [bsz, B // bsz, S, S], the
        layer and head mean of the joint maps; lang_attn_probs, the language-only encoder's per-layer head means reshaped
        to lead with bsz; masked_ids; every lang/ attn/ contr/ temporal/ loss tiled to [bsz]; and the batch's other
        features.  attn/* are the block sums of the exported map (MerlotModel's "layer_mean" export).

        `images` is left out on purpose, unlike the reference: it is the model's input, the evaluation pipeline reproduces
        it from the same seed and batch index, and keeping it would roughly double the output."""
        spec = eval_step(features, k, export_attention_probs="layer_mean")
        m = spec.model
        if m.batch_size != bsz:
            raise ValueError(f"predict: params batch_size {bsz} is not the batch's {m.batch_size} videos")
        out = {name: v for name, v in features.items() if name != "images"}
        sap = m.encoder_info["self_attn_probs"]  # [B, S, S], already the mean over layers
        out["self_attn_probs"] = sap.reshape(bsz, m.B // bsz, *sap.shape[1:])
        lap = m.lang_transformer_info["self_attn_probs"]  # [B_lo, layers, L, L]
        lead = [bsz] if lap.shape[0] == bsz else [bsz, lap.shape[0] // bsz]  # the reference reshapes to [bsz] + shape[1:]
        out["lang_attn_probs"] = lap.reshape(lead + list(lap.shape[1:]))
        out["masked_ids"] = m.lang_mask_info["masked_ids"]
        out.update(spec.metrics)
        return predictions(out, bsz)

    def accumulated_step(micro):
        A = len(micro)
        if A < 1:
            raise ValueError("model_fn needs at least one micro-batch")
        bufs = _Buffers(store)
        seeds = [replica_seed(seed, store.global_step, world, A, rank, j) for j in range(A)]
        # pass 1: every micro-batch's normalised features into rows [j*n, (j+1)*n) of the step's feature buffers
        masks, feat = [], None
        for j, f in enumerate(micro):
            m1 = build_model(f, seeds[j], features_only=True, log_attention_probs=False)
            lang, viz = m1.contrastive_features()
            n, Cs = lang.n, lang.Cs
            if feat is None:
                feat = {k: bufs.get(f"accum.feat.{k}", (A * n, Cs), torch.float32) for k in ("lang", "viz")}
            feat["lang"][j * n:(j + 1) * n].copy_(lang.feat)
            feat["viz"][j * n:(j + 1) * n].copy_(viz.feat)
            # kept, not redrawn: mask_inputs' attention sums use float atomics, so a second draw may pick other tokens
            masks.append({k: v.clone() for k, v in m1.lang_mask_info.items()})
        info, contr_losses = contrastive_head(bufs, config.model, dist, feat["lang"], feat["viz"], n)
        d_feat = contrastive_head_bwd(bufs, dist, info)
        metrics = {f"contr/{k}": v for k, v in contr_losses.items()}
        loss_parts = []

        def train_op():
            acc = {}
            for j, f in enumerate(micro):
                m2 = build_model(f, seeds[j], mask_override=masks[j], log_attention_probs=log_attention_probs)
                lang_loss, lang_losses = m2.mask_loss()
                temp_loss, temp_losses = temporal_loss(m2, f)
                mj = metrics_of(m2, lang_losses, {}, temp_losses)
                mj.update(_lang=lang_loss, _temp=temp_loss)
                accumulate_mean(bufs, acc, mj, j, A)
                dc = (d_feat["lang"][j * n:(j + 1) * n], d_feat["viz"][j * n:(j + 1) * n])
                if j + 1 < A:
                    norm = backward_micro_batch(m2, optimizer, d_contrastive_features=dc)
                else:
                    norm = backward_and_apply(m2, optimizer, dist, metrics=metrics, skip=skip,
                                              vit_grad_buckets=vit_grad_buckets, d_contrastive_features=dc, accum=A)
                if norm is not None and A > 1:
                    accumulate_mean(bufs, acc, {"gradnorms/_overall": norm}, j, A)
            loss_parts[:] = [acc.pop("_lang"), contr_losses["loss_all"], acc.pop("_temp")]
            metrics.update(acc)

        spec = StepSpec(None, loss_parts, metrics, train_op)
        spec.mask_info = masks  # lang_mask_info of every micro-batch, as pass 1 drew it
        return spec

    model_fn.store = store
    model_fn.optimizer = optimizer
    return model_fn


def predictions(features: Dict, bsz: int) -> Dict:
    """The last step of the reference's PREDICT mode (modeling.py:774-784) on the host: every entry, by sorted name, as a
    NumPy array -- a scalar tiled to [bsz], an array whose leading axis is not bsz reshaped to [bsz, -1] -- with
    floating-point values as float32 and integers and booleans as int32."""
    import numpy as np
    out = {}
    for name in sorted(features):
        v = features[name]
        v = v.detach().cpu() if torch.is_tensor(v) else torch.as_tensor(v)
        v = v.float() if v.is_floating_point() else v.to(torch.int32)
        if v.dim() == 0:
            v = v[None].repeat(bsz)
        elif v.shape[0] != bsz:
            v = v.reshape(bsz, -1)
        out[name] = np.ascontiguousarray(v.numpy())
    return out


def eval_seed(seed: int, k: int) -> int:
    """Dropout and masking seed of evaluation batch k: a function of the run seed and k only, so every checkpoint and every
    rank count draws the same masks for batch k (the reference reseeds from the clock)."""
    return seed + k


def _step_for(config: NeatConfig):
    """(model_fn_builder, synthetic batch) of the configured task: downstream.task 'vcr' fine-tunes on VCR
    (downstream/vcr/train.py), 'video_mc' on multiple-choice video QA (video_mc.py), 'video_qa' on open-ended video QA
    (video_qa.py), 'video_fib' on fill-in-the-blank video QA (video_fib.py), anything else pretrains (model/train.py)."""
    if config.downstream.get("task") == "vcr":
        from .vcr import vcr_model_fn_builder
        return vcr_model_fn_builder, synthetic_vcr_batch
    if config.downstream.get("task") == "video_mc":
        from .video_mc import video_mc_model_fn_builder
        return video_mc_model_fn_builder, synthetic_video_mc_batch
    if config.downstream.get("task") == "video_qa":
        from .video_qa import video_qa_model_fn_builder
        return video_qa_model_fn_builder, synthetic_video_qa_batch
    if config.downstream.get("task") == "video_fib":
        from .video_fib import video_fib_model_fn_builder
        return video_fib_model_fn_builder, synthetic_video_fib_batch
    return model_fn_builder, synthetic_batch


def variables_without_gradient(model_cfg: dict, store: ParamStore):
    """Entries whose gradient is None in the training graph, so the reference's apply_gradients neither updates them nor
    creates their Adam slots: the `skip` list model_fn_builder hands AdamW (no viz_viz temporal head without image
    shuffling, no temporal heads at temporal_coef 0).  The VCR, video_mc, video_qa and video_fib graphs reach every variable
    of their store."""
    if store.task in ("vcr", "video_mc", "video_qa", "video_fib"):
        return []
    if model_cfg.get("temporal_coef", 1.0) > 0.0:
        return [] if model_cfg.get("image_shuffle_prob", 0) > 0 else [n for n in store.entries if n.startswith("viz_viz_temporal/")]
    return [n for n in store.entries if "_temporal/" in n]


def main(argv=None):
    """`python -m merlot_b200.train configs/merlot.yaml` (or merlot_vcr.yaml, or a downstream.task: video_mc, video_qa or
    video_fib config) -- the role of model/train.py:9-26 and downstream/vcr/train.py.  Every task reads data.train_file
    when it matches at least one file (pretraining through dataloader.input_fn_builder, VCR fine-tuning through
    vcr_input.input_fn_builder, video_mc through video_mc_input.input_fn_builder, video_qa through
    video_qa_input.input_fn_builder, video_fib through video_fib_input.input_fn_builder) and otherwise trains on synthetic
    batches.

    Checkpoints, as the reference's Estimator keeps them (utils/neat_config.py:136-141): when device.output_dir already names
    a latest checkpoint, every rank restores it (parameters, Adam slots, global_step; this takes precedence over
    init_checkpoint) and training continues from its global_step to num_train_steps.  model.ckpt-<global_step> is written
    whenever global_step is a multiple of device.iterations_per_loop (default 1000) and after the last step, and every
    checkpoint is kept.  Rank 0 writes; all ranks then meet at a barrier.  The input pipeline's position is not saved: a
    resumed run seeds it with the restored global_step so that it does not replay the first batches.

    With device.micro_batch_size every rank draws A = train_batch_size / (world * micro_batch_size) micro-batches per
    optimizer step and accumulates their gradients (config.micro_batching, model_fn_builder); global_step, the learning-rate
    schedule and the checkpoints count optimizer steps."""
    config = NeatConfig.from_args("Train MERLOT (H100-native)", argv=argv)
    output_dir = str(config.device["output_dir"])
    if "://" in output_dir:
        raise ValueError(f"device.output_dir {output_dir!r}: only local directories are supported for checkpoints")
    dist = DataParallel() if int(os.environ.get("WORLD_SIZE", "1")) > 1 else None
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    from .tf_checkpoint import latest_checkpoint, update_checkpoint_state
    builder, make_batch = _step_for(config)
    model_fn = builder(config, dist=dist)
    store = model_fn.store
    skip = variables_without_gradient(config.model, store)
    rank, world = (dist.rank, dist.world) if dist else (0, 1)
    resume = latest_checkpoint(output_dir)
    if resume:
        store.restore_checkpoint(resume, skip=skip)
        if rank == 0:
            print(f"restored {resume}: continuing from global_step {store.global_step}", flush=True)
    num_steps = config.optimizer.get("num_train_steps", 10)
    every = int(config.device.get("iterations_per_loop", 1000))

    def save():
        if rank == 0:
            os.makedirs(output_dir, exist_ok=True)
            prefix = os.path.join(output_dir, f"model.ckpt-{store.global_step}")
            store.save_checkpoint(prefix, skip=skip)
            update_checkpoint_state(output_dir, prefix)
            print(f"saved {prefix}", flush=True)
        if dist is not None:
            dist.barrier()

    accum, per_rank = micro_batching(config.device, world)  # A micro-batches of per_rank examples per step and rank
    pipeline = None
    if train_files(config.data):
        from . import vcr_input, video_fib_input, video_mc_input, video_qa_input
        if make_batch is synthetic_batch:
            build_input = input_fn_builder
        elif make_batch is synthetic_video_mc_batch:
            build_input = video_mc_input.input_fn_builder
        elif make_batch is synthetic_video_qa_batch:
            build_input = video_qa_input.input_fn_builder
        elif make_batch is synthetic_video_fib_batch:
            build_input = video_fib_input.input_fn_builder
        else:
            build_input = vcr_input.input_fn_builder
        pipeline = build_input(config, is_training=True, rank=rank, world=world, seed=store.global_step if resume else 0,
                               batch_size=per_rank)
    elif rank == 0:
        what = {synthetic_batch: f"data.train_file {config.data.get('train_file')!r} matches no file",
                synthetic_video_mc_batch: "video_mc fine-tuning",
                synthetic_video_qa_batch: "video_qa fine-tuning",
                synthetic_video_fib_batch: "video_fib fine-tuning"}.get(make_batch, "VCR fine-tuning")
        print(f"{what}: training on synthetic batches", flush=True)
    try:
        for step in range(store.global_step, num_steps):
            if pipeline is not None:
                feats = [next(pipeline) for _ in range(accum)]
            else:
                feats = [make_batch(config, per_rank, seed=step * accum + j + rank * 100003) for j in range(accum)]
            spec = model_fn(feats[0] if accum == 1 else feats, None, "train", None)
            spec.train_op()
            if step % 10 == 0 and rank == 0:
                print(f"step {step} loss {spec.loss:.4f} lr {spec.metrics['learning_rate']:.3e}", flush=True)
            if store.global_step % every == 0 or store.global_step == num_steps:
                save()
    finally:
        if pipeline is not None:
            pipeline.close()


if __name__ == "__main__":
    main()
