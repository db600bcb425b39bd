"""Driver-loop role of model/train.py + model_fn (model/modeling.py:671-810), re-provided without TPUEstimator.

  * `synthetic_batch`  -- features with the dataloader's output contract (model/dataloader.py:56-126,210-272):
                          images [b*n,H,W,3] bf16, input_ids [b,n,Lc] int32 (START first, zero padded),
                          shuffled_idx_img [B*g] int32, video_src_ids [b,n] int32.
  * `synthetic_vcr_batch` -- the same for VCR fine-tuning (downstream/vcr/dataloader_joint.py:135-189,257-271).
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

from .config import NeatConfig
from .modeling import MerlotModel, START
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


class StepSpec:
    """What TPUEstimatorSpec carries in the reference: loss, metrics and the train op."""

    def __init__(self, model, loss_parts, metrics, train_op):
        self.model, self.loss_parts, self.metrics, self.train_op = model, loss_parts, metrics, train_op

    @property
    def loss(self):
        return sum(float(x) for x in self.loss_parts)


def backward_and_apply(model, optimizer, dist: Optional[DataParallel], *, metrics: dict, skip=(), vit_grad_buckets: int = 4,
                       d_hidden_state=None):
    """The train op of every training step: model.backward (with an external head's gradient `d_hidden_state`, if any, whose
    parameter gradients are already in store.g), the gradient mean over replicas and AdamW.  With clip_norm > 0 the pre-clip
    global norm goes into metrics['gradnorms/_overall']."""
    store = optimizer.store
    world = dist.world if dist is not None else 1
    pending = []
    if optimizer.clip_norm > 0.0:  # local clip needs the complete local gradient first: no bucket overlap
        model.backward(d_hidden_state=d_hidden_state)
        metrics["gradnorms/_overall"] = optimizer.clip_gradients()
        if world > 1:
            dist.all_reduce_grads(store.g)
        optimizer.apply_gradients(grad_scale=1.0 / world, skip=skip, zero_grad=True)
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

        model.backward(on_non_vit_grads_ready=on_rest, vit_layer_groups=groups, on_vit_group_done=on_group,
                       d_hidden_state=d_hidden_state)
        dist.reserve_sms(False)
        vit_pending.append(dist.all_reduce_ranges_async(store.g, vit_ranges[-1]))
        dist.wait_all(pending)
        optimizer.apply_gradients(grad_scale=1.0 / world, skip=skip, zero_grad=True, only=store.rest_ranges, advance=False)
        for k, hs in enumerate(vit_pending):
            dist.wait_all(hs)
            optimizer.apply_gradients(grad_scale=1.0 / world, skip=skip, zero_grad=True, only=vit_ranges[k],
                                      advance=(k + 1 == len(vit_pending)))
    else:
        model.backward(d_hidden_state=d_hidden_state)
        optimizer.apply_gradients(grad_scale=1.0 / world, skip=skip, zero_grad=True)


def model_fn_builder(config: NeatConfig, *, store: Optional[ParamStore] = None, dist: Optional[DataParallel] = None,
                     device="cuda", seed: int = 0, log_attention_probs: bool = True, vit_grad_buckets: int = 4):
    """model/modeling.py:671-810.  `seed` is the run seed of every random draw of the step (dropout masks, Gumbel noise,
    span lengths, 10/80/10 options, replacement ids): replica r at step t uses seed + t*world + r, so replicas draw
    independently like the reference's per-core tf.random ops and two runs with different seeds differ.
    `log_attention_probs` defaults to the reference's model_fn (modeling.py:691-709 computes attn/* every step)."""
    if store is None:
        store = ParamStore(config.model, device=device, optimizer_cfg=config.optimizer)
        store.init_reference(seed=0)
    optimizer, _ = build_optimizer_from_config(loss=None, optimizer_config=config.optimizer, device_config=config.device,
                                               store=store)

    def model_fn(features, labels=None, mode="train", params=None):
        is_training = mode == "train"
        imgs = features["images"]
        if is_training and config.model.get("transpose_input", False) and imgs.shape[-1] != 3:
            imgs = imgs.permute(3, 0, 1, 2).contiguous()  # [H,W,3,N] -> [N,H,W,3], modeling.py:683-685
        model = MerlotModel(config=config.model, is_training=True,  # the reference hard-codes True (:693, SURVEY quirk 3)
                            image=imgs, input_ids=features["input_ids"], use_tpu=config.device.get("use_tpu", False),
                            shuffled_idx_img=features.get("shuffled_idx_img", None), mask_input=True, params=store,
                            dropout_seed=seed + store.global_step * (dist.world if dist is not None else 1) +
                            (dist.rank if dist is not None else 0), dist=dist, log_attention_probs=log_attention_probs)
        lang_loss, lang_losses = model.mask_loss()
        contr_loss, contr_losses = model.contrastive_loss()
        skip = []
        if config.model.get("temporal_coef", 1.0) > 0.0:
            temp_loss, temp_losses = model.temporal_loss(features["shuffled_idx_img"], video_src_ids=features["video_src_ids"])
            if not config.model.get("image_shuffle_prob", 0) > 0:
                skip = [n for n in store.entries if n.startswith("viz_viz_temporal/")]
        else:
            temp_loss, temp_losses = torch.zeros((), device=store.device), {}
            skip = [n for n in store.entries if "_temporal/" in n]
        losses = {f"lang/{k}": v for k, v in lang_losses.items()}
        losses.update({f"contr/{k}": v for k, v in contr_losses.items()})
        losses.update({f"temporal/{k}": v for k, v in temp_losses.items()})
        losses["learning_rate"] = optimizer.current_lr()
        if log_attention_probs:  # modeling.py:709  losses.update(model.attention_log)
            losses.update({f"attn/{k}": v for k, v in model.attention_log.items()})

        def train_op():
            backward_and_apply(model, optimizer, dist, metrics=losses, skip=skip, vit_grad_buckets=vit_grad_buckets)

        return StepSpec(model, (lang_loss, contr_loss, temp_loss), losses, train_op)

    model_fn.store = store
    model_fn.optimizer = optimizer
    return model_fn


def _step_for(config: NeatConfig):
    """(model_fn_builder, synthetic batch) of the configured task: downstream.task 'vcr' fine-tunes on VCR
    (downstream/vcr/train.py), anything else pretrains (model/train.py)."""
    if config.downstream.get("task") == "vcr":
        from .vcr import vcr_model_fn_builder
        return vcr_model_fn_builder, synthetic_vcr_batch
    return model_fn_builder, synthetic_batch


def main(argv=None):
    """`python -m merlot_b200.train configs/merlot.yaml` (or merlot_vcr.yaml) -- the role of model/train.py:9-26 and
    downstream/vcr/train.py on synthetic data."""
    config = NeatConfig.from_args("Train MERLOT (H100-native)", argv=argv)
    dist = DataParallel() if int(os.environ.get("WORLD_SIZE", "1")) > 1 else None
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    builder, make_batch = _step_for(config)
    model_fn = builder(config, dist=dist)
    per_rank = max(1, config.device.get("train_batch_size", 8) // (dist.world if dist else 1))
    for step in range(config.optimizer.get("num_train_steps", 10)):
        feats = make_batch(config, per_rank, seed=step + (dist.rank if dist else 0) * 100003)
        spec = model_fn(feats, None, "train", None)
        spec.train_op()
        if step % 10 == 0 and (dist is None or dist.rank == 0):
            print(f"step {step} loss {spec.loss:.4f} lr {spec.metrics['learning_rate']:.3e}", flush=True)


if __name__ == "__main__":
    main()
