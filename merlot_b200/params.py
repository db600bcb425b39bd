"""Parameter arena: every trainable variable of the reference (SURVEY.md Appendix A) in ONE flat fp32 master buffer, with
matching flat buffers for the fp32 gradients (the NCCL all-reduce bucket), the Adam moments -- bf16 first moment and
sign-packed bf16 second moment with use_bfloat16_adam (utils/optimization.py:371-383), fp32 both without it, the
reference's default (:305) -- and the bf16 compute copy (bfloat16_getter, utils/model_utils.py:572-602).  Layout in HBM:
[hyper-parameter group 0 | group 1 | ...], each variable padded to 64 elements so every slice is 256-byte (fp32) / 128-byte
(bf16) aligned and usable as a TMA base.

Storage differs from the TF variables in three places (converted by load_tf_dict / to_tf_dict):
  * query/key/value kernels [H,H] x3 are fused into `.../qkv/kernel` [H,3H] (and biases into [3H]);
  * dense layers with fewer than 8 outputs (the temporal `logits` [H,4], VCR's `classifier_mlp1` [H/2,1]) are zero-padded
    to 8 columns so their rows are 16-byte aligned for TMA; `Entry.ref_cols` records how many columns the reference has;
  * the patch conv kernel [P,P,3,H] is stored as the im2col matrix [P*P*3, H] (same memory order).

`task` selects the variable set of one reference graph: "pretrain" (model/modeling.py model_fn, every head), "vcr"
(downstream/vcr/modeling.py model_fn: MerlotModel(mask_input=False) + the answer / rationale classifier towers) or
"video_mc" (multiple-choice video QA, merlot_b200/video_mc.py: the VCR graph's model variables + one `mc_cls` tower of the
answer tower's shapes and initialisers) or "video_qa" (open-ended video QA, merlot_b200/video_qa.py: the VCR graph's model
variables + one `qa_cls` tower whose output layer has A = `num_answers` columns, zero-padded to a multiple of 8) or
"video_fib" (fill-in-the-blank video QA, merlot_b200/video_fib.py: the VCR graph's model variables + the pretraining MLM
head's `lm_head/projection` and `lm_head/LayerNorm` (with do_projection) + a `fib_cls/answers` dense layer of A columns,
zero-padded as video_qa's, whose initial values derive_fib_answers computes from the word embeddings).  In pretraining,
`share_params: False` gives the language-only pass its own `langonly_encoder/` stack of num_lang_transformer_hidden_layers
layers beside the joint `encoder/`; the VCR and video_mc graphs have no language-only pass and ignore it (as do video_qa's
and video_fib's).

save_checkpoint / restore_checkpoint write and read the whole training state (parameters, Adam slots, global_step) as the
TensorFlow V2 checkpoints the reference's Estimator keeps in output_dir.
"""
from __future__ import annotations

import math
import os
import re
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from .stem import stem_ops

PAD = 64
TEMPORAL_PAD_N = 8
TASKS = ("pretrain", "vcr", "video_mc", "video_qa", "video_fib")
ANSWER_TASKS = ("video_qa", "video_fib")  # the tasks whose store holds an answer vocabulary of num_answers
VCR_TOWERS = ("answer_cls", "rationale_cls")
VIDEO_MC_TOWERS = ("mc_cls",)
VIDEO_QA_TOWER = "qa_cls"
VIDEO_FIB_ANSWERS = "fib_cls/answers"
VCR_BIAS_PI = 0.25  # cls_head(hidden_state, bias_pi=0.25), downstream/vcr/modeling.py:77


@dataclass
class Entry:
    name: str
    shape: Tuple[int, ...]
    tf_names: Tuple[str, ...]   # reference variable name(s) this entry stores
    offset: int = 0
    numel: int = 0
    padded: int = 0
    hyper: Tuple = ()
    ref_cols: int = 0           # > 0: the last dim is zero-padded; the reference variable has this many columns


def padded_answers(num_answers: int) -> int:
    """A8: the columns of an answer layer (video_qa's tower output, video_fib's fib_cls/answers), num_answers rounded up to
    a multiple of 8 (16-byte rows)."""
    return (num_answers + TEMPORAL_PAD_N - 1) // TEMPORAL_PAD_N * TEMPORAL_PAD_N


def derive_fib_answers(store: "ParamStore", answer_tokens, output_bias: Optional[torch.Tensor] = None) -> None:
    """Write video_fib's answer layer from the MLM head's output layer: column a of fib_cls/answers/kernel is the mean of
    the word-embedding rows (store.P, fp32) of answer a's token ids, bias[a] the mean of `output_bias` [vocab_size] at those
    ids (lm_head/output_bias of a checkpoint; None: zero, the reference's do_bias: False).  Means are taken in float64 and
    rounded to fp32; the padding columns are zero.  For a one-token answer this is that token's MLM logit exactly.  Then
    refreshes the bf16 copy.  Runs once, when a store is set up; the layer is its own variable afterwards."""
    if store.task != "video_fib":
        raise ValueError(f"the fill-in-the-blank answer layer lives in a ParamStore(task='video_fib'), got {store.task!r}")
    A = store.num_answers
    if len(answer_tokens) != A:
        raise ValueError(f"{len(answer_tokens)} answers given, the store holds {A}")
    dev = store.device
    tokens = torch.tensor([t for toks in answer_tokens for t in toks], dtype=torch.int64, device=dev)
    seg = torch.repeat_interleave(torch.arange(A, device=dev), torch.tensor([len(t) for t in answer_tokens], device=dev))
    count = torch.bincount(seg, minlength=A).to(torch.float64)
    with torch.no_grad():
        emb = store.P("word_embeddings/word_embeddings")
        kern = torch.zeros((A, emb.shape[1]), dtype=torch.float64, device=dev).index_add_(0, seg, emb[tokens].double())
        store.P(f"{VIDEO_FIB_ANSWERS}/kernel").zero_()[:, :A] = (kern / count[:, None]).float().t()
        bias = store.P(f"{VIDEO_FIB_ANSWERS}/bias").zero_()
        if output_bias is not None:
            ob = output_bias.to(device=dev, dtype=torch.float64).reshape(-1)
            bias[:A] = (torch.zeros(A, dtype=torch.float64, device=dev).index_add_(0, seg, ob[tokens]) / count).float()
    store.sync_bf16()


def _entries(cfg: dict, task: str = "pretrain", num_answers: int = 0) -> List[Entry]:
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    P = cfg["patch_size"]
    out: List[Entry] = []

    def add(name, shape, tf_names=None, ref_cols=0):
        out.append(Entry(name, tuple(shape), tuple(tf_names) if tf_names else (name,), ref_cols=ref_cols))

    def ln(scope):
        add(f"{scope}/gamma", (H,))
        add(f"{scope}/beta", (H,))

    def lin(scope, i, o):
        add(f"{scope}/kernel", (i, o))
        add(f"{scope}/bias", (o,))

    def stack(scope, n):
        for l in range(n):
            ls = f"{scope}/layer{l:02d}"
            ln(f"{ls}/LayerNorm_attn_ln0")
            add(f"{ls}/qkv/kernel", (H, 3 * H), [f"{ls}/{x}/kernel" for x in ("query_layer", "key_layer", "value_layer")])
            add(f"{ls}/qkv/bias", (3 * H,), [f"{ls}/{x}/bias" for x in ("query_layer", "key_layer", "value_layer")])
            lin(f"{ls}/context_projection_layer", H, H)
            ln(f"{ls}/LayerNorm_mlp_ln0")
            lin(f"{ls}/intermediate", H, I)
            lin(f"{ls}/output", I, H)
        ln(f"{scope}/LayerNorm_ln_final")

    vt = "vision_backbone/vision_transformer"
    resnet_layers = list(cfg.get("resnet_layers", []) or [])
    if not resnet_layers:
        add(f"{vt}/conv2d/kernel", (P * P * 3, H))
        add(f"{vt}/conv2d/bias", (H,))
    else:
        for nm, shp in stem_variables(vt, resnet_layers, 64, H):  # conv kernels stored [kh*kw*cin, cout] (flattened HWIO)
            add(nm, shp if len(shp) == 1 else (shp[0] * shp[1] * shp[2], shp[3]))
    add(f"{vt}/pos_embs/pos_embs", (64 * 64, H))
    add(f"{vt}/pos_embs/cls_emb", (cfg.get("num_cls_emb", 2), H))
    ln(f"{vt}/LayerNorm_ctx_patches_pre_ln")
    stack(vt, cfg.get("num_vision_transformer_hidden_layers", cfg["num_hidden_layers"]))
    add("vision_backbone/img_idx_pe", (cfg.get("max_vision_pos_embeddings", 1024), H))
    add("vision_backbone/final_pe/pos_embs", (64 * 64, H))
    add("vision_backbone/final_pe/cls_emb", (1, H))
    ln("vision_backbone/LayerNorm_final_ln")
    add("word_embeddings/word_embeddings", (V, H))
    if task in ("vcr", "video_mc", "video_qa", "video_fib"):  # mask_input=False: no language-only encoder, no masking
        add("position_embeddings/position_embeddings", (cfg["max_position_embeddings"], H))
        ln("position_embeddings/LayerNorm_embed_norm")
        stack("encoder", cfg["num_hidden_layers"])
        if task == "video_fib":  # the MLM head's projection (model/modeling.py:205-224), then dense(A) stored as A8 columns
            if cfg.get("do_projection", False):
                lin("lm_head/projection", H, H)
                ln("lm_head/LayerNorm")
            A8 = padded_answers(num_answers)
            add(f"{VIDEO_FIB_ANSWERS}/kernel", (H, A8), ref_cols=num_answers)
            add(f"{VIDEO_FIB_ANSWERS}/bias", (A8,), ref_cols=num_answers)
            return out
        if task == "video_qa":  # dense(H/2) + gelu, then dense(A) stored as A8 columns
            lin(f"{VIDEO_QA_TOWER}/classifier_mlp0", H, H // 2)
            A8 = padded_answers(num_answers)
            add(f"{VIDEO_QA_TOWER}/classifier_mlp1/kernel", (H // 2, A8), ref_cols=num_answers)
            add(f"{VIDEO_QA_TOWER}/classifier_mlp1/bias", (A8,), ref_cols=num_answers)
            return out
        # VCR: downstream/vcr/modeling.py:86-121, in creation order; video_mc: one tower of VCR's shapes over C candidates
        for tower in (VCR_TOWERS if task == "vcr" else VIDEO_MC_TOWERS):
            lin(f"{tower}/classifier_mlp0", H, H // 2)
            add(f"{tower}/classifier_mlp1/kernel", (H // 2, TEMPORAL_PAD_N), ref_cols=1)
            add(f"{tower}/classifier_mlp1/bias", (TEMPORAL_PAD_N,), ref_cols=1)
        return out
    for sc in ("position_embeddings", "langonly_embeddings"):
        add(f"{sc}/position_embeddings", (cfg["max_position_embeddings"], H))
        ln(f"{sc}/LayerNorm_embed_norm")
    if cfg.get("share_params", True):  # one stack for both text passes, deep enough for either (model/modeling.py:171-172)
        stack("encoder", max(cfg["num_hidden_layers"], cfg.get("num_lang_transformer_hidden_layers", 0)))
    else:  # langonly_reps builds its own stack (:356-379); after the ViT in every group, so it stays in rest_ranges
        stack("encoder", cfg["num_hidden_layers"])
        stack("langonly_encoder", cfg["num_lang_transformer_hidden_layers"])
    if cfg.get("do_projection", False):
        lin("lm_head/projection", H, H)
        ln("lm_head/LayerNorm")
    if cfg.get("do_bias", False):
        add("lm_head/output_bias", (V,))
    Cs = cfg.get("contrastive_size", H)
    for t in ("lang", "viz"):
        if cfg.get("do_projection", False):
            lin(f"contrastive/{t}_proj_intermediate", H, Cs)
            add(f"contrastive/LayerNorm_{t}_proj_ln/gamma", (Cs,))
            add(f"contrastive/LayerNorm_{t}_proj_ln/beta", (Cs,))
        lin(f"contrastive/{t}_proj", Cs if cfg.get("do_projection", False) else H, Cs)
    for t in ("lang_viz", "viz_viz"):
        lin(f"{t}_temporal/intermediate", 2 * H, H)
        ln(f"{t}_temporal/LayerNorm_ln0")
        add(f"{t}_temporal/logits/kernel", (H, TEMPORAL_PAD_N), ref_cols=4)
        add(f"{t}_temporal/logits/bias", (TEMPORAL_PAD_N,), ref_cols=4)
    return out


def stem_variables(scope: str, layers, width: int, hidden: int):
    """Variables of the hybrid ResNet-lite stem in the reference's creation order (stem.stem_ops), then the 1x1
    conv_postresnet_proj (utils/vision_transformer.py:213-223).  Returns (name, TF shape) pairs with conv kernels HWIO."""
    out, cin = [], width
    for op in stem_ops(scope, tuple(layers), width):
        if op.kind == "conv":
            out.append((op.name, (op.k, op.k, op.cin, op.cout)))
            cin = op.cout
        elif op.kind == "gn":
            out += [(f"{op.name}/gamma", (op.cout,)), (f"{op.name}/beta", (op.cout,))]
    out.append((f"{scope}/conv_postresnet_proj/kernel", (1, 1, cin, hidden)))
    out.append((f"{scope}/conv_postresnet_proj/bias", (hidden,)))
    return out


_CONV_KERNEL = re.compile(r"/(conv2d(_\d+)?|conv_postresnet_proj)/kernel$")


def hyper_for(tf_name: str, optimizer_cfg: dict) -> Tuple[float, float, float, float, float]:
    """(learning_rate, weight_decay_rate, beta_1, beta_2, epsilon) after the regex overrides of
    utils/optimization.py:125-147 (re.search on the variable name; later rules update earlier ones)."""
    hp = {
        "learning_rate": optimizer_cfg["learning_rate"],
        "weight_decay_rate": optimizer_cfg.get("weight_decay_rate", 1e-4),
        "beta_1": 0.9,  # hard-coded, optimization.py:185
        "beta_2": optimizer_cfg.get("beta_2", 0.98),
        "epsilon": optimizer_cfg.get("epsilon", 1e-6),
    }
    overrides = list(optimizer_cfg.get("param_overrides", None) or [])
    if optimizer_cfg.get("freeze_scope") is not None:  # :128-131
        overrides.append([[f"^{optimizer_cfg['freeze_scope']}"], {"learning_rate": 0}])
    for regexes, over in overrides:
        for k in over:
            if k not in ("learning_rate", "weight_decay_rate", "beta_1", "beta_2", "epsilon", "do_factor"):
                raise ValueError("Regex rule {} -> {} isn't OK because {} isn't a changable optimization parameter".format(
                    regexes, over, k))
        for regex in regexes:
            if re.search(regex, tf_name) is not None:
                hp.update({k: v for k, v in over.items() if k in hp})
    return (hp["learning_rate"], hp["weight_decay_rate"], hp["beta_1"], hp["beta_2"], hp["epsilon"])


class ParamStore:
    """Flat arenas + named views.  `optimizer_cfg` fixes the hyper-parameter grouping (needed only for training) and the
    Adam moments' storage: fp32 unless it sets use_bfloat16_adam (the reference's default is False); without an
    optimizer_cfg the moments are bf16.  `num_answers` (tasks "video_qa" and "video_fib" only, >= 2) is the answer
    vocabulary's size A."""

    def __init__(self, model_cfg: dict, device="cuda", optimizer_cfg: Optional[dict] = None, with_optimizer_state=True,
                 task: str = "pretrain", num_answers: Optional[int] = None):
        # resnet_layers != [] selects the hybrid ResNet-lite stem (utils/vision_transformer.py:206-223); forward and backward
        # are provided (K13), its variables follow the reference's creation order (stem_variables).
        if task not in TASKS:
            raise ValueError(f"ParamStore task must be one of {TASKS}, got {task!r}")
        if (task in ANSWER_TASKS) != (num_answers is not None):
            raise ValueError(f"num_answers is the size of the {task if task in ANSWER_TASKS else 'video_qa'} answer "
                             f"vocabulary: task={task!r}, num_answers={num_answers!r}")
        if task in ANSWER_TASKS and int(num_answers) < 2:
            raise ValueError(f"{task}: num_answers must be >= 2, got {num_answers}")
        self.cfg = model_cfg
        self.task = task
        self.num_answers = None if num_answers is None else int(num_answers)
        self.device = torch.device(device)
        ents = _entries(model_cfg, task, self.num_answers or 0)
        ocfg = optimizer_cfg or {"learning_rate": 0.0, "param_overrides": [
            [["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]]}
        for e in ents:
            hs = {hyper_for(t, ocfg) for t in e.tf_names}
            if len(hs) != 1:
                raise NotImplementedError(f"param_overrides treat the fused tensors {e.tf_names} differently")
            e.hyper = hs.pop()
            e.numel = math.prod(e.shape)
            e.padded = (e.numel + PAD - 1) // PAD * PAD
        groups: Dict[Tuple, List[Entry]] = {}
        for e in ents:
            groups.setdefault(e.hyper, []).append(e)
        self.entries: Dict[str, Entry] = {}
        self.groups: List[Tuple[Tuple, int, int]] = []  # (hyper, offset, count)
        off = 0
        for hyper, es in sorted(groups.items(), key=lambda kv: -kv[0][1]):
            start = off
            for e in es:
                e.offset = off
                off += e.padded
                self.entries[e.name] = e
            self.groups.append((hyper, start, off - start))
        self.total = off
        # contiguous [ViT | everything else] split of every group: the non-ViT gradients are final before the ViT backward
        # starts, so their all-reduce can overlap it (train.DataParallel)
        self.vit_ranges, self.rest_ranges = [], []
        for _, goff, gcnt in self.groups:
            ends = [e.offset + e.padded for e in self.entries.values()
                    if goff <= e.offset < goff + gcnt and e.name.startswith("vision_backbone/vision_transformer/")]
            vend = max(ends) if ends else goff
            if vend > goff:
                self.vit_ranges.append((goff, vend))
            if goff + gcnt > vend:
                self.rest_ranges.append((vend, goff + gcnt))
        self.p = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.g = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.pb = torch.zeros(off, dtype=torch.bfloat16, device=self.device)
        use_bf16_adam = optimizer_cfg is None or bool(optimizer_cfg.get("use_bfloat16_adam", False))
        self.moment_dtype = torch.bfloat16 if use_bf16_adam else torch.float32
        if with_optimizer_state:
            self.m = torch.zeros(off, dtype=self.moment_dtype, device=self.device)
            self.v = torch.zeros(off, dtype=self.moment_dtype, device=self.device)
        self.g_acc: Optional[torch.Tensor] = None  # grad_accumulator(): allocated by the first clipped accumulated step
        self.global_step = 0

    def grad_accumulator(self) -> torch.Tensor:
        """The second fp32 gradient arena, in g's layout, of a step with clip_norm > 0 over A > 1 micro-batches: it sums the
        micro-batches' clipped gradients (optimization.AdamOptimizer.clip_accumulate), and the all-reduce and AdamW read it.
        The backward pass keeps writing g, so no captured gradient pointer moves.  Allocated at first use (4 B per
        parameter); zero between steps."""
        if self.g_acc is None:
            self.g_acc = torch.zeros_like(self.g)
        return self.g_acc

    def vit_buckets(self, n_groups: int = 4):
        """Gradient buckets of the ViT for the data-parallel all-reduce, in BACKWARD order.  Returns (layer_groups, ranges):
        layer_groups[k] = (lo, hi) layers walked by the k-th partial stack backward (top-down); ranges[k] = arena ranges whose
        gradients are final once group k has run.  The weight-decayed kernels of a layer group are contiguous in the arena;
        everything else of the ViT (patch/stem kernels, position tables, every LayerNorm and bias) rides in the last bucket."""
        vt = "vision_backbone/vision_transformer/"
        layers = self.cfg.get("num_vision_transformer_hidden_layers", self.cfg["num_hidden_layers"])
        n_groups = max(1, min(n_groups, layers))
        cuts = [round(layers * k / n_groups) for k in range(n_groups + 1)]
        groups = [(cuts[k], cuts[k + 1]) for k in range(n_groups)][::-1]
        ranges, taken = [], []
        for lo, hi in groups[:-1]:
            es = [e for e in self.entries.values() if e.name.startswith(vt + "layer") and e.name.endswith("/kernel")
                  and lo <= int(e.name[len(vt) + 5:len(vt) + 7]) < hi]
            a, b = min(e.offset for e in es), max(e.offset + e.padded for e in es)
            assert sum(e.padded for e in es) == b - a, "ViT layer kernels are not contiguous in the arena"
            ranges.append([(a, b)])
            taken.append((a, b))
        last = []
        for a, b in self.vit_ranges:  # whatever the earlier buckets left
            cur = a
            for ta, tb in sorted(taken):
                if tb <= cur or ta >= b:
                    continue
                if ta > cur:
                    last.append((cur, ta))
                cur = max(cur, tb)
            if cur < b:
                last.append((cur, b))
        ranges.append(last)
        return groups, ranges

    # ---- views ----
    def _view(self, buf: torch.Tensor, name: str) -> torch.Tensor:
        e = self.entries[name]
        return buf[e.offset:e.offset + e.numel].view(e.shape)

    def P(self, name):
        return self._view(self.p, name)

    def G(self, name):
        return self._view(self.g, name)

    def W(self, name):  # bf16 compute copy
        return self._view(self.pb, name)

    def num_params(self) -> int:
        """Trainable scalars as the reference counts them (padding and the zero-padded columns excluded)."""
        n = 0
        for e in self.entries.values():
            n += e.numel if not e.ref_cols else e.numel // e.shape[-1] * e.ref_cols
        return n

    def sync_bf16(self):
        """bf16 compute copy <- fp32 master (one pass; afterwards the fused AdamW keeps it current)."""
        if self.device.type != "cuda":
            self.pb.copy_(self.p.to(torch.bfloat16))
        else:
            ops.cast_f32_to_bf16(self.p, self.pb)

    # ---- interop with the reference's variable names ----
    def load_tf_dict(self, d: Dict[str, torch.Tensor], strict: bool = True):
        """Copy reference-named variables into the arena.  strict=False applies the reference's init-from-checkpoint rule
        (utils/model_utils.py:388-413): a variable is restored iff the checkpoint has it, everything else keeps its current
        value; returns the list of entries that were NOT found."""
        missing = []
        with torch.no_grad():
            for e in self.entries.values():
                if not strict and not all(t in d for t in e.tf_names):
                    missing.append(e.name)
                    continue
                dst = self.P(e.name)
                if len(e.tf_names) == 3:
                    src = torch.cat([d[t] for t in e.tf_names], dim=-1)
                elif e.ref_cols:
                    src = torch.zeros(e.shape, dtype=torch.float32)
                    src[..., :e.ref_cols] = d[e.tf_names[0]]
                else:
                    src = d[e.tf_names[0]].reshape(e.shape)
                dst.copy_(src.to(torch.float32))
        self.sync_bf16()
        return missing

    def load_checkpoint(self, prefix: str):
        """`init_checkpoint` (model/modeling.py:724-740): restore by name from a TensorFlow V2 checkpoint prefix."""
        from .tf_checkpoint import load_checkpoint
        return self.load_tf_dict(load_checkpoint(prefix), strict=False)

    def tf_views(self, buf: torch.Tensor) -> List[Tuple[Entry, str, torch.Tensor]]:
        """(entry, reference name, view of `buf` in the reference variable's shape) for every reference variable, in arena
        entry order: q/k/v split into column views, zero-padded columns (`ref_cols`) left out, conv kernels HWIO, position
        tables [1, 64, 64, H], CLS embeddings [1, n, H].  `buf` is any arena (p, g, m, v); views may be non-contiguous."""
        out = []
        for e in self.entries.values():
            t = self._view(buf, e.name)
            if len(e.tf_names) == 3:
                out.extend((e, nm, part) for nm, part in zip(e.tf_names, t.chunk(3, dim=-1)))
                continue
            if e.ref_cols:
                t = t[..., :e.ref_cols]
            elif e.name.endswith("vision_transformer/conv2d/kernel"):
                Pp = self.cfg["patch_size"]
                t = t.reshape(Pp, Pp, 3, -1)
            elif _CONV_KERNEL.search(e.name):  # hybrid stem: [kh*kw*cin, cout] -> HWIO
                kh = {n_: s_ for n_, s_ in stem_variables("vision_backbone/vision_transformer", self.cfg["resnet_layers"], 64,
                                                          self.cfg["hidden_size"])}[e.name][0]
                t = t.reshape(kh, kh, t.shape[0] // (kh * kh), -1)
            elif e.name.endswith("/pos_embs"):
                t = t.reshape(1, 64, 64, -1)
            elif e.name.endswith("/cls_emb"):
                t = t.reshape(1, t.shape[0], -1)
            out.append((e, e.tf_names[0], t))
        return out

    def to_tf_dict(self, which: str = "p") -> Dict[str, torch.Tensor]:
        buf = {"p": self.p, "g": self.g}[which]
        return {nm: t.detach().float().cpu().contiguous() for _, nm, t in self.tf_views(buf)}

    # ---- full training state as a TensorFlow V2 checkpoint ----
    def slot_entries(self, skip=()) -> List[Entry]:
        """Entries whose reference variables own Adam slots (`<name>/adam_m`, `<name>/adam_v`).  The reference's
        apply_gradients creates them for every variable it updates (utils/optimization.py:339-383): a trainable variable --
        not in a learning-rate-0 group, those are removed from tvars (:149-156) -- whose gradient is not None (:343-344).
        `skip` names the entries whose gradient is None in the training graph (the training step's `skip` list)."""
        skip = set(skip)
        unknown = skip - set(self.entries)
        if unknown:
            raise KeyError(f"skip names entries the store does not have: {sorted(unknown)}")
        return [e for e in self.entries.values() if e.hyper[0] != 0 and e.name not in skip]

    def _checkpoint_tensors(self, skip):
        """(name, TF dtype, device view) of every variable of a checkpoint of this store, in data-file order: global_step,
        the fp32 parameters, then the slots -- bf16 or fp32 as the moments are stored (every offset stays a multiple of
        its element size)."""
        from .tf_checkpoint import DT_BFLOAT16, DT_FLOAT
        if not hasattr(self, "m"):
            raise ValueError("checkpoints hold the optimizer state: build the ParamStore with with_optimizer_state=True")
        slots = {e.name for e in self.slot_entries(skip)}
        views = self.tf_views(self.p)
        out = [(nm, DT_FLOAT, t) for _, nm, t in views]
        slot_dt = DT_FLOAT if self.moment_dtype == torch.float32 else DT_BFLOAT16
        for suffix, buf in (("adam_m", self.m), ("adam_v", self.v)):
            out += [(f"{nm}/{suffix}", slot_dt, t) for e, nm, t in self.tf_views(buf) if e.name in slots]
        return out

    def save_checkpoint(self, prefix: str, skip=()) -> Dict[str, float]:
        """Write the training state as the TensorFlow V2 checkpoint `prefix` (model.ckpt-<step> of the reference's Estimator):
        every variable under its reference name (as to_tf_dict maps it), the `adam_m` / `adam_v` slots of slot_entries(skip)
        bit for bit (bf16 and sign-packed bf16, or fp32 both, as the store keeps them), and `global_step` (int64).  The
        data file is gathered on the device, checksummed there by one K15 launch, copied to pinned host memory at once and
        written by tf_checkpoint.write_bundle.  Extra device memory: one buffer of the data file's size.  Returns the seconds each phase took and the bytes written."""
        import time
        from .tf_checkpoint import DT_INT64, write_bundle
        t0 = time.perf_counter()
        tensors = [("global_step", DT_INT64, torch.tensor(self.global_step, dtype=torch.int64, device=self.device))]
        tensors += self._checkpoint_tensors(skip)
        sizes = [t.numel() * t.element_size() for _, _, t in tensors]
        offs = [0]
        for s in sizes:
            offs.append(offs[-1] + s)
        stage = torch.empty(offs[-1], dtype=torch.uint8, device=self.device)
        for (_, _, t), o, s in zip(tensors, offs, sizes):
            stage[o:o + s].view(t.dtype).view(t.shape).copy_(t)
        torch.cuda.synchronize(self.device)
        t1 = time.perf_counter()
        crcs = ops.crc32c_multi([stage[o:o + s] for o, s in zip(offs, sizes)])
        t2 = time.perf_counter()
        host = torch.empty(offs[-1], dtype=torch.uint8, pin_memory=True)
        host.copy_(stage)
        del stage
        t3 = time.perf_counter()
        arr = host.numpy()
        write_bundle(prefix, [(nm, dt, tuple(t.shape), arr[o:o + s], c)
                              for (nm, dt, t), o, s, c in zip(tensors, offs, sizes, crcs)])
        t4 = time.perf_counter()
        return {"stage_s": t1 - t0, "crc_s": t2 - t1, "d2h_s": t3 - t2, "write_s": t4 - t3, "bytes": float(offs[-1])}

    def restore_checkpoint(self, prefix: str, skip=()) -> None:
        """Restore p, m, v and global_step from a checkpoint written by save_checkpoint (or by the reference's Saver), then
        refresh the bf16 copy.  The data file is copied to the device whole and every tensor's CRC-32C is checked there (K15);
        a mismatch raises CheckpointFormatError naming the tensor.  Like Saver.restore, a variable or slot this store needs
        that the checkpoint lacks raises, as does a shape or dtype mismatch; variables the store does not have are ignored.
        Padding columns and padding elements restore as zero; slots of variables outside slot_entries(skip) restore as zero.
        (load_checkpoint is the other operation: init_checkpoint's restore-by-name of model variables.)"""
        import numpy as np
        from .tf_checkpoint import DT_BFLOAT16, DT_FLOAT, DT_INT64, CheckpointFormatError, _index, mask_crc
        slot_flag = {DT_BFLOAT16: True, DT_FLOAT: False}  # slot dtype -> the use_bfloat16_adam that writes it
        header, entries = _index(prefix, True)
        want = [("global_step", DT_INT64, None)] + self._checkpoint_tensors(skip)
        missing = [nm for nm, _, _ in want if nm not in entries]
        if missing:
            raise CheckpointFormatError(f"{prefix}: {len(missing)} variables the store needs are not in the checkpoint: "
                                        f"{', '.join(missing[:8])}{' ...' if len(missing) > 8 else ''}")
        for nm, dt, t in want:
            e = entries[nm]
            shape = [] if t is None else list(t.shape)
            if int(e["dtype"]) != dt or [int(d) for d in e["shape"]] != shape:
                msg = f"{nm}: checkpoint has dtype {e['dtype']} shape {e['shape']}, the store needs dtype {dt} shape {shape}"
                if nm.endswith(("/adam_m", "/adam_v")) and int(e["dtype"]) != dt and int(e["dtype"]) in slot_flag:
                    msg += (f"; the checkpoint was written with use_bfloat16_adam: {slot_flag[int(e['dtype'])]}, this store "
                            f"keeps its moments for use_bfloat16_adam: {slot_flag[dt]} (slots are not converted)")
                raise CheckpointFormatError(msg)
            if e["slices"]:
                raise NotImplementedError(f"{nm}: partitioned (sliced) variables are not supported")
        if header["num_shards"] != 1 or any(int(e["shard_id"]) for e in entries.values()):
            raise NotImplementedError(f"{prefix}: sharded checkpoints are not supported")
        path = f"{prefix}.data-00000-of-00001"
        size = os.path.getsize(path)
        for nm, e in entries.items():
            if int(e["offset"]) < 0 or int(e["size"]) < 0 or int(e["offset"]) + int(e["size"]) > size:
                raise CheckpointFormatError(f"{nm}: data shard is shorter than the index says")
        host = torch.empty(size, dtype=torch.uint8, pin_memory=True)
        with open(path, "rb") as f:
            if f.readinto(memoryview(host.numpy())) != size:
                raise CheckpointFormatError(f"{path}: short read")
        data = host.to(self.device)
        checked = sorted((nm, e) for nm, e in entries.items() if e["crc32c"] is not None)
        crcs = ops.crc32c_multi([data[int(e["offset"]):int(e["offset"]) + int(e["size"])] for _, e in checked])
        for (nm, e), c in zip(checked, crcs):
            if mask_crc(c) != e["crc32c"]:
                raise CheckpointFormatError(f"{nm}: tensor checksum mismatch")
        with torch.no_grad():
            for buf in (self.p, self.m, self.v):
                buf.zero_()
            for nm, _, t in want[1:]:
                o, s = int(entries[nm]["offset"]), int(entries[nm]["size"])
                src = data[o:o + s]
                if o % t.element_size():
                    src = src.clone()
                t.copy_(src.view(t.dtype).view(t.shape))
        o = int(entries["global_step"]["offset"])
        self.global_step = int(np.frombuffer(host.numpy()[o:o + 8].tobytes(), dtype="<i8")[0])
        self.sync_bf16()

    def init_reference(self, seed: int = 0):
        """Reference initialisers (truncated normal 0.02 / variance-scaling patch kernel / LN 1,0 / zero biases; the VCR
        towers' output bias is -log((1 - pi) / pi), downstream/vcr/modeling.py:71, and so is video_mc's; video_qa's output
        bias stays zero, so that no answer is favoured)."""
        g = torch.Generator().manual_seed(seed)
        std = self.cfg.get("initializer_range", 0.02)
        with torch.no_grad():
            for e in self.entries.values():
                leaf = e.name.rsplit("/", 1)[-1]
                if leaf == "gamma":
                    t = torch.ones(e.shape)
                elif leaf in ("beta", "bias", "output_bias"):
                    t = torch.zeros(e.shape)
                    if e.name.endswith("_cls/classifier_mlp1/bias") and not e.name.startswith(VIDEO_QA_TOWER + "/"):
                        t[0] = -math.log((1 - VCR_BIAS_PI) / VCR_BIAS_PI)
                else:
                    s_ = std
                    if _CONV_KERNEL.search(e.name):  # tf.variance_scaling_initializer(): fan_in = kh*kw*cin = rows of the 2-D view
                        s_ = math.sqrt(1.0 / e.shape[0]) / 0.87962566103423978
                    t = torch.empty(e.shape)
                    torch.nn.init.trunc_normal_(t, 0.0, s_, -2 * s_, 2 * s_, generator=g)
                    if e.ref_cols:
                        t[:, e.ref_cols:] = 0
                self.P(e.name).copy_(t)
        self.sync_bf16()
