"""Parameter arena: every trainable variable of the reference (SURVEY.md Appendix A) in ONE flat fp32 master buffer, with
matching flat buffers for the fp32 gradients (the NCCL all-reduce bucket), the bf16 Adam first moment, the sign-packed
bf16 second moment (utils/optimization.py:371-383) and the bf16 compute copy (bfloat16_getter,
utils/model_utils.py:572-602).  Layout in HBM: [hyper-parameter group 0 | group 1 | ...], each variable padded to 64
elements so every slice is 256-byte (fp32) / 128-byte (bf16) aligned and usable as a TMA base.

Storage differs from the TF variables in three places (converted by load_tf_dict / to_tf_dict):
  * query/key/value kernels [H,H] x3 are fused into `.../qkv/kernel` [H,3H] (and biases into [3H]);
  * dense layers with fewer than 8 outputs (the temporal `logits` [H,4], VCR's `classifier_mlp1` [H/2,1]) are zero-padded
    to 8 columns so their rows are 16-byte aligned for TMA; `Entry.ref_cols` records how many columns the reference has;
  * the patch conv kernel [P,P,3,H] is stored as the im2col matrix [P*P*3, H] (same memory order).

`task` selects the variable set of one reference graph: "pretrain" (model/modeling.py model_fn, every head) or "vcr"
(downstream/vcr/modeling.py model_fn: MerlotModel(mask_input=False) + the answer / rationale classifier towers).
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from . import ops

PAD = 64
TEMPORAL_PAD_N = 8
TASKS = ("pretrain", "vcr")
VCR_TOWERS = ("answer_cls", "rationale_cls")
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


def _entries(cfg: dict, task: str = "pretrain") -> List[Entry]:
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
    if task == "vcr":  # mask_input=False: no language-only encoder, no masking, no pretraining heads
        add("position_embeddings/position_embeddings", (cfg["max_position_embeddings"], H))
        ln("position_embeddings/LayerNorm_embed_norm")
        stack("encoder", cfg["num_hidden_layers"])
        for tower in VCR_TOWERS:  # downstream/vcr/modeling.py:86-121, in creation order
            lin(f"{tower}/classifier_mlp0", H, H // 2)
            add(f"{tower}/classifier_mlp1/kernel", (H // 2, TEMPORAL_PAD_N), ref_cols=1)
            add(f"{tower}/classifier_mlp1/bias", (TEMPORAL_PAD_N,), ref_cols=1)
        return out
    for sc in ("position_embeddings", "langonly_embeddings"):
        add(f"{sc}/position_embeddings", (cfg["max_position_embeddings"], H))
        ln(f"{sc}/LayerNorm_embed_norm")
    stack("encoder", max(cfg["num_hidden_layers"], cfg.get("num_lang_transformer_hidden_layers", 0)))
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
    """Variables of the hybrid ResNet-lite stem in the reference's creation order (utils/vision_transformer.py:69-170,213-223;
    names per SURVEY.md Appendix A: conv2d, conv2d_1, ... / GroupNorm, GroupNorm_1, ... uniquified inside each variable scope).
    Yields (name, TF shape) with conv kernels HWIO."""
    out = []

    class _Scope:
        def __init__(self, s):
            self.s, self.nc, self.ng = s, 0, 0

        def conv(self, kh, cin, cout):
            out.append((f"{self.s}/conv2d{'' if self.nc == 0 else '_%d' % self.nc}/kernel", (kh, kh, cin, cout)))
            self.nc += 1

        def gn(self, c, name=None):
            base = f"{self.s}/GroupNorm_{name}" if name is not None else f"{self.s}/GroupNorm{'' if self.ng == 0 else '_%d' % self.ng}"
            if name is None:
                self.ng += 1
            out.append((f"{base}/gamma", (c,)))
            out.append((f"{base}/beta", (c,)))

    st = _Scope(f"{scope}/resnet50lite/stem")
    for i, (cin, cout) in enumerate(((3, width // 2), (width // 2, width // 2), (width // 2, width))):
        st.conv(3, cin, cout)
        st.gn(cout, f"stem{i}")
    cin = width
    for i, blocks in enumerate(layers):
        f = width * (2 ** i)
        bg = _Scope(f"{scope}/resnet50lite/block_group{i + 1}")
        for b in range(blocks):
            if b == 0:  # projection shortcut is created first (:77-85)
                bg.conv(1, cin, 4 * f)
                bg.gn(4 * f)
            bg.conv(1, cin, f)
            bg.gn(f)
            bg.conv(3, f, f)
            bg.gn(f)
            bg.conv(1, f, 4 * f)
            bg.gn(4 * f)
            cin = 4 * f
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
    """Flat arenas + named views.  `optimizer_cfg` fixes the hyper-parameter grouping (needed only for training)."""

    def __init__(self, model_cfg: dict, device="cuda", optimizer_cfg: Optional[dict] = None, with_optimizer_state=True,
                 task: str = "pretrain"):
        # resnet_layers != [] selects the hybrid ResNet-lite stem (utils/vision_transformer.py:206-223); forward and backward
        # are provided (K13), its variables follow the reference's creation order (stem_variables).
        if task not in TASKS:
            raise ValueError(f"ParamStore task must be one of {TASKS}, got {task!r}")
        self.cfg = model_cfg
        self.task = task
        self.device = torch.device(device)
        ents = _entries(model_cfg, task)
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
        if with_optimizer_state:
            self.m = torch.zeros(off, dtype=torch.bfloat16, device=self.device)
            self.v = torch.zeros(off, dtype=torch.bfloat16, device=self.device)
        self.global_step = 0

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

    def to_tf_dict(self, which: str = "p") -> Dict[str, torch.Tensor]:
        buf = {"p": self.p, "g": self.g}[which]
        out = {}
        for e in self.entries.values():
            t = self._view(buf, e.name).detach().float().cpu()
            if len(e.tf_names) == 3:
                for nm, part in zip(e.tf_names, t.chunk(3, dim=-1)):
                    out[nm] = part.contiguous()
            elif e.ref_cols:
                out[e.tf_names[0]] = t[..., :e.ref_cols].contiguous()
            elif e.name.endswith("vision_transformer/conv2d/kernel"):
                Pp = self.cfg["patch_size"]
                out[e.tf_names[0]] = t.reshape(Pp, Pp, 3, -1)
            elif _CONV_KERNEL.search(e.name):  # hybrid stem: [kh*kw*cin, cout] -> HWIO
                kh = {n_: s_ for n_, s_ in stem_variables("vision_backbone/vision_transformer", self.cfg["resnet_layers"], 64,
                                                          self.cfg["hidden_size"])}[e.name][0]
                out[e.tf_names[0]] = t.reshape(kh, kh, t.shape[0] // (kh * kh), -1)
            elif e.name.endswith("/pos_embs"):
                out[e.tf_names[0]] = t.reshape(1, 64, 64, -1)
            elif e.name.endswith("/cls_emb"):
                out[e.tf_names[0]] = t.reshape(1, t.shape[0], -1)
            else:
                out[e.tf_names[0]] = t
        return out

    def init_reference(self, seed: int = 0):
        """Reference initialisers (truncated normal 0.02 / variance-scaling patch kernel / LN 1,0 / zero biases; the VCR
        towers' output bias is -log((1 - pi) / pi), downstream/vcr/modeling.py:71)."""
        g = torch.Generator().manual_seed(seed)
        std = self.cfg.get("initializer_range", 0.02)
        with torch.no_grad():
            for e in self.entries.values():
                leaf = e.name.rsplit("/", 1)[-1]
                if leaf == "gamma":
                    t = torch.ones(e.shape)
                elif leaf in ("beta", "bias", "output_bias"):
                    t = torch.zeros(e.shape)
                    if e.name.endswith("_cls/classifier_mlp1/bias"):
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
