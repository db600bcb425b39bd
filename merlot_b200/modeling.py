"""Host-side mirror of the reference's `MerlotModel` (model/modeling.py:47-668) over the sm_90a C-ABI.

Same constructor arguments, attributes and methods as the reference class, so `model_fn`-style callers
(model/modeling.py:691-713, downstream/sort_story/get_zero_shot_logits.py:58-79) read the same.  Construction *is* the
forward pass (the reference builds the TF graph there).  Differences forced by leaving TF1:
  * variables live in a `ParamStore` passed as `params=` (the reference keeps them in the TF graph);
  * random draws that the reference takes from tf.random.* are injectable (`mask_draws=`, `dropout_seed=`);
  * the backward pass is explicit: `model.backward()` after the three loss methods (reference: tf.gradients,
    utils/optimization.py:176).
Every tensor is a CUDA tensor; all arithmetic runs in libmerlot_b200.so -- PyTorch only owns memory and streams.
There is no CPU fallback: without the library (or without a GPU) construction raises.
"""
from __future__ import annotations

import copy
import ctypes as C
import math
import os
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L
from . import ops
from .params import ParamStore
from .stem import HybridStem

MASK = 1  # utils/encode/encoder.py:16-22
PADDING = 0
START = 2

_SITE_VIT, _SITE_LANGONLY, _SITE_JOINT, _SITE_EMB_LO, _SITE_EMB_J = 0, 100, 200, 300, 301
# VCR classifier towers (merlot_b200/vcr.py cls_head): dropout of each tower's input and of its hidden layer
_SITE_VCR_ANS_IN, _SITE_VCR_ANS_HID, _SITE_VCR_RAT_IN, _SITE_VCR_RAT_HID = 400, 401, 402, 403
# the multiple-choice video QA tower (merlot_b200/video_mc.py mc_head): dropout of its input and of its hidden layer
_SITE_MC_IN, _SITE_MC_HID = 410, 411
# the open-ended video QA tower (merlot_b200/video_qa.py qa_head): dropout of its input and of its hidden layer
_SITE_QA_IN, _SITE_QA_HID = 420, 421
_VIT = "vision_backbone/vision_transformer"


def get_shape_list_rank(t: torch.Tensor, expected_rank, name="tensor"):
    """utils/model_utils.py:29-56 assert_rank: ValueError on rank mismatch."""
    ranks = expected_rank if isinstance(expected_rank, (list, tuple)) else [expected_rank]
    if t.dim() not in ranks:
        raise ValueError("For the tensor `%s`, the actual rank `%d` (shape = %s) is not equal to the expected rank `%s`" %
                         (name, t.dim(), str(tuple(t.shape)), str(expected_rank)))
    return list(t.shape)


class _Buffers:
    """Named device buffers cached on the ParamStore so pointers stay stable across steps (CUDA-graph friendly)."""

    def __init__(self, store: ParamStore):
        if not hasattr(store, "_bufs"):
            store._bufs = {}
        self.d = store._bufs
        self.dev = store.device

    def get(self, name, shape, dtype, zero=False):
        key = (name, tuple(shape), dtype)
        t = self.d.get(key)
        if t is None:
            t = torch.zeros(shape, dtype=dtype, device=self.dev) if zero else torch.empty(shape, dtype=dtype, device=self.dev)
            self.d[key] = t
        elif zero:
            t.zero_()
        return t


class _LayerNorm:
    """LayerNorm `scope` of the rows of x into y (ops.layernorm_fwd), keeping the input and statistics its backward reads.
    Keyword arguments of forward / backward override the ones given here (rows, remap, dropout)."""

    def __init__(self, store, scope, x, mean, rstd, **kw):
        self.st, self.scope, self.x, self.mean, self.rstd, self.kw = store, scope, x, mean, rstd, kw

    def forward(self, y, **kw):
        st, s = self.st, self.scope
        return ops.layernorm_fwd(self.x, y, st.P(f"{s}/gamma"), st.P(f"{s}/beta"), self.mean, self.rstd, **{**self.kw, **kw})

    def backward(self, dy, dx, **kw):
        st, s = self.st, self.scope
        return ops.layernorm_bwd(dy, self.x, self.mean, self.rstd, st.P(f"{s}/gamma"), dx, st.G(f"{s}/gamma"), st.G(f"{s}/beta"),
                                 **{**self.kw, **kw})


class _Dense:
    """tf.layers.dense `scope` on a small head tensor: bf16 rows x, fp32 accumulate and output (+bias).  Keeps x for its
    backward; `tag` names the backward's buffers."""

    def __init__(self, store, bufs, tag, scope, x):
        self.st, self.bf, self.tag, self.scope, self.x = store, bufs, tag, scope, x

    def forward(self, out):
        st, s = self.st, self.scope
        return ops.gemm(self.x, st.W(f"{s}/kernel"), b_mn_major=True, bias=st.P(f"{s}/bias"), out=out)

    def backward(self, dy):
        """Accumulates the kernel and bias gradients of dy fp32 [R, N]; returns d_x fp32 [R, Kin]."""
        st, bf, s = self.st, self.bf, self.scope
        (R, N), Kin = dy.shape, self.x.shape[1]
        ops.bias_grad(dy, st.G(f"{s}/bias"), rows=R, N=N)
        dyb = bf.get(f"{self.tag}.dyb.{s}", (R, N), torch.bfloat16)
        ops.cast_f32_to_bf16(dy, dyb)
        ops.gemm(self.x, dyb, a_mn_major=True, b_mn_major=True, out=st.G(f"{s}/kernel"), atomic=True, M=Kin, N=N, K=R)
        dx = bf.get(f"{self.tag}.dx.{s}", (R, Kin), torch.float32)
        return ops.gemm(dyb, st.W(f"{s}/kernel"), out=dx, M=R, N=Kin, K=N)


class _MlpLn:
    """dense + gelu -> layer_norm of bf16 rows x (the heads' repeated pattern, e.g. :28-35, :208-215, :582-589), run at
    construction: bf16 output `out` [R, Hout]."""

    def __init__(self, store, bufs, tag, x, dense_scope, ln_scope, Hout):
        R = x.shape[0]
        self.bf, self.tag = bufs, tag
        self.dense = _Dense(store, bufs, tag, dense_scope, x)
        self.pre = self.dense.forward(bufs.get(f"{tag}.pre", (R, Hout), torch.float32))
        act = ops.gelu_f32(self.pre, bufs.get(f"{tag}.act", (R, Hout), torch.float32))
        self.out = bufs.get(f"{tag}.an", (R, Hout), torch.bfloat16)
        self.ln = _LayerNorm(store, ln_scope, act, bufs.get(f"{tag}.mean", (R,), torch.float32),
                             bufs.get(f"{tag}.rstd", (R,), torch.float32), rows=R)
        self.ln.forward(self.out)

    def backward(self, d_out):
        """d_out fp32 [R, Hout] -> parameter gradients accumulated, d_x fp32 [R, Hin] returned."""
        bf, tag = self.bf, self.tag
        d_act = self.ln.backward(d_out, bf.get(f"{tag}.d_act", self.pre.shape, torch.float32))
        d_pre = ops.gelu_bwd_f32(d_act, self.pre, bf.get(f"{tag}.d_pre", self.pre.shape, torch.float32))
        return self.dense.backward(d_pre)


class _SoftmaxCE:
    """Softmax cross entropy of fp32 logits [R, >= C] against int32 labels (ops.softmax_ce_fwd), reduced by ops.weighted_loss
    with the caller's weights, nz_labels, denom_mode and scale into `out2` = (loss, accuracy; the accuracy only with
    accuracy=True).  Keeps what its backward reads; `tag` names its buffers."""

    def __init__(self, bufs, tag, logits, labels, C, weights=None, nz_labels=None, denom_mode=0, scale=1.0, accuracy=False):
        R = logits.shape[0]
        self.logits, self.labels, self.C = logits, labels, C
        per, self.lse = bufs.get(f"{tag}.l", (R,), torch.float32), bufs.get(f"{tag}.lse", (R,), torch.float32)
        corr = bufs.get(f"{tag}.corr", (R,), torch.float32) if accuracy else None
        ops.softmax_ce_fwd(logits, labels, C, per, self.lse, corr)
        self.out2, self.coeff = bufs.get(f"{tag}.out", (2,), torch.float32), bufs.get(f"{tag}.coeff", (R,), torch.float32)
        ops.weighted_loss(per, corr, weights, nz_labels, denom_mode, scale, self.out2, self.coeff)

    def backward(self, dlogits):
        ops.softmax_ce_bwd(self.logits, self.labels, self.C, self.lse, self.coeff, dlogits)
        return dlogits


class _Tower:
    """project_and_norm (:18-44) of fp32 rows x [n, H] under scope 'contrastive', run at construction: l2-normalised fp32
    features `feat` [n, Cs]."""

    def __init__(self, store, bufs, cfg, tag, x, name):
        self.n, H = x.shape
        self.Cs = cfg.get("contrastive_size", H)
        self.bf, self.tag = bufs, tag
        xb = ops.cast_f32_to_bf16(x, bufs.get(f"{tag}.xb", (self.n, H), torch.bfloat16))
        self.inter = None
        if cfg.get("do_projection", False):
            self.inter = _MlpLn(store, bufs, f"{tag}.inter", xb, f"contrastive/{name}_intermediate",
                                f"contrastive/LayerNorm_{name}_ln", self.Cs)
        self.dense = _Dense(store, bufs, tag, f"contrastive/{name}", self.inter.out if self.inter else xb)
        proj = self.dense.forward(bufs.get(f"{tag}.proj", (self.n, self.Cs), torch.float32))
        self.feat = bufs.get(f"{tag}.feat", (self.n, self.Cs), torch.float32)
        self.inv = bufs.get(f"{tag}.inv", (self.n,), torch.float32)
        ops.l2norm_fwd(proj, self.feat, self.inv)

    def backward(self, d_feat):
        d_proj = self.bf.get(f"{self.tag}.d_proj", (self.n, self.Cs), torch.float32)
        ops.l2norm_bwd(d_feat, self.feat, self.inv, d_proj)
        d_in = self.dense.backward(d_proj)
        return self.inter.backward(d_in) if self.inter else d_in


def _layer_params(store: ParamStore, scope: str, layers: int):
    key = ("_lp", scope, layers)
    if key in store._bufs:
        return store._bufs[key]
    arr = (L.merlot_layer_params_t * layers)()
    for l in range(layers):
        ls = f"{scope}/layer{l:02d}"
        lp = arr[l]
        for field, name, bf in (("ln1_gamma", "LayerNorm_attn_ln0/gamma", 0), ("ln1_beta", "LayerNorm_attn_ln0/beta", 0),
                                ("w_qkv", "qkv/kernel", 1), ("b_qkv", "qkv/bias", 0),
                                ("w_o", "context_projection_layer/kernel", 1), ("b_o", "context_projection_layer/bias", 0),
                                ("ln2_gamma", "LayerNorm_mlp_ln0/gamma", 0), ("ln2_beta", "LayerNorm_mlp_ln0/beta", 0),
                                ("w_1", "intermediate/kernel", 1), ("b_1", "intermediate/bias", 0),
                                ("w_2", "output/kernel", 1), ("b_2", "output/bias", 0)):
            full = f"{ls}/{name}"
            setattr(lp, field, (store.W(full) if bf else store.P(full)).data_ptr())
            setattr(lp, "g_" + field, store.G(full).data_ptr())
    store._bufs[key] = arr
    return arr


def _grid_idxmap(bufs: _Buffers, nh: int, nw: int):
    key = ("_grid", nh, nw)
    if key not in bufs.d:
        i = torch.arange(nh, device=bufs.dev)[:, None]
        j = torch.arange(nw, device=bufs.dev)[None]
        bufs.d[key] = (i * 64 + j).reshape(-1).to(torch.int32)
    return bufs.d[key]


class _Stack:
    """One transformer stack invocation (utils/transformer.py:171-247) through merlot_stack_forward/backward."""

    def __init__(self, store, bufs, tag, scope, layers, B, S, valid, h_in, cfg, dropout_p, seed, site, save, colsum=None,
                 colsum2=None, colsum_split=0, colsum_valid_q=0, probs=None, pair=(0, 0), probs_layer_mean=False):
        """probs: f32 [layers, B, S, S] of every layer's head-mean attention map, or with probs_layer_mean one [B, S, S]
        that receives their mean over layers."""
        H, I, heads = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_attention_heads"]
        if H % heads != 0 or H // heads != 64:
            raise ValueError("passed in a tensor of shape {} when size_per_head={} and num_attention_heads={}".format(
                (B * S, H), H // max(heads, 1), heads) + " (this build provides size_per_head=64 only)")
        d = L.merlot_stack_t()
        d.B, d.S, d.H, d.I, d.heads, d.layers = B, S, H, I, heads, layers
        self._lp = _layer_params(store, scope, layers)
        d.layer_params = C.addressof(self._lp)
        fg, fb = f"{scope}/LayerNorm_ln_final/gamma", f"{scope}/LayerNorm_ln_final/beta"
        d.final_gamma, d.final_beta = store.P(fg).data_ptr(), store.P(fb).data_ptr()
        d.d_final_gamma, d.d_final_beta = store.G(fg).data_ptr(), store.G(fb).data_ptr()
        d.valid = valid.data_ptr() if valid is not None else None
        d.h_in = h_in.data_ptr()
        self.y = bufs.get(f"{tag}.y", (B * S, H), torch.bfloat16)
        d.y = self.y.data_ptr()
        d.save_for_backward = int(save)
        d.hidden_dropout_p = float(dropout_p)
        d.attention_dropout_p = float(cfg.get("attention_probs_dropout_prob", 0.0) or 0.0)
        d.dropout_seed, d.dropout_site_base = seed, site
        self.arena = bufs.get(f"{tag}.act", (L.lib().merlot_stack_activation_bytes(C.byref(d)),), torch.uint8)
        d.act_arena = self.arena.data_ptr()
        d.attn_colsum = colsum.data_ptr() if colsum is not None else None
        d.attn_colsum2 = colsum2.data_ptr() if colsum2 is not None else None
        d.attn_colsum_split, d.attn_colsum_valid_q = int(colsum_split), int(colsum_valid_q)
        d.attn_probs = probs.data_ptr() if probs is not None else None
        d.attn_probs_layer_mean = int(probs_layer_mean)
        d.pair_viz_len, d.pair_chunk_len = int(pair[0]), int(pair[1])  # disable_pairwise_lang_attn (model/modeling.py:160-168)
        self.d, self.bufs, self.tag, self.keep = d, bufs, tag, (valid, h_in, colsum, probs)

    def forward(self):
        L.lib().merlot_stack_forward(C.byref(self.d), ops._stream())
        return self.y

    def backward(self, dy, dh_in, layer_groups=None, on_group_done=None):
        """layer_groups = [(lo, hi), ...] top-down (hi of the first = layers, lo of the last = 0): one C call per group, with
        on_group_done(k) in between -- the parameter gradients of group k are final when its kernels have run."""
        d = self.d
        scratch = self.bufs.get(f"{self.tag}.scratch", (L.lib().merlot_stack_scratch_bytes(C.byref(d)),), torch.uint8)
        d.dy, d.dh_in, d.scratch = dy.data_ptr(), dh_in.data_ptr(), scratch.data_ptr()
        if not layer_groups:
            d.bwd_lo, d.bwd_hi = 0, 0
            L.lib().merlot_stack_backward(C.byref(d), ops._stream())
            return dh_in
        assert layer_groups[0][1] == d.layers and layer_groups[-1][0] == 0
        for k, (lo, hi) in enumerate(layer_groups):
            d.bwd_lo, d.bwd_hi = lo, hi
            L.lib().merlot_stack_backward(C.byref(d), ops._stream())
            if on_group_done is not None:
                on_group_done(k)
        d.bwd_lo, d.bwd_hi = 0, 0
        return dh_in


class _Embedding:
    """embed_words (:262-297) of int32 ids [G, Lseq] into the rows of `out` through `remap`, run at construction."""

    def __init__(self, store, bufs, cfg, tag, scope, ids, out, remap, dropout):
        R, Lseq = ids.numel(), ids.shape[1]
        if Lseq > cfg["max_position_embeddings"]:  # tf.assert_less_equal, utils/model_utils.py:282
            raise ValueError(f"sequence length {Lseq} exceeds max_position_embeddings {cfg['max_position_embeddings']}")
        self.st, self.bf, self.tag, self.scope, self.ids = store, bufs, tag, scope, ids
        xsum = bufs.get(f"{tag}.xsum", (R, cfg["hidden_size"]), torch.float32)
        ops.embed_fwd(ids, store.P("word_embeddings/word_embeddings"), store.P(f"{scope}/position_embeddings"), xsum, Lseq)
        self.ln = _LayerNorm(store, f"{scope}/LayerNorm_embed_norm", xsum, bufs.get(f"{tag}.mean", (R,), torch.float32),
                             bufs.get(f"{tag}.rstd", (R,), torch.float32), rows=R, remap=remap, dropout=dropout)
        self.ln.forward(out)

    def backward(self, dy):
        st, (G, Lseq) = self.st, self.ids.shape
        dx = self.ln.backward(dy, self.bf.get(f"bwd.dxsum.{self.tag}", self.ln.x.shape, torch.float32))
        ops.scatter_add_rows(dx, self.ids.reshape(-1), st.G("word_embeddings/word_embeddings"))
        ops.group_rowsum(dx, G, Lseq, 0, Lseq, None, st.G(f"{self.scope}/position_embeddings"), dx.shape[1])


class _VitInput:
    """The ViT input (utils/vision_transformer.py:189-232) of NHWC bf16 images, run at construction: the patch conv2d, or the
    hybrid stem (:206-223) and its 1x1 conv_postresnet_proj; cls / position embeddings; the pre-LN into bf16 `out`."""

    def __init__(self, store, bufs, cfg, img, save):
        N, h0, w0, _ = img.shape
        H, Pp, ncls, resnet_layers = cfg["hidden_size"], cfg["patch_size"], cfg.get("num_cls_emb", 2), cfg.get("resnet_layers")
        self.st, self.bf, self.N, self.h1, self.w1, self.ncls = store, bufs, N, h0 // Pp, w0 // Pp, ncls
        Mp, Mv = N * self.h1 * self.w1, N * (self.h1 * self.w1 + ncls)
        patch = bufs.get("vit.patch", (Mp, H), torch.float32)
        self.stem = None
        if not resnet_layers:
            self.proj, self.a = f"{_VIT}/conv2d", bufs.get("vit.A", (Mp, Pp * Pp * 3), torch.bfloat16)
            ops.patch_im2col(img, self.a, Pp)
        else:  # the stem, then conv_postresnet_proj: 1x1 with bias, not weight-standardised
            if Pp != 16:
                raise ValueError("the hybrid ResNet stem needs patch_size 16 (utils/vision_transformer.py:208)")
            self.proj, self.stem = f"{_VIT}/conv_postresnet_proj", HybridStem(store, bufs, list(resnet_layers), save)
            self.a, hs, ws_ = self.stem.forward(img, N, h0, w0)
            if (hs, ws_) != (self.h1, self.w1):
                raise ValueError(f"stem output {hs}x{ws_} != patch grid {self.h1}x{self.w1}")
        ops.gemm(self.a, store.W(f"{self.proj}/kernel"), b_mn_major=True, bias=store.P(f"{self.proj}/bias"), out=patch)
        xsum = bufs.get("vit.xsum", (Mv, H), torch.float32)
        ops.vit_assemble_fwd(patch, store.P(f"{_VIT}/pos_embs/pos_embs"), store.P(f"{_VIT}/pos_embs/cls_emb"), xsum, N, self.h1,
                             self.w1, ncls, H)
        self.out = bufs.get("vit.h0", (Mv, H), torch.bfloat16)
        self.ln = _LayerNorm(store, f"{_VIT}/LayerNorm_ctx_patches_pre_ln", xsum, bufs.get("vit.mean0", (Mv,), torch.float32),
                             bufs.get("vit.rstd0", (Mv,), torch.float32))
        self.ln.forward(self.out)

    def backward(self, dy):
        """dy: bf16 gradient of `out`.  Returns the gradient HybridStem.backward took (bf16, shaped as its output) or None."""
        st, bf, N, ncls, H, np_ = self.st, self.bf, self.N, self.ncls, dy.shape[1], self.h1 * self.w1
        dx = self.ln.backward(dy, bf.get("bwd.dxsum_v", self.ln.x.shape, torch.float32))
        ops.group_rowsum(dx, N, np_ + ncls, 0, ncls, None, st.G(f"{_VIT}/pos_embs/cls_emb"), H)
        ops.group_rowsum(dx, N, np_ + ncls, ncls, np_, _grid_idxmap(bf, self.h1, self.w1), st.G(f"{_VIT}/pos_embs/pos_embs"), H)
        dpatch = bf.get("bwd.dpatch", (N * np_, H), torch.bfloat16)
        ops.vit_assemble_bwd(dx, dpatch, N, np_, ncls, H)
        ops.bias_grad(dpatch, st.G(f"{self.proj}/bias"), rows=N * np_, N=H)
        ops.gemm(self.a, dpatch, a_mn_major=True, b_mn_major=True, out=st.G(f"{self.proj}/kernel"), atomic=True,
                 M=self.a.shape[1], N=H, K=N * np_)
        if self.stem is not None:
            d_rc = bf.get("bwd.d_rc", self.a.shape, torch.bfloat16)
            ops.gemm(dpatch, st.W(f"{self.proj}/kernel"), out=d_rc)  # [M, H] . [Cr, H]^T
            self.stem.backward(d_rc)
            return d_rc


class _VizTokens:
    """The viz tokens (:95-133) of the ViT output hv on the patch grid geom = (N, h1, w1, ncls, sp), run at construction: for
    each of the nc frame copies, viz_assemble_fwd, then LayerNorm_final_ln into the joint-input rows of each of its nt texts."""

    def __init__(self, store, bufs, hv, img_idx, joint_in, geom, Pz, Sj, nt, nc):
        N, H, Bi = geom[0], hv.shape[1], joint_in.shape[0] // (Sj * nt * nc)  # Bi image groups
        self.st, self.bf, self.img_idx, self.geom = store, bufs, img_idx, geom
        # joint-input rows of copy d, text j (model/modeling.py:111-119): image group g's Pz rows at (g*nc*nt + d*nt + j) * Sj
        self.remaps = [[(Pz, nt * nc * Sj, (d * nt + j) * Sj) for j in range(nt)] for d in range(nc)]
        xsum = bufs.get("viz.xsum", (Bi * Pz, H), torch.float32)
        self.img_trg = bufs.get("viz.img_trg", (N, H), torch.float32)
        self.ln = _LayerNorm(store, "vision_backbone/LayerNorm_final_ln", xsum, bufs.get("viz.mean", (Bi * Pz,), torch.float32),
                             bufs.get("viz.rstd", (Bi * Pz,), torch.float32), rows=Bi * Pz)
        for d in range(nc):  # copy d of image group g: its own image indices, joint rows of group g*nc + d
            idx_d = img_idx if img_idx.numel() == N else img_idx.view(Bi, nc, -1)[:, d].contiguous()
            ops.viz_assemble_fwd(hv, store.P("vision_backbone/img_idx_pe"), idx_d, store.P("vision_backbone/final_pe/pos_embs"),
                                 store.P("vision_backbone/final_pe/cls_emb"), xsum, self.img_trg, *geom, H)
            for remap in self.remaps[d]:
                self.ln.forward(joint_in, remap=remap)

    def backward(self, d_joint_in, d_img_trg):
        """The gradient of the one frame copy a backward allows (nc == 1); returns d_hv bf16, shaped as hv."""
        st, bf, (N, h1, w1, ncls, sp), H = self.st, self.bf, self.geom, d_img_trg.shape[1]
        dx = None
        for j, remap in enumerate(self.remaps[0]):  # the nt texts of an image group all send gradient into its viz tokens
            dx = self.ln.backward(d_joint_in, bf.get(f"bwd.dxsum_z.{j & 1}", self.ln.x.shape, torch.float32), dres=dx, remap=remap)
        d_hv = bf.get("bwd.d_hv", (N * (h1 * w1 + ncls), H), torch.bfloat16)
        ops.viz_assemble_bwd(dx, d_img_trg, d_hv, *self.geom, H)
        h2, w2 = h1 // sp, w1 // sp
        ops.segment_rowsum_scatter(dx, N, h2 * w2 + 1, self.img_idx, st.G("vision_backbone/img_idx_pe"), H)
        ops.group_rowsum(dx, N, h2 * w2 + 1, 0, 1, None, st.G("vision_backbone/final_pe/cls_emb"), H)
        ops.group_rowsum(dx, N, h2 * w2 + 1, 1, h2 * w2, _grid_idxmap(bf, h2, w2), st.G("vision_backbone/final_pe/pos_embs"), H)
        return d_hv


class _LangOnly:
    """langonly_reps (:339-379) of model.input_ids with hidden dropout p, run at construction: the ids regrouped by
    langonly_num_chunks_in_group, _Embedding, _Stack, and each chunk's first row gathered into fp32 `lang_trg`.  The stack is
    the joint encoder's `encoder/` variables with share_params (the default), its own `langonly_encoder/` without
    (:356-362)."""

    def __init__(self, model, p):
        cfg, st, bf, Lc, nch = model.config, model.store, model._bufs, model.lang_chunk_length, model.num_chunks
        layers = cfg["num_lang_transformer_hidden_layers"]
        scope = "encoder" if cfg.get("share_params", True) else "langonly_encoder"
        need = [f"{scope}/layer{l:02d}/qkv/kernel" for l in range(layers)] + [f"{scope}/LayerNorm_ln_final/gamma"]
        if any(n not in st.entries for n in need):
            raise ValueError(f"share_params: {cfg.get('share_params', True)} runs the language-only encoder on {scope}/ "
                             f"({layers} layers), but the ParamStore has no such stack: build it from a config with the "
                             f"same share_params and num_lang_transformer_hidden_layers")
        g = cfg.get("langonly_num_chunks_in_group", nch)
        assert nch // g > 0 and nch % g == 0
        ids = model.input_ids.reshape(-1, Lc * g).contiguous()
        (Blo, Llo), H = ids.shape, model.hidden_size
        h0 = bf.get("lo.h0", (Blo * Llo, H), torch.bfloat16)
        self.emb = _Embedding(st, bf, cfg, "emb_lo", "langonly_embeddings", ids, h0, (0, 0, 0), (p, model._seed, _SITE_EMB_LO))
        valid = bf.get("lo.valid", (Blo * Llo,), torch.uint8)
        ops.ids_valid(ids, valid)
        summ = bf.get("lo.attn_summ", (Blo * Llo,), torch.float32, zero=True)
        probs = bf.get("lo.probs", (layers, Blo, Llo, Llo), torch.float32) if model._export_probs else None
        self.stack = _Stack(st, bf, "lo", scope, layers, Blo, Llo, valid, h0, cfg, p, model._seed, _SITE_LANGONLY,
                            model._save_arenas, colsum=summ, probs=probs)
        y = self.stack.forward()
        self.bf, nrows = bf, model.batch_size * nch
        self.pool_idx = bf.get("lo.pool_idx", (nrows,), torch.int32)
        self.pool_idx.copy_(torch.arange(nrows, dtype=torch.int32, device=st.device) * Lc)
        self.lang_trg = bf.get("lo.lang_trg", (nrows, H), torch.float32)
        ops.gather_rows(y, self.pool_idx, self.lang_trg)
        # lang_transformer_info; attention_summs of mask_inputs (:428-431): sum over (layers, queries) of head-mean probs, [B, L]
        self.info = {"hidden_state": y.view(Blo, Llo, H), "attention_summs": summ.view(model.B, model.L)}
        if probs is not None:
            self.info["self_attn_probs"] = probs.permute(1, 0, 2, 3)

    def backward(self, d_lang_trg):
        d_y = self.bf.get("bwd.d_ylo", self.stack.y.shape, torch.bfloat16, zero=True)
        ops.scatter_add_rows(d_lang_trg, self.pool_idx, d_y)
        d_h0 = self.bf.get("bwd.d_h0lo", self.stack.y.shape, torch.bfloat16)
        self.emb.backward(self.stack.backward(d_y, d_h0))


def check_num_imgs(cfg, batch_size, num_chunks, B, n_images, img_mask=None, mask_input=False, shuffled_idx_img=None,
                   frame_copies=1):
    """The several-images-per-text input of model/modeling.py:106-122 (`num_imgs` = ni, `img_mask`), checked on the host.
    B is the joint encoder's batch (MerlotModel.B).  Returns ni.  With ni > 1 the reshapes at :112 and :121 hold only for
    num_chunks == 1, and then `image` holds (batch_size // num_texts) * ni images, image group g = images g*ni .. g*ni+ni-1
    for texts g*nt .. g*nt+nt-1.  `img_mask` is any bool or integer tensor of B // num_texts * ni entries (:109); non-zero
    means valid.  Raises ValueError on shapes the reference cannot reshape, NotImplementedError on combinations
    the reference cannot run or that no program of it uses."""
    ni, nt = int(cfg.get("num_imgs", 1)), int(cfg.get("num_texts", 1))
    if ni < 1:
        raise ValueError(f"num_imgs must be >= 1, got {ni}")
    new_path = ni > 1 or img_mask is not None
    if not new_path:
        return ni
    if ni > 1 and shuffled_idx_img is not None:
        raise NotImplementedError("num_imgs > 1 with shuffled_idx_img: the reference asserts num_imgs == 1 there "
                                  "(model/modeling.py:319)")
    if mask_input:
        raise NotImplementedError("num_imgs > 1 / img_mask with mask_input=True: the pretraining heads index viz tokens through "
                                  "P (one image per chunk) and model_fn never passes an img_mask")
    if cfg.get("disable_pairwise_lang_attn", False):
        raise NotImplementedError("num_imgs > 1 / img_mask with disable_pairwise_lang_attn: the reference builds a P + L segment "
                                  "mask (model/modeling.py:162) for a P * num_imgs + L sequence")
    if frame_copies > 1:
        raise NotImplementedError("num_imgs > 1 / img_mask with frame_copies > 1 (the zero-shot story forward) is not provided")
    if not cfg.get("share_params", True):
        raise NotImplementedError("num_imgs > 1 / img_mask with share_params: False is not provided: the separate "
                                  "language-only encoder is a pretraining path and does not extend the multi-image input")
    max_vpe = int(cfg.get("max_vision_pos_embeddings", 1024))
    if ni > max_vpe:
        raise ValueError(f"num_imgs {ni} exceeds max_vision_pos_embeddings {max_vpe} (model/modeling.py:305-311)")
    if ni > 1:
        if num_chunks != 1:
            raise ValueError(f"num_imgs {ni} > 1 needs num_chunks == 1 (the reshapes at model/modeling.py:112,121), "
                             f"got num_chunks {num_chunks}")
        if batch_size % nt != 0 or n_images != (batch_size // nt) * ni:
            raise ValueError(f"image batch {n_images} != (batch_size {batch_size} // num_texts {nt}) x num_imgs {ni}"
                             + ("" if batch_size % nt == 0 else " (batch_size is not a multiple of num_texts)"))
    if img_mask is not None:
        if img_mask.dtype.is_floating_point or img_mask.dtype.is_complex:
            raise ValueError(f"img_mask must be a bool or integer tensor, got {img_mask.dtype}")
        want = B // nt * ni
        if B % nt != 0 or img_mask.numel() != want:
            raise ValueError(f"img_mask has {img_mask.numel()} entries (shape {tuple(img_mask.shape)}); it must reshape to "
                             f"[B // num_texts, num_imgs] = [{want // ni}, {ni}] (model/modeling.py:109)")
    return ni


class MerlotModel(object):
    def __init__(self, config, is_training, use_tpu, image, input_ids, mask_input=False, shuffled_idx_img=None,
                 img_mask=None, log_attention_probs=True, *, params: ParamStore, mask_draws: Optional[Dict] = None,
                 mask_override: Optional[Dict] = None, dropout_seed: int = 0, save_for_backward: Optional[bool] = None,
                 dist=None, export_attention_probs=False, frame_copies: int = 1, features_only: bool = False):
        """Arguments as model/modeling.py:48-66.  `use_tpu` is accepted and ignored (it only selects one-hot vs gather
        embedding lookups in the reference, utils/model_utils.py:259-263 -- same values either way).

        `frame_copies` = c > 1 is the evaluation forward of c copies of every group that share their frames (zero-shot story
        unshuffling scores two shuffles of each story, downstream/sort_story/get_zero_shot_logits.py:44-56): `image` holds
        batch_size // c groups of frames, `input_ids` and `shuffled_idx_img` hold batch_size groups, copy d of group s at
        s*c + d.  The ViT runs once per group of frames; each copy assembles its own viz tokens with its own image indices.

        `num_imgs` = ni > 1 in the config and `img_mask` (model/modeling.py:106-122) put several images before every text:
        `image` holds (batch_size // num_texts) * ni images, the joint sequence P * ni viz tokens then L language tokens, and
        an image masked in `img_mask` [B // num_texts, ni] drops out of the joint attention (check_num_imgs has the rules).

        `export_attention_probs` materialises the head-mean attention maps model_fn's PREDICT mode returns
        (model/modeling.py:762-770): True puts every layer's into encoder_info and lang_transformer_info['self_attn_probs'],
        [B, layers, S, S] each; "layer_mean" puts the joint encoder's mean over layers, [B, S, S], into encoder_info (the
        reduce_mean of :765, accumulated layer by layer in one buffer, so no per-layer buffer of the joint encoder exists)
        and keeps the language-only encoder's maps per layer, as the reference returns them.  With "layer_mean",
        attention_log is the reference's block sums of that map (:186-203) in a fixed summation order, so two runs on the
        same input give the same bits; otherwise it comes from K4's column sums, which add with float atomics.

        `features_only` runs what contrastive_features() needs and nothing more: the ViT, the language-only encoder and
        mask_inputs (with the dropout of is_training), but not the joint encoder, and it allows no backward.  The
        first pass of a gradient-accumulation step (train.model_fn_builder) computes every micro-batch's features this way."""
        frame_copies = int(frame_copies)
        if features_only and not mask_input:
            raise ValueError("features_only needs mask_input=True: the language features come from the language-only encoder")
        if features_only and save_for_backward:
            raise ValueError("features_only saves nothing for backward")
        self.features_only = bool(features_only)
        if features_only:
            save_for_backward = False
        if frame_copies < 1:
            raise ValueError(f"frame_copies must be >= 1, got {frame_copies}")
        if frame_copies > 1 and (is_training or mask_input or save_for_backward or config.get("num_texts", 1) > 1):
            raise NotImplementedError("frame_copies > 1 is an evaluation forward: it is not combined with training, "
                                      "save_for_backward, mask_input or num_texts > 1")
        self.frame_copies = frame_copies
        self.config = copy.deepcopy(config)
        self.is_training = is_training
        self.use_tpu = use_tpu
        self.store = params
        self.dist = dist
        cfg = self.config
        if not image.is_cuda or not input_ids.is_cuda:
            raise L.MerlotError(L.MERLOT_EINVAL, "MerlotModel needs CUDA tensors: merlot_b200 has no CPU fallback")
        if not cfg.get("use_bfloat16", False):
            raise NotImplementedError("use_bfloat16: False (fp32 activations) is not provided; every shipped config sets True")
        if cfg.get("num_texts", 1) > 1 and (mask_input or shuffled_idx_img is not None):
            raise NotImplementedError("num_texts > 1 (VCR, model/modeling.py:111-119) is a finetuning/inference path: mask_input and "
                                      "shuffled_idx_img are not combined with it in the reference either (:319-320)")

        input_ids_shape = get_shape_list_rank(input_ids, [2, 3], "input_ids")
        if len(input_ids_shape) == 2:  # :72-77
            self.num_chunks = 1
            self.num_chunks_in_group = 1
            self.batch_size, self.lang_chunk_length = input_ids_shape
            self.input_ids = input_ids[:, None]
        else:
            self.input_ids = input_ids
            self.batch_size, self.num_chunks, self.lang_chunk_length = input_ids_shape
            self.num_chunks_in_group = cfg.get("num_chunks_in_group", self.num_chunks)
            assert self.num_chunks % self.num_chunks_in_group == 0  # :82
        self.input_ids = self.input_ids.to(torch.int32).contiguous()
        self.num_imgs = check_num_imgs(cfg, self.batch_size, self.num_chunks, self.B, image.shape[0] if image.dim() == 4 else None,
                                       img_mask, mask_input, shuffled_idx_img, frame_copies)
        self.num_texts = cfg.get("num_texts", 1)
        self.img_batch_size = self.batch_size // self.num_texts
        if not is_training:  # :88-90
            cfg["hidden_dropout_prob"] = 0.0
            cfg["attention_probs_dropout_prob"] = 0.0
        self._save = bool(is_training) if save_for_backward is None else bool(save_for_backward)
        # features_only writes into the training forward's activation arenas (the next training forward overwrites them), so
        # that a features-only pass takes no memory of its own
        self._save_arenas = self._save or self.features_only
        self._seed = int(dropout_seed)
        self._bufs = _Buffers(params)
        self._mask_input = mask_input
        self._log_attention_probs = log_attention_probs
        # PREDICT-mode outputs of model_fn (model/modeling.py:762-770): encoder_info / lang_transformer_info['self_attn_probs']
        # = head-mean probabilities [B, layers, S, S].  Materialised only on request (60 MB per joint layer at configs[1]).
        if export_attention_probs not in (False, True, "layer_mean"):
            raise ValueError(f"export_attention_probs must be False, True or 'layer_mean', got {export_attention_probs!r}")
        self._export_probs = export_attention_probs is True or export_attention_probs == "layer_mean"
        self._probs_layer_mean = export_attention_probs == "layer_mean"
        self._forward(image, shuffled_idx_img, img_mask, mask_draws, mask_override)

    # ---- shapes (:226-260) ----
    @property
    def hidden_size(self):
        return self.config["hidden_size"]

    @property
    def vocab_size(self):
        return self.config["vocab_size"]

    @property
    def B(self):
        return self.batch_size * (self.num_chunks // self.num_chunks_in_group)

    @property
    def L(self):
        return self.lang_chunk_length * self.num_chunks_in_group

    @property
    def viz_chunk_length(self):
        return self.vision_transformer_info["num_h"] * self.vision_transformer_info["num_w"] + 1

    @property
    def P(self):
        return self.viz_chunk_length * self.num_chunks_in_group

    @property
    def dropout_prob(self):
        return self.config["hidden_dropout_prob"]

    @property
    def use_bfloat16(self):
        return self.config["use_bfloat16"]

    @property
    def word_embedding_table(self):
        return self.store.P("word_embeddings/word_embeddings")

    # ---------------------------------------------------------------------------------------------------------
    def _forward(self, image, shuffled_idx_img, img_mask, mask_draws, mask_override):
        cfg, st, bf = self.config, self.store, self._bufs
        H = self.hidden_size
        dev = st.device
        get_shape_list_rank(image, 4, "image")
        N, h0, w0, c3 = image.shape
        Pp = cfg["patch_size"]
        assert h0 % Pp == 0  # utils/vision_transformer.py:189
        assert w0 % Pp == 0  # :190
        if c3 != 3:
            raise ValueError(f"image must be [N,h,w,3], got {tuple(image.shape)}")
        nt, nc, ni = self.num_texts, self.frame_copies, self.num_imgs
        if ni == 1 and N * nt * nc != self.batch_size * self.num_chunks:  # ni > 1: check_num_imgs
            raise ValueError(f"image batch {N} x num_texts {nt} x frame_copies {nc} != batch_size*num_chunks "
                             f"{self.batch_size * self.num_chunks}")
        ncls = cfg.get("num_cls_emb", 2)
        h1, w1 = h0 // Pp, w0 // Pp
        Sv = h1 * w1 + ncls
        sp = max(cfg["spatial_pool_size"], 1)
        self.vision_transformer_info = {"num_h": h1 // sp, "num_w": w1 // sp}
        ncg, B, Lj = self.num_chunks_in_group, self.B, self.L
        Pz = self.P * ni  # the ni images of a text side by side (model/modeling.py:121)
        Sj = Pz + Lj
        self._dims = dict(N=N, Sv=Sv, Pz=Pz, Sj=Sj)
        p_hid = float(cfg["hidden_dropout_prob"] or 0.0)  # 0 unless training (:88-90)
        p_vit = float(cfg.get("vit_hidden_dropout_prob", cfg["hidden_dropout_prob"]) or 0.0) if self.is_training else 0.0

        # ---- language-only encoder (:135-137) on a side stream: it only needs input_ids, and its small latency-bound grids
        # fill the SMs the ViT kernels leave idle.  Joined before mask_inputs.
        side = self._side_stream()
        if self._mask_input:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._lo = _LangOnly(self, p_hid)
            self.lang_trg_h, self.lang_transformer_info = self._lo.lang_trg, self._lo.info

        # ---- ViT (utils/vision_transformer.py:173-274) ----
        img = image.to(torch.bfloat16).contiguous()
        self._vit_in = _VitInput(st, bf, cfg, img, self._save_arenas)
        self._stem, self.d_rc = self._vit_in.stem, None  # d_rc: the gradient backward() hands to the hybrid stem
        self._vit = _Stack(st, bf, "vit", _VIT, cfg.get("num_vision_transformer_hidden_layers", cfg["num_hidden_layers"]), N,
                           Sv, None, self._vit_in.out, cfg, p_vit, self._seed, _SITE_VIT, self._save_arenas)
        hv = self._vit.forward()

        # ---- viz tokens (:95-133) ----
        if shuffled_idx_img is None:
            img_idx = bf.get("img_idx.arange", (N,), torch.int32)
            img_idx.copy_(torch.arange(ncg * ni, dtype=torch.int32, device=dev).repeat(B // (nt * nc)))  # :312-315
        else:
            assert self.num_imgs == 1 and self.num_texts == 1  # :319-320
            img_idx = shuffled_idx_img.reshape(-1).to(torch.int32).contiguous()
            if img_idx.numel() != N * nc:
                raise ValueError(f"shuffled_idx_img has {img_idx.numel()} entries, expected B*num_chunks_in_group = {N * nc}")
        joint_in = bf.get("joint.in", (B * Sj, H), torch.bfloat16)
        self._viz = _VizTokens(st, bf, hv, img_idx, joint_in, (N, h1, w1, ncls, sp), Pz, Sj, nt, nc)
        self.img_trg_h = self._viz.img_trg

        # ---- language-only encoder + masking (:135-139) ----
        ids_j = self.input_ids.reshape(B, Lj)
        if self._mask_input:
            torch.cuda.current_stream().wait_stream(side)
            if mask_override is not None:
                self.lang_mask_info = {"masked_ids": mask_override["masked_ids"].to(dev).to(torch.int32).reshape(B, Lj).contiguous(),
                                       "masked_idx": mask_override["masked_idx"].to(dev).to(torch.int32).contiguous()}
            else:
                self.lang_mask_info = self.mask_inputs(mask_draws)
            ids_j = self.lang_mask_info["masked_ids"].reshape(B, Lj)
        self._mlm = self._ctr = self._tmp = None  # what mask_loss / contrastive_loss / temporal_loss keep for backward()
        if self.features_only:
            return

        # ---- joint encoder (:143-184) ----
        self._emb_j = _Embedding(st, bf, cfg, "emb_j", "position_embeddings", ids_j, joint_in, (Lj, Sj, Pz),
                                 (p_hid, self._seed, _SITE_EMB_J))
        valid_j = bf.get("joint.valid", (B * Sj,), torch.uint8)
        if ni > 1 or img_mask is not None:  # :106-122: image i of row b valid iff img_mask[b // nt, i], over its P tokens
            mask_u8 = None
            if img_mask is not None:
                mask_u8 = bf.get("joint.img_mask", (B // nt, ni), torch.uint8)
                mask_u8.copy_(img_mask.reshape(B // nt, ni) != 0)
            ops.joint_valid_img(ids_j, mask_u8, valid_j, B, nt, ni, self.P, Lj)
        else:
            ops.joint_valid(ids_j, valid_j, B, Pz, Lj)
        c_viz = c_lang = None
        # with the layer-mean map at hand attention_log is taken from it (a fixed summation order), not from K4's column sums
        log_from_colsum = self._log_attention_probs and not self._probs_layer_mean
        if log_from_colsum:  # split column sums of the joint attention maps for attention_log (:186-203)
            c_viz = bf.get("joint.c_viz", (B * Sj,), torch.float32, zero=True)
            c_lang = bf.get("joint.c_lang", (B * Sj,), torch.float32, zero=True)
        probs_j = None
        if self._probs_layer_mean:
            probs_j = bf.get("joint.probs_mean", (B, Sj, Sj), torch.float32)
        elif self._export_probs:
            probs_j = bf.get("joint.probs", (cfg["num_hidden_layers"], B, Sj, Sj), torch.float32)
        self._joint = _Stack(st, bf, "joint", "encoder", cfg["num_hidden_layers"], B, Sj, valid_j, joint_in, cfg,
                             p_hid, self._seed, _SITE_JOINT, self._save, colsum=c_viz, colsum2=c_lang,
                             colsum_split=Pz, colsum_valid_q=1, probs=probs_j, probs_layer_mean=self._probs_layer_mean,
                             # :160-168: language chunks attend to the vision tokens and to themselves only
                             pair=(Pz, self.lang_chunk_length) if cfg.get("disable_pairwise_lang_attn", False) else (0, 0))
        self._y_j = self._joint.forward()
        self._attn_log = None
        if log_from_colsum:
            out4 = bf.get("joint.attn_log", (4,), torch.float32)
            L.lib().merlot_attention_log_blocks(c_viz.data_ptr(), c_lang.data_ptr(), valid_j.data_ptr(), B, Sj, Pz,
                                                out4.data_ptr(), ops._stream())
            self._attn_log = out4
        elif self._log_attention_probs:
            self._attn_log = ops.attention_log_probs(probs_j, valid_j, Pz, bf.get("joint.attn_log", (4,), torch.float32))
        self.encoder_info = {"hidden_state": self._y_j.view(B, Sj, H)}
        if self._probs_layer_mean:  # already the mean over layers, [B, S, S]
            self.encoder_info["self_attn_probs"] = probs_j
        elif probs_j is not None:  # [layers,B,S,S] -> the reference's [B, layers, S, S] (utils/transformer.py:238), a view
            self.encoder_info["self_attn_probs"] = probs_j.permute(1, 0, 2, 3)
        self._hidden_f32 = {}
        self.encoder_pieces = [{"name": "viz", "start": 0, "end": Pz}, {"name": "lang", "start": Pz, "end": Sj}]

    def _side_stream(self):
        """Stream for the language-only stack (set MERLOT_NO_SIDE_STREAM=1 to serialise everything on one stream)."""
        st = self.store
        if os.environ.get("MERLOT_NO_SIDE_STREAM", "0") == "1":
            return torch.cuda.current_stream()
        if not hasattr(st, "_side"):
            st._side = torch.cuda.Stream(device=st.device)
        return st._side

    # ---------------------------------------------------------------------------------------------------------
    def embed_words(self, input_ids_2d, norm_scope_name="position_embeddings", reuse=None):
        """Public mirror of :262-297; returns bf16 [B, L, H]."""
        get_shape_list_rank(input_ids_2d, 2, "input_ids_2d")
        ids = input_ids_2d.to(torch.int32).contiguous()
        out = torch.empty((ids.numel(), self.hidden_size), dtype=torch.bfloat16, device=ids.device)
        _Embedding(self.store, self._bufs, self.config, f"emb_pub.{norm_scope_name}", norm_scope_name, ids, out, (0, 0, 0),
                   (float(self.dropout_prob or 0.0), self._seed, _SITE_EMB_J))
        return out.view(ids.shape[0], ids.shape[1], -1)

    def langonly_reps(self):
        return self.lang_trg_h, self.lang_transformer_info

    def mask_inputs(self, draws: Optional[Dict] = None):
        """mask_inputs (:381-489) on device; `draws` injects the reference's five tf.random tensors."""
        cfg, bf = self.config, self._bufs
        B, Lj = self.B, self.L
        dev = self.store.device
        topk_perc = cfg.get("masking_use_topk_from_attn_perc", 0.20)
        choose_topk_prob = cfg.get("masking_choose_topk_prob", 0.5)
        masking_rate = cfg.get("masking_rate", 0.2)
        do_spanbert = cfg.get("masking_do_spanbert", True)
        span_probs = cfg.get("masking_spanbert_len_probs", [0.625, 0.25, 0.125])
        use_attn = cfg.get("masking_use_attn", True)
        num_topk = int(Lj * topk_perc)
        num_to_mask = int(Lj * masking_rate)
        nontopk_val = 0.01
        topk_val = nontopk_val * choose_topk_prob * (1.0 - topk_perc) / (topk_perc * (1.0 - choose_topk_prob))  # :418-419
        if use_attn:
            w = torch.tensor([1.0, 0.0]) * np.float32(topk_val - nontopk_val) + np.float32(nontopk_val)  # :437
            logw = torch.log(w)
            consts = (float(np.float32(topk_val - nontopk_val)), float(np.float32(nontopk_val)), float(logw[0]), float(logw[1]),
                      float(w.max()))
        else:
            consts = (0.0, 1.0, 0.0, 0.0, 1.0)
        if draws is None:  # drawn on device (Philox keyed by the step seed): nothing in the step waits for the host
            key = ("mask.draws", B, Lj, num_to_mask)
            draws = ops.mask_draws(B, Lj, num_to_mask, self.vocab_size, span_probs, 1234567 + self._seed, dev, out=bf.d.get(key))
            bf.d[key] = draws
        else:  # injected draws (tests, reproducing a reference run's tf.random tensors)
            draws = {k: v.to(dev).contiguous() for k, v in draws.items()}
        masked_ids = bf.get("mask.ids", (B, Lj), torch.int32)
        masked_idx = bf.get("mask.idx", (B, num_to_mask), torch.int32)
        summ = self.lang_transformer_info["attention_summs"] if use_attn else None
        ops.mask_inputs(self.input_ids.reshape(B, Lj), summ, draws, masked_ids, masked_idx, None, num_topk, num_to_mask,
                        do_spanbert, MASK, consts)
        return {"masked_ids": masked_ids.view(self.input_ids.shape), "masked_idx": masked_idx}

    @staticmethod
    def make_mask_draws(B, Lj, num_to_mask, vocab_size, span_probs, device, seed=0):
        """The tf.random.* draws of mask_inputs (:445-481) from a torch generator."""
        g = torch.Generator(device="cpu").manual_seed(1234567 + seed)
        u = torch.rand(B, Lj, generator=g).clamp_(1e-9, 1.0 - 1e-7)
        probs = torch.tensor(span_probs, dtype=torch.float32)
        return {
            "gumbel": (-torch.log(-torch.log(u))).float(),
            "span_lower": torch.multinomial(probs, B * num_to_mask, True, generator=g).reshape(B, num_to_mask).int(),
            "span_upper": torch.multinomial(probs, B * num_to_mask, True, generator=g).reshape(B, num_to_mask).int(),
            "option": torch.multinomial(torch.tensor([0.1, 0.8, 0.1]), B * Lj, True, generator=g).int(),
            "rand_ids": torch.randint(100, vocab_size, (B * Lj,), generator=g).int(),
        }

    # ---- attributes the callers read (:176-203) ----
    @property
    def encoder_hidden_states(self):
        """{'viz': fp32 [B,P,H], 'lang': fp32 [B,L,H]} (:176-184)."""
        if not self._hidden_f32:
            H, B, Sj, Pz = self.hidden_size, self.B, self._dims["Sj"], self._dims["Pz"]
            y3 = self._y_j.view(B, Sj, H)
            for name, sl in (("viz", slice(0, Pz)), ("lang", slice(Pz, Sj))):
                piece = y3[:, sl].contiguous()
                out = torch.empty(piece.shape, dtype=torch.float32, device=piece.device)
                ops.cast_bf16_to_f32(piece, out)
                self._hidden_f32[name] = out
        return self._hidden_f32

    @property
    def attention_log(self):
        """{'encoder/lang2lang', 'encoder/lang2viz', 'encoder/viz2lang', 'encoder/viz2viz'} (:186-203); logging only."""
        if self._attn_log is None:
            raise ValueError("attention_log needs log_attention_probs=True at construction (model/modeling.py:186)")
        names = ("lang2lang", "lang2viz", "viz2lang", "viz2viz")
        return {f"encoder/{n}": self._attn_log[i] for i, n in enumerate(names)}

    # ---------------------------------------------------------------------------------------------------------
    # heads
    # ---------------------------------------------------------------------------------------------------------
    def lm_head(self, hidden_state):
        """lm_head (:205-224) on bf16 rows [R,H]; returns fp32 logits [R, ldV] (columns >= vocab_size are padding)."""
        return self._lm_head("lm_pub", hidden_state.contiguous())[2][:, :self.vocab_size]

    def _lm_head(self, tag, pooled):
        """Returns (the projection's _MlpLn or None, the bf16 rows hn [R, H] the output layer reads, fp32 logits [R, ldV])."""
        cfg, st, bf = self.config, self.store, self._bufs
        R, H, V = pooled.shape[0], self.hidden_size, self.vocab_size
        proj = None
        if cfg.get("do_projection", False):
            proj = _MlpLn(st, bf, f"{tag}.proj", pooled, "lm_head/projection", "lm_head/LayerNorm", H)
        hn = proj.out if proj else pooled
        logits = bf.get(f"{tag}.logits", (R, (V + 63) // 64 * 64), torch.float32)
        bias = st.P("lm_head/output_bias") if cfg.get("do_bias", False) else None
        ops.gemm(hn, st.W("word_embeddings/word_embeddings"), bias=bias, out=logits, M=R, N=V, K=H)
        return proj, hn, logits

    def mask_loss(self):
        """mask_loss (:528-551).  Returns (loss, {'loss','acc'}) as 0-d CUDA tensors."""
        bf = self._bufs
        B, Lj = self.B, self.L
        k = self.lang_mask_info["masked_idx"].shape[1]
        nm = B * k
        rows = bf.get("mlm.rows", (nm,), torch.int32)
        targets = bf.get("mlm.targets", (nm,), torch.int32)
        ops.mlm_index(self.input_ids.reshape(B, Lj), self.lang_mask_info["masked_idx"], rows, targets, B, Lj, k, self._dims["Pz"])
        pooled = bf.get("mlm.pooled", (nm, self.hidden_size), torch.bfloat16)
        ops.gather_rows(self._y_j, rows, pooled)
        proj, hn, logits = self._lm_head("mlm", pooled)
        ce = _SoftmaxCE(bf, "mlm", logits, targets, self.vocab_size, nz_labels=targets, denom_mode=1, accuracy=True)
        self._mlm = (rows, proj, hn, ce)
        return ce.out2[0], {"loss": ce.out2[0], "acc": ce.out2[1]}

    def _mask_loss_bwd(self, d_yj):
        st, bf = self.store, self._bufs
        rows, proj, hn, ce = self._mlm
        V, H = self.vocab_size, self.hidden_size
        nm, ldV = ce.logits.shape
        dlog = ce.backward(bf.get("mlm.dlogits", (nm, ldV), torch.bfloat16))
        if self.config.get("do_bias", False):
            gb_pad = st.g[st.entries["lm_head/output_bias"].offset:st.entries["lm_head/output_bias"].offset + ldV]
            ops.bias_grad(dlog, gb_pad, rows=nm, N=ldV)
        # tied embedding: dE += dlogits^T hn ; d_hn = dlogits E
        ops.gemm(dlog, hn, a_mn_major=True, b_mn_major=True, out=st.G("word_embeddings/word_embeddings"), atomic=True,
                 M=V, N=H, K=nm)
        d_hn = bf.get("mlm.d_hn", (nm, H), torch.float32, zero=True)  # split-K over the 50370-long contraction
        ops.gemm(dlog, st.W("word_embeddings/word_embeddings"), b_mn_major=True, out=d_hn, atomic=True, M=nm, N=H, K=V)
        d_pooled = proj.backward(d_hn) if proj else d_hn
        ops.scatter_add_rows(d_pooled, rows, d_yj)

    def contrastive_features(self):
        """The projection towers (project_and_norm, :18-44) of this batch's lang / viz rows, as two _Tower records whose
        `feat` fp32 [n, Cs] are the l2-normalised features contrastive_loss compares.  The tensors are buffers the next
        model on the same ParamStore overwrites."""
        st, bf, cfg = self.store, self._bufs, self.config
        return (_Tower(st, bf, cfg, "ctr.lang", self.lang_trg_h, "lang_proj"),
                _Tower(st, bf, cfg, "ctr.viz", self.img_trg_h, "viz_proj"))

    def contrastive_loss(self):
        """contrastive_loss (:491-526).  Multi-GPU: features are all-gathered over the data-parallel group
        (tpu_cross_replica_stack, utils/model_utils.py:673-707) and labels are offset by rank*N (:519)."""
        lang, viz = self.contrastive_features()
        info, outs = contrastive_head(self._bufs, self.config, self.dist, lang.feat, viz.feat, lang.n)
        self._ctr = (info, lang, viz)
        return outs["loss_all"], outs

    def _temporal_index(self):
        bf, dev = self._bufs, self.store.device
        B, n, Sj, Pz, vcl, Lc = self.B, self.num_chunks_in_group, self._dims["Sj"], self._dims["Pz"], self.viz_chunk_length, \
            self.lang_chunk_length
        key = ("_tidx", B, n, Sj, Pz, vcl, Lc)
        if key not in bf.d:
            b = torch.arange(B, device=dev)[:, None]
            s = torch.arange(n, device=dev)[None]
            idx_l = (b * Sj + Pz + s * Lc).reshape(-1).to(torch.int32)
            idx_v = (b * Sj + s * vcl).reshape(-1).to(torch.int32)
            bi = torch.arange(B, device=dev)[:, None, None]
            i = torch.arange(n, device=dev)[None, :, None]
            j = torch.arange(n, device=dev)[None, None, :]
            idxA = (bi * n + i + 0 * j).reshape(-1).to(torch.int32)  # row b*n*n + i*n + j takes xa[b, i]   (:573-574)
            idxB = (bi * n + j + 0 * i).reshape(-1).to(torch.int32)  # ... and xb[b, j]                       (:576-577)
            bf.d[key] = (idx_l, idx_v, idxA, idxB)
        return bf.d[key]

    def allpairs_temporal_logits(self, xa, xb, scope_name="temporal_paired"):
        """allpairs_temporal_logits (:553-596). xa, xb: [B, n, H] (fp32 or bf16). Returns fp32 logits [B*n*n, 4]."""
        get_shape_list_rank(xa, 3, "xa")
        B, n, H = xa.shape
        assert list(xa.shape) == [B, self.num_chunks_in_group, self.hidden_size]
        assert list(xb.shape) == [B, self.num_chunks_in_group, self.hidden_size]
        xa2 = xa.reshape(B * n, H).to(torch.bfloat16).contiguous()
        xb2 = xb.reshape(B * n, H).to(torch.bfloat16).contiguous()
        return self._temporal_head(f"tmp_pub.{scope_name}", scope_name, xa2, xb2)[2][:, :4]

    def _temporal_head(self, tag, scope, xa_bf16, xb_bf16):
        """Returns (its _MlpLn, its output _Dense, fp32 logits [B*n*n, 8])."""
        st, bf = self.store, self._bufs
        B, n, H = self.B, self.num_chunks_in_group, self.hidden_size
        _, _, idxA, idxB = self._temporal_index()
        R = B * n * n
        hj = bf.get(f"{tag}.hj", (R, 2 * H), torch.bfloat16)
        ops.gather_rows(xa_bf16, idxA, hj[:, :H], H=H)
        ops.gather_rows(xb_bf16, idxB, hj[:, H:], H=H)
        mlp = _MlpLn(st, bf, f"{tag}.mlp", hj, f"{scope}/intermediate", f"{scope}/LayerNorm_ln0", H)
        dense = _Dense(st, bf, tag, f"{scope}/logits", mlp.out)
        return mlp, dense, dense.forward(bf.get(f"{tag}.logits", (R, 8), torch.float32))

    def allpairs_temporal_labels(self, video_src_ids, shuffled_idx_img=None):
        """allpairs_temporal_labels (:598-620)."""
        return self._temporal_labels(video_src_ids, shuffled_idx_img)[0]

    def _temporal_labels(self, video_src_ids, shuffled_idx_img):
        """(labels int32, pair weights fp32 (:635, :649-652)), [B*n*n] each."""
        bf = self._bufs
        B, n = self.B, self.num_chunks_in_group
        labels = bf.get("tmp.labels", (B * n * n,), torch.int32)
        w = bf.get("tmp.w", (B * n * n,), torch.float32)
        v = video_src_ids.reshape(B, n).to(torch.int32).contiguous()
        s = (shuffled_idx_img if shuffled_idx_img is not None else torch.zeros_like(v)).reshape(B, n).to(torch.int32).contiguous()
        ops.temporal_labels(v, s, labels, w, B, n)
        return labels, w

    def temporal_loss(self, shuffled_idx_img, video_src_ids):
        """temporal_loss (:622-668)."""
        cfg, bf = self.config, self._bufs
        B, n, H = self.B, self.num_chunks_in_group, self.hidden_size
        idx_l, idx_v, _, _ = self._temporal_index()
        h_lang = bf.get("tmp.h_lang", (B * n, H), torch.bfloat16)
        h_viz = bf.get("tmp.h_viz", (B * n, H), torch.bfloat16)
        ops.gather_rows(self._y_j, idx_l, h_lang)
        ops.gather_rows(self._y_j, idx_v, h_viz)
        labels, w = self._temporal_labels(video_src_ids, shuffled_idx_img)
        coef = cfg.get("temporal_coef", 1.0)
        use_vv = cfg.get("image_shuffle_prob", 0) > 0  # :664-665
        info, out2s, in_loss = {}, {}, []
        for name, xa, xb in (("lang_viz", h_lang, h_viz), ("viz_viz", h_viz, h_viz)):
            mlp, dense, logits = self._temporal_head(f"tmp.{name}", f"{name}_temporal", xa, xb)
            ce = _SoftmaxCE(bf, f"tmp.{name}", logits, labels, 4, weights=w, scale=coef, accuracy=True)
            info[f"{name}_loss"], info[f"{name}_acc"], out2s[name] = ce.out2[0], ce.out2[1], ce.out2
            if name == "lang_viz" or use_vv:
                in_loss.append((mlp, dense, ce))
        tot = bf.get("tmp.loss", (1,), torch.float32)
        ops.axpby(out2s["lang_viz"][:1], tot, 1.0, 0.0)
        if use_vv:
            ops.axpby(out2s["viz_viz"][:1], tot, 1.0, 1.0)
        info["loss"] = tot[0]
        loss = bf.get("tmp.loss_scaled", (1,), torch.float32)
        ops.axpby(tot, loss, coef, 0.0)
        self._tmp = in_loss
        return loss[0], info

    def _temporal_bwd(self, d_yj):
        bf = self._bufs
        B, n, H = self.B, self.num_chunks_in_group, self.hidden_size
        idx_l, idx_v, idxA, idxB = self._temporal_index()
        d_hl = bf.get("tmp.d_hl", (B * n, H), torch.float32, zero=True)
        d_hv = bf.get("tmp.d_hv", (B * n, H), torch.float32, zero=True)
        # lang_viz, then viz_viz when it is in the loss
        for (mlp, dense, ce), da, db in zip(self._tmp, (d_hl, d_hv), (d_hv, d_hv)):
            dlog = ce.backward(bf.get(f"{dense.tag}.dlogits", ce.logits.shape, torch.float32))
            d_hj = mlp.backward(dense.backward(dlog))  # fp32 [R, 2H]
            ops.scatter_add_rows(d_hj[:, :H], idxA, da, H=H)
            ops.scatter_add_rows(d_hj[:, H:], idxB, db, H=H)
        ops.scatter_add_rows(d_hl, idx_l, d_yj)
        ops.scatter_add_rows(d_hv, idx_v, d_yj)

    # ---------------------------------------------------------------------------------------------------------
    # backward of the whole model: call after mask_loss / contrastive_loss / temporal_loss (whichever are in the loss)
    # ---------------------------------------------------------------------------------------------------------
    def backward(self, on_non_vit_grads_ready=None, vit_layer_groups=None, on_vit_group_done=None, d_hidden_state=None,
                 d_contrastive_features=None):
        """d(lang_loss + contr_loss + temp_loss)/d(params) accumulated into store.g  (model/modeling.py:713 loss,
        utils/optimization.py:176 tf.gradients).  Order: heads -> joint encoder -> language-only encoder -> (callback: every
        gradient outside vision_backbone/vision_transformer is final; data-parallel training starts their all-reduce here)
        -> ViT.

        `d_contrastive_features` = (d_lang, d_viz), fp32 [n, Cs] each: the gradient of a contrastive loss computed elsewhere
        (over the features of several micro-batches, contrastive_head) w.r.t. this batch's contrastive_features().  The
        projection towers run forward again and backward from it, in place of this model's own contrastive_loss()."""
        if not self._save:
            raise RuntimeError("MerlotModel was built without save_for_backward (is_training=False)")
        if d_contrastive_features is not None:
            if self._ctr is not None:
                raise ValueError("d_contrastive_features replaces this model's contrastive_loss(): do not call both")
            if not self._mask_input:
                raise ValueError("d_contrastive_features needs mask_input=True (the language features)")
        bf, H, B, Sj = self._bufs, self.hidden_size, self.B, self._dims["Sj"]
        d_yj = bf.get("bwd.d_yj", (B * Sj, H), torch.bfloat16, zero=True)
        if d_hidden_state is not None:  # gradient of an external head (e.g. downstream/vcr's classifier) w.r.t. encoder_info['hidden_state']
            if tuple(d_hidden_state.shape) not in ((B * Sj, H), (B, Sj, H)) or d_hidden_state.dtype != torch.bfloat16:
                raise ValueError("d_hidden_state must be bf16 [B, P+L, H]")
            d_yj.copy_(d_hidden_state.reshape(B * Sj, H))
        d_img_trg = bf.get("bwd.d_img_trg", self.img_trg_h.shape, torch.float32, zero=True)
        d_lang_trg = None
        if self._mask_input:
            d_lang_trg = bf.get("bwd.d_lang_trg", (self.batch_size * self.num_chunks, H), torch.float32, zero=True)
        if self._mlm is not None:
            self._mask_loss_bwd(d_yj)
        if self._ctr is not None or d_contrastive_features is not None:
            if self._ctr is not None:
                info, lang, viz = self._ctr
                d_feat = contrastive_head_bwd(bf, self.dist, info)
                d_l, d_v = d_feat["lang"], d_feat["viz"]
            else:
                lang, viz = self.contrastive_features()
                d_l, d_v = d_contrastive_features
                shape = (lang.n, lang.Cs)
                if tuple(d_l.shape) != shape or tuple(d_v.shape) != shape or d_l.dtype != torch.float32 or d_v.dtype != torch.float32:
                    raise ValueError(f"d_contrastive_features must be two fp32 {list(shape)} tensors")
                d_l, d_v = d_l.contiguous(), d_v.contiguous()
            dl, dv = lang.backward(d_l), viz.backward(d_v)
            ops.axpby(dl, d_lang_trg, 1.0, 1.0)
            ops.axpby(dv, d_img_trg, 1.0, 1.0)
        if self._tmp is not None:
            self._temporal_bwd(d_yj)
        # ---- language-only encoder backward on the side stream: it needs only d_lang_trg (contrastive head) and runs
        # concurrently with the joint-encoder backward below, whose small grids leave a third of the SMs idle ----
        side = self._side_stream()
        main = torch.cuda.current_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            if self._mask_input:
                self._lo.backward(d_lang_trg)
        d_jin = bf.get("bwd.d_jin", (B * Sj, H), torch.bfloat16)
        self._joint.backward(d_yj, d_jin)
        self._emb_j.backward(d_jin)
        d_hv = self._viz.backward(d_jin, d_img_trg)
        # join the language-only backward (side stream); every gradient outside the ViT is final now
        main.wait_stream(side)
        if on_non_vit_grads_ready is not None:
            on_non_vit_grads_ready()
        # ---- ViT ----
        d_h0v = bf.get("bwd.d_h0v", self._vit_in.out.shape, torch.bfloat16)
        self._vit.backward(d_hv, d_h0v, vit_layer_groups, on_vit_group_done)
        self.d_rc = self._vit_in.backward(d_h0v)


def _pad8(k: int) -> int:
    return (k + 7) // 8 * 8


def contrastive_head(bufs: _Buffers, cfg: dict, dist, lang_feat, viz_feat, per_replica: int):
    """The contrastive loss (:491-526) over rows of l2-normalised features, fp32 [n, Cs]: the rows of this rank, made of
    n / per_replica (virtual) replicas of `per_replica` rows each.  Features are all-gathered over the data-parallel group
    (tpu_cross_replica_stack, utils/model_utils.py:673-707), so row i's label is rank*n + i (:519).  Every replica's loss is
    the mean over its own rows; the backward coefficients are those of the SUM of the replicas' losses, the reported losses
    are their mean.  Returns (info for contrastive_head_bwd, {'lang_to_viz', 'viz_to_lang', 'loss_all'} 0-d tensors).
    The products run on K16 (csrc/contrastive.cu): K1 tensor-core GEMMs over a three-term bf16 split of the fp32 features,
    deterministic, at any n and world."""
    bf = bufs
    n, Cs = lang_feat.shape
    if n % per_replica != 0:
        raise ValueError(f"{n} contrastive rows are not a whole number of replicas of {per_replica} rows")
    world, rank = (dist.world, dist.rank) if dist is not None else (1, 0)
    if world > 1:
        all_lang, all_viz = dist.all_gather_rows(lang_feat), dist.all_gather_rows(viz_feat)
    else:
        all_lang, all_viz = lang_feat, viz_feat
    temp = cfg.get("contrast_temp", 0.05)
    coef = cfg.get("contrast_coef", 1.0)
    labels = bf.get("ctr.labels", (n,), torch.int32)
    labels.copy_(torch.arange(n, dtype=torch.int32, device=labels.device) + rank * n)
    nW = n * world
    outs, out2s = {}, {}
    feats = {"lang": lang_feat, "viz": viz_feat}
    if Cs % 8 != 0:
        raise ValueError(f"contrastive_size {Cs} must be a multiple of 8 (K16's bf16 operand rows)")
    info = dict(feats=feats, all_lang=all_lang, all_viz=all_viz, labels=labels, nW=nW, temp=temp, dirs={})
    for name, x, y in (("lang_to_viz", lang_feat, all_viz), ("viz_to_lang", viz_feat, all_lang)):
        # K16: S = [xh | xh | xl] . [yh | yl | yh]^T / temp, one K1 GEMM over K = 3 Cs
        xc = bf.get(f"ctr.{name}.xcat", (n, 3 * Cs), torch.bfloat16)
        yc = bf.get(f"ctr.{name}.ycat", (nW, 3 * Cs), torch.bfloat16)
        ops.ctr_split(x, xc, 3 * Cs, Cs, 0b100)
        ops.ctr_split(y, yc, 3 * Cs, Cs, 0b010)
        logits = bf.get(f"ctr.{name}.logits", (n, _pad8(nW)), torch.float32)[:, :nW]
        ops.gemm(xc, yc, out=logits, alpha=1.0 / temp, M=n, N=nW, K=3 * Cs)
        # out2[0] = mean over all rows = mean of the replicas' losses; coeff[i] = coef / (2 * per_replica)
        ce = _SoftmaxCE(bf, f"ctr.{name}", logits, labels, nW, scale=coef / 2.0 * (n // per_replica))
        outs[name], out2s[name] = ce.out2[0], ce.out2
        info["dirs"][name] = ce
    loss_all = bf.get("ctr.loss_all", (1,), torch.float32)
    ops.axpby(out2s["lang_to_viz"][:1], loss_all, coef / 2.0, 0.0)
    ops.axpby(out2s["viz_to_lang"][:1], loss_all, coef / 2.0, 1.0)
    outs["loss_all"] = loss_all[0]
    return info, outs


def contrastive_head_bwd(bufs: _Buffers, dist, info) -> Dict[str, torch.Tensor]:
    """Gradient of contrastive_head's loss w.r.t. this rank's feature rows: {'lang', 'viz'} fp32 [n, Cs] buffers."""
    bf, c = bufs, info
    nW, temp = c["nW"], c["temp"]
    n, Cs = c["feats"]["lang"].shape
    world = dist.world if dist is not None else 1
    d_feat = {"lang": bf.get("ctr.d_feat.lang", (n, Cs), torch.float32), "viz": bf.get("ctr.d_feat.viz", (n, Cs), torch.float32)}
    d_all = {"lang": bf.get("ctr.d_all.lang", (nW, Cs), torch.float32), "viz": bf.get("ctr.d_all.viz", (nW, Cs), torch.float32)}
    for name, xk, yk, y_all in (("lang_to_viz", "lang", "viz", c["all_viz"]), ("viz_to_lang", "viz", "lang", c["all_lang"])):
        ce = c["dirs"][name]
        # K16: dS = coeff (softmax - onehot) / temp straight into its hi/lo operands, side by side and stacked
        dsh = bf.get(f"ctr.{name}.dsh", (n, _pad8(3 * nW)), torch.bfloat16)
        dsv = bf.get(f"ctr.{name}.dsv", (3 * n, _pad8(nW)), torch.bfloat16)
        ops.ctr_dlogits(ce.logits, c["labels"], nW, ce.lse, ce.coeff, 1.0 / temp, dsh, dsv)
        ys = bf.get(f"ctr.{name}.ystack", (3 * nW, Cs), torch.bfloat16)
        xs = bf.get(f"ctr.{name}.xstack", (3 * n, Cs), torch.bfloat16)
        ops.ctr_split(y_all, ys, Cs, nW * Cs, 0b010)
        ops.ctr_split(c["feats"][xk], xs, Cs, n * Cs, 0b010)
        # d_x = [dSh | dSh | dSl] . [yh ; yl ; yh]            (K = 3 nW)
        ops.gemm(dsh, ys, b_mn_major=True, out=d_feat[xk], M=n, N=Cs, K=3 * nW)
        # d_y_all = [dSh ; dSh ; dSl]^T . [xh ; xl ; xh]      (K = 3 n)
        ops.gemm(dsv, xs, a_mn_major=True, b_mn_major=True, out=d_all[yk], M=nW, N=Cs, K=3 * n)
    for k in ("lang", "viz"):
        # gradient of the gather = reduce-scatter(sum) of every rank's d_all (utils/model_utils.py:699-706)
        mine = dist.reduce_scatter_rows(d_all[k]) if world > 1 else d_all[k]
        ops.axpby(mine, d_feat[k], 1.0, 1.0)
    return d_feat
