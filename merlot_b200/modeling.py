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

MASK = 1  # utils/encode/encoder.py:16-22
PADDING = 0
START = 2

_SITE_VIT, _SITE_LANGONLY, _SITE_JOINT, _SITE_EMB_LO, _SITE_EMB_J = 0, 100, 200, 300, 301
# VCR classifier towers (merlot_b200/vcr.py cls_head): dropout of each tower's input and of its hidden layer
_SITE_VCR_ANS_IN, _SITE_VCR_ANS_HID, _SITE_VCR_RAT_IN, _SITE_VCR_RAT_HID = 400, 401, 402, 403


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


class _Stack:
    """One transformer stack invocation (utils/transformer.py:171-247) through merlot_stack_forward/backward."""

    def __init__(self, store, bufs, tag, scope, layers, B, S, valid, h_in, cfg, dropout_p, seed, site, save, colsum=None,
                 colsum2=None, colsum_split=0, colsum_valid_q=0, probs=None, pair=(0, 0)):
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


class MerlotModel(object):
    def __init__(self, config, is_training, use_tpu, image, input_ids, mask_input=False, shuffled_idx_img=None,
                 img_mask=None, log_attention_probs=True, *, params: ParamStore, mask_draws: Optional[Dict] = None,
                 mask_override: Optional[Dict] = None, dropout_seed: int = 0, save_for_backward: Optional[bool] = None,
                 dist=None, export_attention_probs: bool = False):
        """Arguments as model/modeling.py:48-66.  `use_tpu` is accepted and ignored (it only selects one-hot vs gather
        embedding lookups in the reference, utils/model_utils.py:259-263 -- same values either way)."""
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
        if cfg.get("num_imgs", 1) != 1 or img_mask is not None:
            raise NotImplementedError("num_imgs > 1 / img_mask (model/modeling.py:106-122) not provided (no shipped config uses them)")
        if cfg.get("num_texts", 1) > 1 and (mask_input or shuffled_idx_img is not None):
            raise NotImplementedError("num_texts > 1 (VCR, model/modeling.py:111-119) is a finetuning/inference path: mask_input and "
                                      "shuffled_idx_img are not combined with it in the reference either (:319-320)")
        if not cfg.get("share_params", True):
            raise NotImplementedError("share_params: False (separate langonly_encoder, model/modeling.py:361) not provided yet")
        # hybrid ResNet-lite stem (utils/vision_transformer.py:206-223) instead of the 16x16 patch embedding: forward provided
        self._resnet_layers = list(cfg.get("resnet_layers", []) or [])

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
        self.num_imgs = cfg.get("num_imgs", 1)
        self.num_texts = cfg.get("num_texts", 1)
        self.img_batch_size = self.batch_size // self.num_texts
        if not is_training:  # :88-90
            cfg["hidden_dropout_prob"] = 0.0
            cfg["attention_probs_dropout_prob"] = 0.0
        self._save = bool(is_training) if save_for_backward is None else bool(save_for_backward)
        self._seed = int(dropout_seed)
        self._bufs = _Buffers(params)
        self._mask_input = mask_input
        self._log_attention_probs = log_attention_probs
        # PREDICT-mode outputs of model_fn (model/modeling.py:762-770): encoder_info / lang_transformer_info['self_attn_probs']
        # = head-mean probabilities [B, layers, S, S].  Materialised only on request (60 MB per joint layer at configs[1]).
        self._export_probs = bool(export_attention_probs)
        self._forward(image, shuffled_idx_img, mask_draws, mask_override)

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
    def _forward(self, image, shuffled_idx_img, mask_draws, mask_override):
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
        nt = self.num_texts
        if N * nt != self.batch_size * self.num_chunks:
            raise ValueError(f"image batch {N} x num_texts {nt} != batch_size*num_chunks {self.batch_size * self.num_chunks}")
        ncls = cfg.get("num_cls_emb", 2)
        h1, w1 = h0 // Pp, w0 // Pp
        np_ = h1 * w1
        Sv = np_ + ncls
        Mv = N * Sv
        sp = cfg["spatial_pool_size"]
        h2, w2 = (h1 // sp, w1 // sp) if sp > 1 else (h1, w1)
        self.vision_transformer_info = {"num_h": h2, "num_w": w2}
        vcl, ncg, B, Lj = self.viz_chunk_length, self.num_chunks_in_group, self.B, self.L
        Pz = self.P
        Sj = Pz + Lj
        self._dims = dict(N=N, h1=h1, w1=w1, np=np_, ncls=ncls, Sv=Sv, Mv=Mv, sp=max(sp, 1), h2=h2, w2=w2, vcl=vcl, Pz=Pz,
                          Sj=Sj, Kp=Pp * Pp * 3)
        train = self.is_training
        p_hid = float(cfg["hidden_dropout_prob"] or 0.0)
        p_vit = float(cfg.get("vit_hidden_dropout_prob", cfg["hidden_dropout_prob"]) or 0.0) if train else 0.0
        vt = "vision_backbone/vision_transformer"

        # ---- language-only encoder (:135-137) on a side stream: it only needs input_ids, and its small latency-bound grids
        # fill the SMs the ViT kernels leave idle.  Joined before mask_inputs.
        side = self._side_stream()
        if self._mask_input:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._langonly_reps()

        # ---- ViT (utils/vision_transformer.py:173-274) ----
        img = image if image.dtype == torch.bfloat16 else image.to(torch.bfloat16)
        img = img.contiguous()
        patch = bf.get("vit.patch", (N * np_, H), torch.float32)
        if not self._resnet_layers:
            A = bf.get("vit.A", (N * np_, Pp * Pp * 3), torch.bfloat16)
            ops.patch_im2col(img, A, Pp)
            ops.gemm(A, st.W(f"{vt}/conv2d/kernel"), b_mn_major=True, bias=st.P(f"{vt}/conv2d/bias"), out=patch)
        else:  # hybrid stem (:206-223): lite_resnet50 -> 1x1 conv_postresnet_proj with bias (not standardised)
            if Pp != 16:
                raise ValueError("the hybrid ResNet stem needs patch_size 16 (utils/vision_transformer.py:208)")
            rc, hs, ws_ = self._hybrid_stem(img, N, h0, w0)
            if (hs, ws_) != (h1, w1):
                raise ValueError(f"stem output {hs}x{ws_} != patch grid {h1}x{w1}")
            ops.gemm(rc, st.W(f"{vt}/conv_postresnet_proj/kernel"), b_mn_major=True, bias=st.P(f"{vt}/conv_postresnet_proj/bias"),
                     out=patch)
        xsum_v = bf.get("vit.xsum", (Mv, H), torch.float32)
        ops.vit_assemble_fwd(patch, st.P(f"{vt}/pos_embs/pos_embs"), st.P(f"{vt}/pos_embs/cls_emb"), xsum_v, N, h1, w1, ncls, H)
        h0_v = bf.get("vit.h0", (Mv, H), torch.bfloat16)
        mean_v, rstd_v = bf.get("vit.mean0", (Mv,), torch.float32), bf.get("vit.rstd0", (Mv,), torch.float32)
        ops.layernorm_fwd(xsum_v, h0_v, st.P(f"{vt}/LayerNorm_ctx_patches_pre_ln/gamma"),
                          st.P(f"{vt}/LayerNorm_ctx_patches_pre_ln/beta"), mean_v, rstd_v)
        self._vit = _Stack(st, bf, "vit", vt, cfg.get("num_vision_transformer_hidden_layers", cfg["num_hidden_layers"]), N, Sv,
                           None, h0_v, cfg, p_vit, self._seed, _SITE_VIT, self._save)
        hv = self._vit.forward()

        # ---- viz tokens (:95-133) ----
        if shuffled_idx_img is None:
            img_idx = bf.get("img_idx.arange", (N,), torch.int32)
            img_idx.copy_(torch.arange(ncg, dtype=torch.int32, device=dev).repeat(B // nt))
            self._shuffled = None
        else:
            assert self.num_imgs == 1 and self.num_texts == 1  # :319-320
            img_idx = shuffled_idx_img.reshape(-1).to(torch.int32).contiguous()
            if img_idx.numel() != N:
                raise ValueError(f"shuffled_idx_img has {img_idx.numel()} entries, expected B*num_chunks_in_group = {N}")
        self._img_idx = img_idx
        Bi = B // nt  # image groups; with num_texts > 1 every group's tokens are tiled to its nt texts (model/modeling.py:111-119)
        xsum_z = bf.get("viz.xsum", (Bi * Pz, H), torch.float32)
        self.img_trg_h = bf.get("viz.img_trg", (N, H), torch.float32)
        ops.viz_assemble_fwd(hv, st.P("vision_backbone/img_idx_pe"), img_idx, st.P("vision_backbone/final_pe/pos_embs"),
                             st.P("vision_backbone/final_pe/cls_emb"), xsum_z, self.img_trg_h, N, h1, w1, ncls, max(sp, 1), H)
        joint_in = bf.get("joint.in", (B * Sj, H), torch.bfloat16)
        mean_z, rstd_z = bf.get("viz.mean", (Bi * Pz,), torch.float32), bf.get("viz.rstd", (Bi * Pz,), torch.float32)
        for j in range(nt):  # image group g feeds joint rows of texts g*nt + j: row remap (group stride nt*Sj, offset j*Sj)
            ops.layernorm_fwd(xsum_z, joint_in, st.P("vision_backbone/LayerNorm_final_ln/gamma"),
                              st.P("vision_backbone/LayerNorm_final_ln/beta"), mean_z, rstd_z, rows=Bi * Pz, remap=(Pz, nt * Sj, j * Sj))

        # ---- language-only encoder + masking (:135-139) ----
        ids_bl = self.input_ids.reshape(B, Lj)
        if self._mask_input:
            torch.cuda.current_stream().wait_stream(side)
            if mask_override is not None:
                self.lang_mask_info = {"masked_ids": mask_override["masked_ids"].to(dev).to(torch.int32).reshape(B, Lj).contiguous(),
                                       "masked_idx": mask_override["masked_idx"].to(dev).to(torch.int32).contiguous()}
            else:
                self.lang_mask_info = self.mask_inputs(mask_draws)
            ids_to_use = self.lang_mask_info["masked_ids"].reshape(B, Lj)
        else:
            ids_to_use = ids_bl
        self._ids_j = ids_to_use.contiguous()

        # ---- joint encoder (:143-184) ----
        self._embed_words_into(self._ids_j, "position_embeddings", "emb_j", _SITE_EMB_J, joint_in, remap=(Lj, Sj, Pz))
        valid_j = bf.get("joint.valid", (B * Sj,), torch.uint8)
        ops.joint_valid(self._ids_j, valid_j, B, Pz, Lj)
        c_viz = c_lang = None
        if self._log_attention_probs:  # split column sums of the joint attention maps for attention_log (:186-203)
            c_viz = bf.get("joint.c_viz", (B * Sj,), torch.float32, zero=True)
            c_lang = bf.get("joint.c_lang", (B * Sj,), torch.float32, zero=True)
        probs_j = None
        if self._export_probs:
            probs_j = bf.get("joint.probs", (cfg["num_hidden_layers"], B, Sj, Sj), torch.float32)
        self._joint = _Stack(st, bf, "joint", "encoder", cfg["num_hidden_layers"], B, Sj, valid_j, joint_in, cfg,
                             p_hid if train else 0.0, self._seed, _SITE_JOINT, self._save, colsum=c_viz, colsum2=c_lang,
                             colsum_split=Pz, colsum_valid_q=1, probs=probs_j,
                             # :160-168: language chunks attend to the vision tokens and to themselves only
                             pair=(Pz, self.lang_chunk_length) if cfg.get("disable_pairwise_lang_attn", False) else (0, 0))
        self._y_j = self._joint.forward()
        self._attn_log = None
        if self._log_attention_probs:
            out4 = bf.get("joint.attn_log", (4,), torch.float32)
            L.lib().merlot_attention_log_blocks(c_viz.data_ptr(), c_lang.data_ptr(), valid_j.data_ptr(), B, Sj, Pz,
                                                out4.data_ptr(), ops._stream())
            self._attn_log = out4
        self.encoder_info = {"hidden_state": self._y_j.view(B, Sj, H)}
        if probs_j is not None:  # [layers,B,S,S] -> the reference's [B, layers, S, S] (utils/transformer.py:238), a view
            self.encoder_info["self_attn_probs"] = probs_j.permute(1, 0, 2, 3)
        self._hidden_f32 = {}
        self.encoder_pieces = [{"name": "viz", "start": 0, "end": Pz}, {"name": "lang", "start": Pz, "end": Sj}]
        self._heads = {}

    def _hybrid_stem(self, img, N, h0, w0):
        """lite_resnet50 (utils/vision_transformer.py:118-170): NHWC bf16 activations as [N*h*w, C] matrices, every conv a K1 GEMM
        on weight-standardised bf16 kernels (1x1: the activation matrix itself; 3x3: an im2col matrix), GroupNorm32 (+ReLU /
        +shortcut) and the avg-pool striding as K13 kernels (csrc/stem.cu).  Variables are consumed in the reference's creation
        order (params.stem_variables).  With save_for_backward every op keeps its own buffers and is recorded on a tape for
        _hybrid_stem_backward.  Returns ([N*h*w, 4*f_last] bf16, h, w)."""
        st, bf = self.store, self._bufs
        vt = "vision_backbone/vision_transformer"
        save = bool(getattr(self, "_save", False))
        tape = []
        site = [0]

        class _Names:  # tf default-name uniquification inside one variable scope
            def __init__(self, scope):
                self.scope, self.nc, self.ng = scope, 0, 0

            def conv(self):
                n = f"{self.scope}/conv2d{'' if self.nc == 0 else '_%d' % self.nc}/kernel"
                self.nc += 1
                return n

            def gn(self, name=None):
                if name is not None:
                    return f"{self.scope}/GroupNorm_{name}"
                n = f"{self.scope}/GroupNorm{'' if self.ng == 0 else '_%d' % self.ng}"
                self.ng += 1
                return n

        def T(tag, rows, cols):  # training: one buffer per op (the backward pass reads them); inference: reuse by tag and shape
            site[0] += 1
            return bf.get(f"stem.{tag}.{site[0]}" if save else f"stem.{tag}", (rows, cols), torch.bfloat16)

        plan = self._ws_plan()
        plan.standardise()  # :56-60 (fp32 moments, bf16 operand) for every conv kernel of the stem in one launch

        def conv(x, h, w, cin, kname, k, tag, stride=1, sub_half=False):
            wk = st.P(kname)  # fp32 [k*k*cin, cout]
            rows, cout = wk.shape
            assert rows == k * k * cin, (kname, rows, k, cin)
            kp = (rows + 7) // 8 * 8
            wstd = plan.wstd[kname]
            if k == 1:
                a, ho, wo = x, h, w
            else:
                ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
                a = bf.get("stem.col", (N * ho * wo, kp), torch.bfloat16)  # recomputed in the backward pass: never per-op
                ops.im2col3x3(x, N, h, w, cin, stride, a, sub_half=sub_half)
            y = T(tag, N * ho * wo, cout)
            ops.gemm(a, wstd, b_mn_major=True, out=y)
            tape.append(("conv", dict(x=x, h=h, w=w, cin=cin, kname=kname, k=k, stride=stride, sub_half=sub_half, y=y, ho=ho, wo=wo,
                                      cout=cout, kp=kp)))
            return y, ho, wo, cout

        def gn(x, hw, c, scope_name, tag, relu=True, shortcut=None):
            y = T(tag, N * hw, c)
            stats = bf.get(f"stem.gn_stats.{site[0]}" if save else "stem.gn_stats", (N * 64,), torch.float32)
            ops.group_norm_fwd(x, st.P(f"{scope_name}/gamma"), st.P(f"{scope_name}/beta"), y, stats, N, hw, c, 32, 1e-4, relu, shortcut)
            tape.append(("gn", dict(x=x, y=y, scope=scope_name, hw=hw, c=c, relu=relu, shortcut=shortcut, stats=stats)))
            return y

        def pool(x, h, w, c, tag):
            ho, wo = (h + 1) // 2, (w + 1) // 2
            y = T(tag, N * ho * wo, c)
            ops.avgpool2_same(x, N, h, w, c, y)
            tape.append(("pool", dict(x=x, h=h, w=w, c=c, y=y)))
            return y, ho, wo

        nm = _Names(f"{vt}/resnet50lite/stem")
        x, h, w, c = conv(img, h0, w0, 3, nm.conv(), 3, "s0", stride=2, sub_half=True)  # :138-144 on image - 0.5 (:193)
        x = gn(x, h * w, c, nm.gn("stem0"), "s0g")
        x, h, w, c = conv(x, h, w, c, nm.conv(), 3, "s1")
        x = gn(x, h * w, c, nm.gn("stem1"), "s1g")
        x, h, w, c = conv(x, h, w, c, nm.conv(), 3, "s2")
        x = gn(x, h * w, c, nm.gn("stem2"), "s2g")
        x, h, w = pool(x, h, w, c, "s2p")  # :159
        for i, blocks in enumerate(self._resnet_layers):
            nm = _Names(f"{vt}/resnet50lite/block_group{i + 1}")
            f = 64 * (2 ** i)
            for b in range(blocks):  # bottleneck_block (:69-96); only the first block of a group projects and strides (:109-113)
                stride = 2 if (b == 0 and i > 0) else 1
                shortcut = x
                if b == 0:
                    sx, sh, sw = pool(x, h, w, c, f"g{i}sp") if stride > 1 else (x, h, w)
                    sy, _, _, c4 = conv(sx, sh, sw, c, nm.conv(), 1, f"g{i}sc")
                    shortcut = gn(sy, sh * sw, c4, nm.gn(), f"g{i}scg", relu=False)
                y, _, _, c1 = conv(x, h, w, c, nm.conv(), 1, f"g{i}a")
                y = gn(y, h * w, c1, nm.gn(), f"g{i}ag")
                y, _, _, c2 = conv(y, h, w, c1, nm.conv(), 3, f"g{i}b")
                y = gn(y, h * w, c2, nm.gn(), f"g{i}bg")
                hh, ww = h, w
                if stride > 1:
                    y, hh, ww = pool(y, h, w, c2, f"g{i}bp")
                y, _, _, c3 = conv(y, hh, ww, c2, nm.conv(), 1, f"g{i}c")
                x = gn(y, hh * ww, c3, nm.gn(), f"g{i}out{b % 2}", relu=True, shortcut=shortcut)  # relu(GN(y) + shortcut) (:95-96)
                h, w, c = hh, ww, c3
                assert c3 == 4 * f
        self._stem_tape = tape if save else None
        return x, h, w

    def _ws_plan(self):
        """The stem's conv kernels as one table (ops.WsPlan), cached on the store (the arenas' addresses never change)."""
        st = self.store
        names = [n for n in st.entries if "resnet50lite" in n and n.endswith("/kernel")]
        key = tuple(st.P(n).data_ptr() for n in names)
        plan = getattr(st, "_ws_plan_cache", None)
        if plan is None or plan.key != key:
            plan = ops.WsPlan({n: st.P(n) for n in names}, {n: st.G(n) for n in names}, st.device)
            st._ws_plan_cache = plan
        return plan

    def _hybrid_stem_backward(self, d_out, N):
        """Gradient of _hybrid_stem: walks the tape backwards.  d_out: bf16 gradient of the stem output.  Parameter gradients are
        ACCUMULATED into the arena (conv kernels through the weight-standardisation backward, GroupNorm gamma/beta directly);
        activation gradients meet by tensor identity (a block input feeds the first 1x1 and the shortcut)."""
        st, bf = self.store, self._bufs
        tape = self._stem_tape
        trace = getattr(self, "_stem_trace", None)  # tests set this to a list: every op's (dy, dx, d_shortcut) is recorded
        grads = {tape[-1][1]["y"].data_ptr(): d_out}
        red = bf.get("stem.gn_red", (N * 64,), torch.float32)
        ctr = [0]
        plan = self._ws_plan()  # holds the forward's standardised operands; the wgrad GEMMs accumulate into its gradient arena
        plan.zero_grads()

        def D(rows, cols):
            ctr[0] += 1
            return bf.get(f"stem.d.{ctr[0]}", (rows, cols), torch.bfloat16)

        def acc(t, g):
            k = t.data_ptr()
            if k in grads:
                ops.add_bf16(grads[k], g, grads[k])
            else:
                grads[k] = g

        for kind, r in reversed(tape):
            dy = grads.pop(r["y"].data_ptr(), None)
            if dy is None:
                continue
            if kind == "gn":
                dx = D(*r["x"].shape)
                dsc = D(*r["y"].shape) if r["shortcut"] is not None else None
                ops.group_norm_bwd(dy, r["x"], r["y"] if r["relu"] else None, r["stats"], st.P(f"{r['scope']}/gamma"), dx, dsc,
                                   st.G(f"{r['scope']}/gamma"), st.G(f"{r['scope']}/beta"), red, N, r["hw"], r["c"], 32, 1e-4, r["relu"])
                if trace is not None:
                    trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=dx.clone(), dsc=None if dsc is None else dsc.clone()))
                acc(r["x"], dx)
                if dsc is not None:
                    acc(r["shortcut"], dsc)
            elif kind == "pool":
                dx = D(*r["x"].shape)
                ops.avgpool2_same_bwd(dy, N, r["h"], r["w"], r["c"], dx)
                if trace is not None:
                    trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=dx.clone()))
                acc(r["x"], dx)
            else:  # conv
                wk = st.P(r["kname"])
                kp, cout, M = r["kp"], r["cout"], N * r["ho"] * r["wo"]
                if r["k"] == 1:
                    a = r["x"]
                else:
                    a = bf.get("stem.col", (M, kp), torch.bfloat16)
                    ops.im2col3x3(r["x"], N, r["h"], r["w"], r["cin"], r["stride"], a, sub_half=r["sub_half"])
                dws = plan.dws[r["kname"]]
                ops.gemm(a, dy, a_mn_major=True, b_mn_major=True, out=dws, atomic=True, M=kp, N=cout, K=M)  # d(standardised kernel)
                if r["sub_half"]:
                    if trace is not None:
                        trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=None))
                    continue  # the image itself needs no gradient
                wstd = plan.wstd[r["kname"]]
                if r["k"] == 1:
                    dx = D(M, kp)
                    ops.gemm(dy, wstd, out=dx)  # dx[M, cin] = dy[M, cout] . wstd[cin, cout]^T
                else:
                    dcol = bf.get("stem.dcol", (M, kp), torch.bfloat16)
                    ops.gemm(dy, wstd, out=dcol)
                    dx = D(N * r["h"] * r["w"], r["cin"])
                    ops.col2im3x3(dcol, N, r["h"], r["w"], r["cin"], r["stride"], dx)
                if trace is not None:
                    trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=dx.clone()))
                acc(r["x"], dx)
        plan.backward()  # weight-standardisation backward of every conv kernel: arena gradients += d(standardise)/dw . dws

    def _side_stream(self):
        """Stream for the language-only stack (set MERLOT_NO_SIDE_STREAM=1 to serialise everything on one stream)."""
        st = self.store
        if os.environ.get("MERLOT_NO_SIDE_STREAM", "0") == "1":
            return torch.cuda.current_stream()
        if not hasattr(st, "_side"):
            st._side = torch.cuda.Stream(device=st.device)
        return st._side

    # ---------------------------------------------------------------------------------------------------------
    def _embed_words_into(self, ids_2d, norm_scope_name, tag, site, out, remap):
        """embed_words (:262-297): E[ids] + Pos[0:L] -> LN embed_norm -> dropout -> bf16, written into `out` rows."""
        st, bf, cfg = self.store, self._bufs, self.config
        H = self.hidden_size
        R, Lseq = ids_2d.numel(), ids_2d.shape[1]
        if Lseq > cfg["max_position_embeddings"]:  # tf.assert_less_equal, utils/model_utils.py:282
            raise ValueError(f"sequence length {Lseq} exceeds max_position_embeddings {cfg['max_position_embeddings']}")
        xsum = bf.get(f"{tag}.xsum", (R, H), torch.float32)
        ops.embed_fwd(ids_2d, st.P("word_embeddings/word_embeddings"), st.P(f"{norm_scope_name}/position_embeddings"), xsum, Lseq)
        mean, rstd = bf.get(f"{tag}.mean", (R,), torch.float32), bf.get(f"{tag}.rstd", (R,), torch.float32)
        p = float(self.dropout_prob or 0.0) if self.is_training else 0.0
        ops.layernorm_fwd(xsum, out, st.P(f"{norm_scope_name}/LayerNorm_embed_norm/gamma"),
                          st.P(f"{norm_scope_name}/LayerNorm_embed_norm/beta"), mean, rstd, rows=R, remap=remap,
                          dropout=(p, self._seed, site))
        return xsum, mean, rstd

    def embed_words(self, input_ids_2d, norm_scope_name="position_embeddings", reuse=None):
        """Public mirror of :262-297; returns bf16 [B, L, H]."""
        get_shape_list_rank(input_ids_2d, 2, "input_ids_2d")
        ids = input_ids_2d.to(torch.int32).contiguous()
        out = torch.empty((ids.numel(), self.hidden_size), dtype=torch.bfloat16, device=ids.device)
        self._embed_words_into(ids, norm_scope_name, f"emb_pub.{norm_scope_name}", _SITE_EMB_J, out, (0, 0, 0))
        return out.view(ids.shape[0], ids.shape[1], -1)

    def _langonly_reps(self):
        """langonly_reps (:339-379)."""
        cfg, st, bf = self.config, self.store, self._bufs
        H = self.hidden_size
        if "langonly_num_chunks_in_group" in cfg:
            g = cfg["langonly_num_chunks_in_group"]
            ng = self.num_chunks // g
            assert ng > 0
            assert self.num_chunks % g == 0
            ids = self.input_ids.reshape(self.batch_size * ng, self.lang_chunk_length * g)
        else:
            ids = self.input_ids.reshape(self.batch_size, self.lang_chunk_length * self.num_chunks)
        ids = ids.contiguous()
        Blo, Llo = ids.shape
        self._ids_lo = ids
        h0 = bf.get("lo.h0", (Blo * Llo, H), torch.bfloat16)
        self._embed_words_into(ids, "langonly_embeddings", "emb_lo", _SITE_EMB_LO, h0, (0, 0, 0))
        valid = bf.get("lo.valid", (Blo * Llo,), torch.uint8)
        ops.ids_valid(ids, valid)
        summ = bf.get("lo.attn_summ", (Blo * Llo,), torch.float32, zero=True)
        p = float(self.dropout_prob or 0.0) if self.is_training else 0.0
        probs_lo = None
        if self._export_probs:
            probs_lo = bf.get("lo.probs", (cfg["num_lang_transformer_hidden_layers"], Blo, Llo, Llo), torch.float32)
        self._lo = _Stack(st, bf, "lo", "encoder", cfg["num_lang_transformer_hidden_layers"], Blo, Llo, valid, h0, cfg, p,
                          self._seed, _SITE_LANGONLY, self._save, colsum=summ, probs=probs_lo)
        y = self._lo.forward()
        nch = self.batch_size * self.num_chunks
        pool_idx = bf.get("lo.pool_idx", (nch,), torch.int32)
        pool_idx.copy_(torch.arange(nch, dtype=torch.int32, device=st.device) * self.lang_chunk_length)
        self._pool_idx_lo = pool_idx
        self.lang_trg_h = bf.get("lo.lang_trg", (nch, H), torch.float32)
        ops.gather_rows(y, pool_idx, self.lang_trg_h)
        # attention_summs of mask_inputs (:428-431): sum over (layers, queries) of head-mean probabilities, as [B, L]
        self.lang_transformer_info = {"hidden_state": y.view(Blo, Llo, H), "attention_summs": summ.view(self.B, self.L)}
        if probs_lo is not None:
            self.lang_transformer_info["self_attn_probs"] = probs_lo.permute(1, 0, 2, 3)
        return self.lang_trg_h, self.lang_transformer_info

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
    def _dense_f32(self, x_bf16, scope, out):
        """tf.layers.dense on a small head tensor: bf16 operands, fp32 accumulate/output (+bias)."""
        st = self.store
        return ops.gemm(x_bf16, st.W(f"{scope}/kernel"), b_mn_major=True, bias=st.P(f"{scope}/bias"), out=out)

    def _mlp_ln(self, tag, x_bf16, dense_scope, ln_scope, R, Hout):
        """dense + gelu -> layer_norm (the repeated head pattern, e.g. :28-35, :208-215, :582-589). Returns bf16 output."""
        st, bf = self.store, self._bufs
        pre = bf.get(f"{tag}.pre", (R, Hout), torch.float32)
        self._dense_f32(x_bf16, dense_scope, pre)
        act = bf.get(f"{tag}.act", (R, Hout), torch.float32)
        ops.gelu_f32(pre, act)
        an = bf.get(f"{tag}.an", (R, Hout), torch.bfloat16)
        mean, rstd = bf.get(f"{tag}.mean", (R,), torch.float32), bf.get(f"{tag}.rstd", (R,), torch.float32)
        ops.layernorm_fwd(act, an, st.P(f"{ln_scope}/gamma"), st.P(f"{ln_scope}/beta"), mean, rstd, rows=R)
        return dict(x=x_bf16, pre=pre, act=act, an=an, mean=mean, rstd=rstd, dense=dense_scope, ln=ln_scope, R=R, Hout=Hout, tag=tag)

    def _mlp_ln_bwd(self, t, d_an_f32, need_dx=True):
        """Backward of _mlp_ln: accumulates parameter grads, returns d_x fp32 [R, Hin]."""
        st, bf = self.store, self._bufs
        R, Hout, tag = t["R"], t["Hout"], t["tag"]
        d_act = bf.get(f"{tag}.d_act", (R, Hout), torch.float32)
        ops.layernorm_bwd(d_an_f32, t["act"], t["mean"], t["rstd"], st.P(f"{t['ln']}/gamma"), d_act, st.G(f"{t['ln']}/gamma"),
                          st.G(f"{t['ln']}/beta"), rows=R)
        d_pre = bf.get(f"{tag}.d_pre", (R, Hout), torch.float32)
        ops.gelu_bwd_f32(d_act, t["pre"], d_pre)
        return self._dense_bwd(tag, t["x"], t["dense"], d_pre, need_dx)

    def _dense_bwd(self, tag, x_bf16, scope, dy_f32, need_dx=True):
        st, bf = self.store, self._bufs
        R, N = dy_f32.shape
        Kin = x_bf16.shape[1]
        ops.bias_grad(dy_f32, st.G(f"{scope}/bias"), rows=R, N=N)
        dyb = bf.get(f"{tag}.dyb.{scope}", (R, N), torch.bfloat16)
        ops.cast_f32_to_bf16(dy_f32, dyb)
        ops.gemm(x_bf16, dyb, a_mn_major=True, b_mn_major=True, out=st.G(f"{scope}/kernel"), atomic=True, M=Kin, N=N, K=R)
        if not need_dx:
            return None
        dx = bf.get(f"{tag}.dx.{scope}", (R, Kin), torch.float32)
        ops.gemm(dyb, st.W(f"{scope}/kernel"), out=dx, M=R, N=Kin, K=N)
        return dx

    def lm_head(self, hidden_state):
        """lm_head (:205-224) on bf16 rows [R,H]; returns fp32 logits [R, ldV] (columns >= vocab_size are padding)."""
        return self._lm_head("lm_pub", hidden_state.contiguous())["logits"][:, :self.vocab_size]

    def _lm_head(self, tag, pooled):
        cfg, st, bf = self.config, self.store, self._bufs
        R, H, V = pooled.shape[0], self.hidden_size, self.vocab_size
        t = {}
        hn = pooled
        if cfg.get("do_projection", False):
            t = self._mlp_ln(f"{tag}.proj", pooled, "lm_head/projection", "lm_head/LayerNorm", R, H)
            hn = t["an"]
        ldV = (V + 63) // 64 * 64
        logits = bf.get(f"{tag}.logits", (R, ldV), torch.float32)
        bias = st.P("lm_head/output_bias") if cfg.get("do_bias", False) else None
        ops.gemm(hn, st.W("word_embeddings/word_embeddings"), bias=bias, out=logits, M=R, N=V, K=H)
        return dict(proj=t, hn=hn, logits=logits, ldV=ldV)

    def mask_loss(self):
        """mask_loss (:528-551).  Returns (loss, {'loss','acc'}) as 0-d CUDA tensors."""
        bf = self._bufs
        B, Lj, V = self.B, self.L, self.vocab_size
        k = self.lang_mask_info["masked_idx"].shape[1]
        nm = B * k
        rows = bf.get("mlm.rows", (nm,), torch.int32)
        targets = bf.get("mlm.targets", (nm,), torch.int32)
        ops.mlm_index(self.input_ids.reshape(B, Lj), self.lang_mask_info["masked_idx"], rows, targets, B, Lj, k, self._dims["Pz"])
        pooled = bf.get("mlm.pooled", (nm, self.hidden_size), torch.bfloat16)
        ops.gather_rows(self._y_j, rows, pooled)
        hd = self._lm_head("mlm", pooled)
        per, lse, corr = (bf.get(f"mlm.{n}", (nm,), torch.float32) for n in ("l", "lse", "corr"))
        ops.softmax_ce_fwd(hd["logits"], targets, V, per, lse, corr)
        out2 = bf.get("mlm.out", (2,), torch.float32)
        coeff = bf.get("mlm.coeff", (nm,), torch.float32)
        ops.weighted_loss(per, corr, None, targets, 1, 1.0, out2, coeff)
        self._heads["mlm"] = dict(rows=rows, targets=targets, pooled=pooled, lse=lse, coeff=coeff, nm=nm, **hd)
        return out2[0], {"loss": out2[0], "acc": out2[1]}

    def _mask_loss_bwd(self, d_yj):
        st, bf = self.store, self._bufs
        h = self._heads["mlm"]
        V, H, nm, ldV = self.vocab_size, self.hidden_size, h["nm"], h["ldV"]
        dlog = bf.get("mlm.dlogits", (nm, ldV), torch.bfloat16)
        ops.softmax_ce_bwd(h["logits"], h["targets"], V, h["lse"], h["coeff"], dlog)
        if self.config.get("do_bias", False):
            gb = st.G("lm_head/output_bias")
            gb_pad = st.g[st.entries["lm_head/output_bias"].offset:st.entries["lm_head/output_bias"].offset + ldV]
            ops.bias_grad(dlog, gb_pad, rows=nm, N=ldV)
        # tied embedding: dE += dlogits^T hn ; d_hn = dlogits E
        ops.gemm(dlog, h["hn"], a_mn_major=True, b_mn_major=True, out=st.G("word_embeddings/word_embeddings"), atomic=True,
                 M=V, N=H, K=nm)
        d_hn = bf.get("mlm.d_hn", (nm, H), torch.float32, zero=True)  # split-K over the 50370-long contraction
        ops.gemm(dlog, st.W("word_embeddings/word_embeddings"), b_mn_major=True, out=d_hn, atomic=True, M=nm, N=H, K=V)
        d_pooled = self._mlp_ln_bwd(h["proj"], d_hn) if h["proj"] else d_hn
        ops.scatter_add_rows(d_pooled, h["rows"], d_yj)

    def _tower(self, tag, x_f32, name):
        """project_and_norm (:18-44) under scope 'contrastive'."""
        cfg, bf = self.config, self._bufs
        n, H = x_f32.shape
        Cs = cfg.get("contrastive_size", H)
        xb = bf.get(f"{tag}.xb", (n, H), torch.bfloat16)
        ops.cast_f32_to_bf16(x_f32, xb)
        t = {}
        inp = xb
        if cfg.get("do_projection", False):
            t = self._mlp_ln(f"{tag}.inter", xb, f"contrastive/{name}_intermediate", f"contrastive/LayerNorm_{name}_ln", n, Cs)
            inp = t["an"]
        proj = bf.get(f"{tag}.proj", (n, Cs), torch.float32)
        self._dense_f32(inp, f"contrastive/{name}", proj)
        feat = bf.get(f"{tag}.feat", (n, Cs), torch.float32)
        inv = bf.get(f"{tag}.inv", (n,), torch.float32)
        ops.l2norm_fwd(proj, feat, inv)
        return dict(tag=tag, name=name, xb=xb, inter=t, inp=inp, feat=feat, inv=inv, n=n, Cs=Cs)

    def _tower_bwd(self, t, d_feat):
        bf = self._bufs
        d_proj = bf.get(f"{t['tag']}.d_proj", (t["n"], t["Cs"]), torch.float32)
        ops.l2norm_bwd(d_feat, t["feat"], t["inv"], d_proj)
        d_inp = self._dense_bwd(t["tag"], t["inp"], f"contrastive/{t['name']}", d_proj)
        return self._mlp_ln_bwd(t["inter"], d_inp) if t["inter"] else d_inp

    def contrastive_loss(self):
        """contrastive_loss (:491-526).  Multi-GPU: features are all-gathered over the data-parallel group
        (tpu_cross_replica_stack, utils/model_utils.py:673-707) and labels are offset by rank*N (:519)."""
        cfg, bf = self.config, self._bufs
        lang = self._tower("ctr.lang", self.lang_trg_h, "lang_proj")
        viz = self._tower("ctr.viz", self.img_trg_h, "viz_proj")
        n, Cs = lang["n"], lang["Cs"]
        world, rank = (self.dist.world, self.dist.rank) if self.dist is not None else (1, 0)
        if world > 1:
            all_lang, all_viz = self.dist.all_gather_rows(lang["feat"]), self.dist.all_gather_rows(viz["feat"])
        else:
            all_lang, all_viz = lang["feat"], viz["feat"]
        temp = cfg.get("contrast_temp", 0.05)
        coef = cfg.get("contrast_coef", 1.0)
        labels = bf.get("ctr.labels", (n,), torch.int32)
        labels.copy_(torch.arange(n, dtype=torch.int32, device=labels.device) + rank * n)
        nW = n * world
        outs = {}
        info = dict(lang=lang, viz=viz, all_lang=all_lang, all_viz=all_viz, labels=labels, nW=nW, temp=temp, dirs={})
        for name, x, y in (("lang_to_viz", lang["feat"], all_viz), ("viz_to_lang", viz["feat"], all_lang)):
            logits = bf.get(f"ctr.{name}.logits", (n, nW), torch.float32)
            ops.small_gemm(x, Cs, 1, y, Cs, 1, logits, n, nW, Cs, alpha=1.0 / temp)
            per, lse = bf.get(f"ctr.{name}.l", (n,), torch.float32), bf.get(f"ctr.{name}.lse", (n,), torch.float32)
            ops.softmax_ce_fwd(logits, labels, nW, per, lse, None)
            out2 = bf.get(f"ctr.{name}.out", (2,), torch.float32)
            coeff = bf.get(f"ctr.{name}.coeff", (n,), torch.float32)
            ops.weighted_loss(per, None, None, None, 0, coef / 2.0, out2, coeff)
            outs[name] = out2[0]
            info["dirs"][name] = dict(logits=logits, lse=lse, coeff=coeff)
        loss_all = bf.get("ctr.loss_all", (1,), torch.float32)
        ops.axpby(bf.get("ctr.lang_to_viz.out", (2,), torch.float32)[:1], loss_all, coef / 2.0, 0.0)
        ops.axpby(bf.get("ctr.viz_to_lang.out", (2,), torch.float32)[:1], loss_all, coef / 2.0, 1.0)
        outs["loss_all"] = loss_all[0]
        self._heads["ctr"] = info
        return loss_all[0], outs

    def _contrastive_bwd(self, d_lang_trg, d_img_trg):
        bf = self._bufs
        c = self._heads["ctr"]
        lang, viz, nW, temp = c["lang"], c["viz"], c["nW"], c["temp"]
        n, Cs = lang["n"], lang["Cs"]
        world = self.dist.world if self.dist is not None else 1
        d_feat = {"lang": bf.get("ctr.d_feat.lang", (n, Cs), torch.float32), "viz": bf.get("ctr.d_feat.viz", (n, Cs), torch.float32)}
        d_all = {"lang": bf.get("ctr.d_all.lang", (nW, Cs), torch.float32), "viz": bf.get("ctr.d_all.viz", (nW, Cs), torch.float32)}
        for name, xk, yk, y_all in (("lang_to_viz", "lang", "viz", c["all_viz"]), ("viz_to_lang", "viz", "lang", c["all_lang"])):
            d = c["dirs"][name]
            dlog = bf.get(f"ctr.{name}.dlogits", (n, nW), torch.float32)
            ops.softmax_ce_bwd(d["logits"], c["labels"], nW, d["lse"], d["coeff"], dlog)
            x = c[xk]["feat"]
            # d_x[i,c] = sum_j dlog[i,j] y_all[j,c] / temp
            ops.small_gemm(dlog, nW, 1, y_all, 1, Cs, d_feat[xk], n, Cs, nW, alpha=1.0 / temp, beta=0.0)
            # d_y_all[j,c] = sum_i dlog[i,j] x[i,c] / temp
            ops.small_gemm(dlog, 1, nW, x, 1, Cs, d_all[yk], nW, Cs, n, alpha=1.0 / temp, beta=0.0)
        for k in ("lang", "viz"):
            # gradient of the gather = reduce-scatter(sum) of every rank's d_all (utils/model_utils.py:699-706)
            mine = self.dist.reduce_scatter_rows(d_all[k]) if world > 1 else d_all[k]
            ops.axpby(mine, d_feat[k], 1.0, 1.0)
        dl = self._tower_bwd(lang, d_feat["lang"])
        dv = self._tower_bwd(viz, d_feat["viz"])
        ops.axpby(dl, d_lang_trg, 1.0, 1.0)
        ops.axpby(dv, d_img_trg, 1.0, 1.0)

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
        return self._temporal_head(f"tmp_pub.{scope_name}", scope_name, xa2, xb2)["logits"][:, :4]

    def _temporal_head(self, tag, scope, xa_bf16, xb_bf16):
        st, bf = self.store, self._bufs
        B, n, H = self.B, self.num_chunks_in_group, self.hidden_size
        _, _, idxA, idxB = self._temporal_index()
        R = B * n * n
        hj = bf.get(f"{tag}.hj", (R, 2 * H), torch.bfloat16)
        ops.gather_rows(xa_bf16, idxA, hj[:, :H], H=H)
        ops.gather_rows(xb_bf16, idxB, hj[:, H:], H=H)
        t = self._mlp_ln(f"{tag}.mlp", hj, f"{scope}/intermediate", f"{scope}/LayerNorm_ln0", R, H)
        logits = bf.get(f"{tag}.logits", (R, 8), torch.float32)
        self._dense_f32(t["an"], f"{scope}/logits", logits)
        return dict(tag=tag, scope=scope, hj=hj, mlp=t, logits=logits, R=R)

    def allpairs_temporal_labels(self, video_src_ids, shuffled_idx_img=None):
        """allpairs_temporal_labels (:598-620)."""
        bf = self._bufs
        B, n = self.B, self.num_chunks_in_group
        labels = bf.get("tmp.labels", (B * n * n,), torch.int32)
        w = bf.get("tmp.w", (B * n * n,), torch.float32)
        v = video_src_ids.reshape(B, n).to(torch.int32).contiguous()
        s = (shuffled_idx_img if shuffled_idx_img is not None else torch.zeros_like(v)).reshape(B, n).to(torch.int32).contiguous()
        ops.temporal_labels(v, s, labels, w, B, n)
        self._tmp_w = w
        return labels

    def temporal_loss(self, shuffled_idx_img, video_src_ids):
        """temporal_loss (:622-668)."""
        cfg, bf = self.config, self._bufs
        B, n, H = self.B, self.num_chunks_in_group, self.hidden_size
        idx_l, idx_v, _, _ = self._temporal_index()
        h_lang = bf.get("tmp.h_lang", (B * n, H), torch.bfloat16)
        h_viz = bf.get("tmp.h_viz", (B * n, H), torch.bfloat16)
        ops.gather_rows(self._y_j, idx_l, h_lang)
        ops.gather_rows(self._y_j, idx_v, h_viz)
        labels = self.allpairs_temporal_labels(video_src_ids, shuffled_idx_img)
        w = self._tmp_w
        coef = cfg.get("temporal_coef", 1.0)
        use_vv = cfg.get("image_shuffle_prob", 0) > 0  # :664-665
        info, heads = {}, {}
        for name, xa, xb in (("lang_viz", h_lang, h_viz), ("viz_viz", h_viz, h_viz)):
            hd = self._temporal_head(f"tmp.{name}", f"{name}_temporal", xa, xb)
            R = hd["R"]
            per, lse, corr = (bf.get(f"tmp.{name}.{k}", (R,), torch.float32) for k in ("l", "lse", "corr"))
            ops.softmax_ce_fwd(hd["logits"], labels, 4, per, lse, corr)
            out2 = bf.get(f"tmp.{name}.out", (2,), torch.float32)
            coeff = bf.get(f"tmp.{name}.coeff", (R,), torch.float32)
            ops.weighted_loss(per, corr, w, None, 0, coef, out2, coeff)
            info[f"{name}_loss"], info[f"{name}_acc"] = out2[0], out2[1]
            heads[name] = dict(lse=lse, coeff=coeff, in_loss=(name == "lang_viz" or use_vv), **hd)
        tot = bf.get("tmp.loss", (1,), torch.float32)
        ops.axpby(bf.get("tmp.lang_viz.out", (2,), torch.float32)[:1], tot, 1.0, 0.0)
        if use_vv:
            ops.axpby(bf.get("tmp.viz_viz.out", (2,), torch.float32)[:1], tot, 1.0, 1.0)
        info["loss"] = tot[0]
        loss = bf.get("tmp.loss_scaled", (1,), torch.float32)
        ops.axpby(tot, loss, coef, 0.0)
        self._heads["tmp"] = dict(heads=heads, labels=labels, idx_l=idx_l, idx_v=idx_v)
        return loss[0], info

    def _temporal_bwd(self, d_yj):
        st, bf = self.store, self._bufs
        B, n, H = self.B, self.num_chunks_in_group, self.hidden_size
        t = self._heads["tmp"]
        _, _, idxA, idxB = self._temporal_index()
        d_hl = bf.get("tmp.d_hl", (B * n, H), torch.float32, zero=True)
        d_hv = bf.get("tmp.d_hv", (B * n, H), torch.float32, zero=True)
        for name, da, db in (("lang_viz", d_hl, d_hv), ("viz_viz", d_hv, d_hv)):
            hd = t["heads"][name]
            if not hd["in_loss"]:
                continue
            R, scope, tag = hd["R"], hd["scope"], hd["tag"]
            dlog = bf.get(f"{tag}.dlogits", (R, 8), torch.float32)
            ops.softmax_ce_bwd(hd["logits"], t["labels"], 4, hd["lse"], hd["coeff"], dlog)
            d_an = self._dense_bwd(tag, hd["mlp"]["an"], f"{scope}/logits", dlog)
            d_hj = self._mlp_ln_bwd(hd["mlp"], d_an)  # fp32 [R, 2H]
            ops.scatter_add_rows(d_hj[:, :H], idxA, da, H=H)
            ops.scatter_add_rows(d_hj[:, H:], idxB, db, H=H)
        ops.scatter_add_rows(d_hl, t["idx_l"], d_yj)
        ops.scatter_add_rows(d_hv, t["idx_v"], d_yj)

    # ---------------------------------------------------------------------------------------------------------
    # backward of the whole model: call after mask_loss / contrastive_loss / temporal_loss (whichever are in the loss)
    # ---------------------------------------------------------------------------------------------------------
    def backward(self, on_non_vit_grads_ready=None, vit_layer_groups=None, on_vit_group_done=None, d_hidden_state=None):
        """d(lang_loss + contr_loss + temp_loss)/d(params) accumulated into store.g  (model/modeling.py:713 loss,
        utils/optimization.py:176 tf.gradients).  Order: heads -> joint encoder -> language-only encoder -> (callback: every
        gradient outside vision_backbone/vision_transformer is final; data-parallel training starts their all-reduce here)
        -> ViT."""
        if not self._save:
            raise RuntimeError("MerlotModel was built without save_for_backward (is_training=False)")
        cfg, st, bf, D = self.config, self.store, self._bufs, self._dims
        H, B, Lj, N = self.hidden_size, self.B, self.L, D["N"]
        Sj, Pz, vcl, Sv, Mv, np_, ncls = D["Sj"], D["Pz"], D["vcl"], D["Sv"], D["Mv"], D["np"], D["ncls"]
        vt = "vision_backbone/vision_transformer"
        d_yj = bf.get("bwd.d_yj", (B * Sj, H), torch.bfloat16, zero=True)
        if d_hidden_state is not None:  # gradient of an external head (e.g. downstream/vcr's classifier) w.r.t. encoder_info['hidden_state']
            if tuple(d_hidden_state.shape) not in ((B * Sj, H), (B, Sj, H)) or d_hidden_state.dtype != torch.bfloat16:
                raise ValueError("d_hidden_state must be bf16 [B, P+L, H]")
            d_yj.copy_(d_hidden_state.reshape(B * Sj, H))
        d_img_trg = bf.get("bwd.d_img_trg", (N, H), torch.float32, zero=True)
        d_lang_trg = None
        if self._mask_input:
            d_lang_trg = bf.get("bwd.d_lang_trg", (self.batch_size * self.num_chunks, H), torch.float32, zero=True)
        if "mlm" in self._heads:
            self._mask_loss_bwd(d_yj)
        if "ctr" in self._heads:
            self._contrastive_bwd(d_lang_trg, d_img_trg)
        if "tmp" in self._heads:
            self._temporal_bwd(d_yj)
        p_emb = float(self.dropout_prob or 0.0)
        # ---- language-only encoder backward on the side stream: it needs only d_lang_trg (contrastive head) and runs
        # concurrently with the joint-encoder backward below, whose small grids leave a third of the SMs idle ----
        side = self._side_stream()
        main = torch.cuda.current_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            if self._mask_input:
                Blo, Llo = self._ids_lo.shape
                d_ylo = bf.get("bwd.d_ylo", (Blo * Llo, H), torch.bfloat16, zero=True)
                ops.scatter_add_rows(d_lang_trg, self._pool_idx_lo, d_ylo)
                d_h0lo = bf.get("bwd.d_h0lo", (Blo * Llo, H), torch.bfloat16)
                self._lo.backward(d_ylo, d_h0lo)
                self._embed_bwd("emb_lo", "langonly_embeddings", self._ids_lo, d_h0lo, (0, 0, 0), (p_emb, self._seed, _SITE_EMB_LO),
                                Blo, Llo)
        # ---- joint encoder ----
        d_jin = bf.get("bwd.d_jin", (B * Sj, H), torch.bfloat16)
        self._joint.backward(d_yj, d_jin)
        # lang piece: embed_norm(position_embeddings) -> word / position tables
        self._embed_bwd("emb_j", "position_embeddings", self._ids_j, d_jin, (Lj, Sj, Pz), (p_emb, self._seed, _SITE_EMB_J), B, Lj)
        # viz piece: final_ln -> K7 backward
        nt = self.num_texts
        Bi = B // nt
        dxz = None
        for j in range(nt):  # the nt texts of an image group all send gradient into the same viz tokens: summed through `dres`
            dxj = bf.get(f"bwd.dxsum_z.{j & 1}", (Bi * Pz, H), torch.float32)
            ops.layernorm_bwd(d_jin, bf.get("viz.xsum", (Bi * Pz, H), torch.float32), bf.get("viz.mean", (Bi * Pz,), torch.float32),
                              bf.get("viz.rstd", (Bi * Pz,), torch.float32), st.P("vision_backbone/LayerNorm_final_ln/gamma"), dxj,
                              st.G("vision_backbone/LayerNorm_final_ln/gamma"), st.G("vision_backbone/LayerNorm_final_ln/beta"),
                              dres=dxz, rows=Bi * Pz, remap=(Pz, nt * Sj, j * Sj))
            dxz = dxj
        d_hv = bf.get("bwd.d_hv", (Mv, H), torch.bfloat16)
        ops.viz_assemble_bwd(dxz, d_img_trg, d_hv, N, D["h1"], D["w1"], ncls, D["sp"], H)
        ops.segment_rowsum_scatter(dxz, N, vcl, self._img_idx, st.G("vision_backbone/img_idx_pe"), H)
        ops.group_rowsum(dxz, N, vcl, 0, 1, None, st.G("vision_backbone/final_pe/cls_emb"), H)
        ops.group_rowsum(dxz, N, vcl, 1, D["h2"] * D["w2"], self._grid_idxmap(D["h2"], D["w2"]),
                         st.G("vision_backbone/final_pe/pos_embs"), H)
        # join the language-only backward (side stream); every gradient outside the ViT is final now
        main.wait_stream(side)
        if on_non_vit_grads_ready is not None:
            on_non_vit_grads_ready()
        # ---- ViT ----
        d_h0v = bf.get("bwd.d_h0v", (Mv, H), torch.bfloat16)
        self._vit.backward(d_hv, d_h0v, vit_layer_groups, on_vit_group_done)
        dxv = bf.get("bwd.dxsum_v", (Mv, H), torch.float32)
        ops.layernorm_bwd(d_h0v, bf.get("vit.xsum", (Mv, H), torch.float32), bf.get("vit.mean0", (Mv,), torch.float32),
                          bf.get("vit.rstd0", (Mv,), torch.float32), st.P(f"{vt}/LayerNorm_ctx_patches_pre_ln/gamma"), dxv,
                          st.G(f"{vt}/LayerNorm_ctx_patches_pre_ln/gamma"), st.G(f"{vt}/LayerNorm_ctx_patches_pre_ln/beta"), rows=Mv)
        ops.group_rowsum(dxv, N, Sv, 0, ncls, None, st.G(f"{vt}/pos_embs/cls_emb"), H)
        ops.group_rowsum(dxv, N, Sv, ncls, np_, self._grid_idxmap(D["h1"], D["w1"]), st.G(f"{vt}/pos_embs/pos_embs"), H)
        dpatch = bf.get("bwd.dpatch", (N * np_, H), torch.bfloat16)
        ops.vit_assemble_bwd(dxv, dpatch, N, np_, ncls, H)
        if not self._resnet_layers:
            ops.bias_grad(dpatch, st.G(f"{vt}/conv2d/bias"), rows=N * np_, N=H)
            ops.gemm(bf.get("vit.A", (N * np_, D["Kp"]), torch.bfloat16), dpatch, a_mn_major=True, b_mn_major=True,
                     out=st.G(f"{vt}/conv2d/kernel"), atomic=True, M=D["Kp"], N=H, K=N * np_)
        else:  # conv_postresnet_proj (1x1 + bias, not standardised), then the stem's tape
            rc = self._stem_tape[-1][1]["y"]
            Cr = rc.shape[1]
            ops.bias_grad(dpatch, st.G(f"{vt}/conv_postresnet_proj/bias"), rows=N * np_, N=H)
            ops.gemm(rc, dpatch, a_mn_major=True, b_mn_major=True, out=st.G(f"{vt}/conv_postresnet_proj/kernel"), atomic=True,
                     M=Cr, N=H, K=N * np_)
            d_rc = bf.get("bwd.d_rc", (N * np_, Cr), torch.bfloat16)
            ops.gemm(dpatch, st.W(f"{vt}/conv_postresnet_proj/kernel"), out=d_rc)  # [M, H] . [Cr, H]^T
            self._hybrid_stem_backward(d_rc, N)
    def _embed_bwd(self, tag, norm_scope_name, ids_2d, dy, remap, dropout, groups, Lseq):
        st, bf = self.store, self._bufs
        H, R = self.hidden_size, ids_2d.numel()
        dx = bf.get(f"bwd.dxsum.{tag}", (R, H), torch.float32)
        ops.layernorm_bwd(dy, bf.get(f"{tag}.xsum", (R, H), torch.float32), bf.get(f"{tag}.mean", (R,), torch.float32),
                          bf.get(f"{tag}.rstd", (R,), torch.float32), st.P(f"{norm_scope_name}/LayerNorm_embed_norm/gamma"), dx,
                          st.G(f"{norm_scope_name}/LayerNorm_embed_norm/gamma"), st.G(f"{norm_scope_name}/LayerNorm_embed_norm/beta"),
                          rows=R, remap=remap, dropout=dropout if self.is_training else (0.0, 0, 0))
        ops.scatter_add_rows(dx, ids_2d.reshape(-1), st.G("word_embeddings/word_embeddings"))
        ops.group_rowsum(dx, groups, Lseq, 0, Lseq, None, st.G(f"{norm_scope_name}/position_embeddings"), H)

    def _grid_idxmap(self, nh, nw):
        key = ("_grid", nh, nw)
        d = self._bufs.d
        if key not in d:
            i = torch.arange(nh, device=self.store.device)[:, None]
            j = torch.arange(nw, device=self.store.device)[None]
            d[key] = (i * 64 + j).reshape(-1).to(torch.int32)
        return d[key]
