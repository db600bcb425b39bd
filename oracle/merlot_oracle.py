"""ORACLE -- TEST INFRASTRUCTURE ONLY.  CPU restatement (torch fp32/fp64, autograd) of rowanz/merlot's dense hot path.

PARITY UNPINNED: the reference ships no tests, golden vectors or fixtures (SURVEY.md section 4), and TensorFlow 1.15
cannot be installed in this environment (Python 3.12, no network), so this restatement cannot be checked against
outputs of the reference itself.  It is pinned only by (a) the hand-derived known-answer tests of SURVEY.md 8(c)
(tests/test_oracle_kats.py), (b) an independent NumPy-fp64 restatement of the primitives (oracle/oracle_np.py)
that must agree with this file to 1e-5, and (c) line-by-line citations of the reference source below.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
The product path (merlot_b200/) never does.

Third-party arithmetic restated here lives in TensorFlow 1.15.5 (requirements.txt:70, not vendored):
tf.layers.dense (y = x W + b, W [in,out]), tf.layers.conv2d (HWIO, NHWC), tf.nn.moments (biased variance),
tf.nn.softmax/log_softmax, tf.erf, tf.math.l2_normalize (x * rsqrt(max(sum x^2, 1e-12))), tf.nn.avg_pool2d VALID,
tf.math.top_k (ties -> lower index first), tf.argmax (first occurrence), tf.sort.

All `file:line` citations are relative to /root/reference.
Parameters are a dict keyed by the reference's TF variable names (SURVEY.md Appendix A).
"""
from __future__ import annotations

import copy
import math
import re
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

MASK = 1      # utils/encode/encoder.py:16-22
PADDING = 0
START = 2

Params = Dict[str, torch.Tensor]


# ------------------------------------------------------------------------------------------------------------
# primitives (utils/model_utils.py)
# ------------------------------------------------------------------------------------------------------------
def gelu(x: torch.Tensor) -> torch.Tensor:
    """utils/model_utils.py:96-110 -- x * 0.5 * (1 + erf(x / sqrt(2)))."""
    return x * (0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))))


def layer_norm(x: torch.Tensor, p: Params, scope: str, eps: float = 1e-5) -> torch.Tensor:
    """utils/model_utils.py:113-130 -- biased variance; y = x*s - mean*s + beta with s = rsqrt(var+eps)*gamma."""
    gamma, beta = p[f"{scope}/gamma"], p[f"{scope}/beta"]
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    s = torch.rsqrt(var + eps) * gamma
    return x * s - mean * s + beta


def dense(x: torch.Tensor, p: Params, scope: str, activation=None) -> torch.Tensor:
    """tf.layers.dense: x @ kernel[in,out] + bias."""
    y = x @ p[f"{scope}/kernel"] + p[f"{scope}/bias"]
    return activation(y) if activation is not None else y


def raw_cross_entropy_with_logits(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """utils/model_utils.py:313-332 -- -sum(one_hot * log_softmax)."""
    logp = F.log_softmax(logits, dim=-1)
    return -logp.gather(-1, labels.long().unsqueeze(-1)).squeeze(-1)


def l2_normalize(x: torch.Tensor) -> torch.Tensor:
    """tf.math.l2_normalize(axis=-1, epsilon=1e-12): x * rsqrt(max(sum(x^2), eps))."""
    return x * torch.rsqrt(torch.clamp((x * x).sum(-1, keepdim=True), min=1e-12))


def top_k_tf(x: torch.Tensor, k: int):
    """tf.math.top_k: descending values, ties broken by LOWER index first (stable sort of -x)."""
    vals, idx = torch.sort(-x, dim=-1, stable=True)
    return -vals[..., :k], idx[..., :k]


def position_embedder2d(p: Params, scope: str, num_h: int, num_w: int, num_cls_emb: int) -> torch.Tensor:
    """utils/model_utils.py:710-739 with num_img=1, max_nimg=1: [num_cls_emb + num_h*num_w, H]."""
    pe = p[f"{scope}/pos_embs"][0, :num_h, :num_w].reshape(num_h * num_w, -1)
    if num_cls_emb > 0:
        pe = torch.cat([p[f"{scope}/cls_emb"][0, :num_cls_emb], pe], 0)
    return pe


# ------------------------------------------------------------------------------------------------------------
# transformer (utils/transformer.py)
# ------------------------------------------------------------------------------------------------------------
def attention_core(q, k, v, mask):
    """utils/transformer.py:98-120 on [B,h,S,d] tensors; mask [B,S,S] in {0,1} or None. Returns (probs, probs @ v)."""
    d = q.shape[-1]
    scores = (q @ k.transpose(-1, -2)) * (1.0 / math.sqrt(float(d)))  # :98-100
    if mask is not None:
        m = mask[:, None]
        scores = scores * m - 1e10 * (1 - m)  # :109-110 (masked entries become exactly -1e10)
    probs = torch.softmax(scores, dim=-1)  # :112
    return probs, probs @ v  # :120


def attention_layer(x_flat, mask, batch, seq, heads, p: Params, scope: str):
    """utils/transformer.py:33-138 (no cache, attention dropout 0).  mask [B,S,S] in {0,1}.
    Returns (projected context [B*S,H], probs [B,h,S,S])."""
    H = x_flat.shape[-1]
    d = H // heads

    def proj(name):  # :8-30
        y = dense(x_flat, p, f"{scope}/{name}")
        return y.reshape(batch, seq, heads, d).permute(0, 2, 1, 3)

    q, k, v = proj("query_layer"), proj("key_layer"), proj("value_layer")
    probs, ctx4 = attention_core(q, k, v, mask)
    ctx = ctx4.permute(0, 2, 1, 3).reshape(batch * seq, H)  # :123-127
    out = dense(ctx, p, f"{scope}/context_projection_layer")  # :130-135
    return out, probs


def mlp_block(x, p: Params, scope: str):
    """utils/transformer.py:141-163."""
    return dense(dense(x, p, f"{scope}/intermediate", gelu), p, f"{scope}/output")


def _scoped(dropout, name):
    """The dropout hook of one stack: the stack's keys (layer, kind) become (name, layer, kind)."""
    if dropout is None:
        return None
    return lambda key, x: dropout((name,) + tuple(key), x)


def transformer(hidden, mask, p: Params, scope: str, num_layers: int, heads: int, return_attn_probs=False, dropout=None):
    """utils/transformer.py:171-247, pre-LN.  hidden [B,S,H]; mask [B,S,S].
    self_attn_probs (if requested) is the head-MEAN, stacked over layers: [B, layers, S, S] (:208-209,238).
    dropout: None (dropout 0) or a callable dropout(key, x [B*S, H]) applied to the projected context, bias included
    (:136, key (layer, "attn")) and to the FFN output (:162, key (layer, "ffn")), each before its residual add."""
    B, S, H = hidden.shape
    h = hidden.reshape(B * S, H)
    probs_all = []
    for l in range(num_layers):
        ls = f"{scope}/layer{l:02d}"
        a, probs = attention_layer(layer_norm(h, p, f"{ls}/LayerNorm_attn_ln0"), mask, B, S, heads, p, ls)
        if return_attn_probs:
            probs_all.append(probs.mean(1))
        if dropout is not None:
            a = dropout((l, "attn"), a)
        h = h + a
        f = mlp_block(layer_norm(h, p, f"{ls}/LayerNorm_mlp_ln0"), p, ls)
        if dropout is not None:
            f = dropout((l, "ffn"), f)
        h = h + f
    h = layer_norm(h, p, f"{scope}/LayerNorm_ln_final")
    out = {"_hidden_state_flat": h, "hidden_state": h.reshape(B, S, H)}
    if return_attn_probs:
        out["self_attn_probs"] = torch.stack(probs_all, 1)
    return out


# ------------------------------------------------------------------------------------------------------------
# Hybrid ResNet-lite stem (utils/vision_transformer.py:8-170) -- SURVEY.md 8(f) next-row 1 / Appendix D.
# The checker of the CUDA stem (K13, merlot_b200/csrc/stem.cu), forward and backward (DESIGN.md section 5).
# ------------------------------------------------------------------------------------------------------------
def _ident(t: torch.Tensor) -> torch.Tensor:
    return t


def bf16_round(t: torch.Tensor) -> torch.Tensor:
    """Pass as `rnd=` to the stem functions to materialise every tensor the reference holds in bfloat16 (conv operands and
    outputs, the cast standardised kernel :62-63, GroupNorm outputs model_utils.py:219-220, pooled maps, residual sums) with
    bf16 rounding, i.e. the reference's own precision policy instead of the fp32 restatement."""
    return t.to(torch.bfloat16).to(t.dtype)


def group_norm(x: torch.Tensor, p: Params, scope: str, num_groups: int = 32, eps: float = 1e-4, rnd=_ident) -> torch.Tensor:
    """utils/model_utils.py:133-222 as called by batch_norm_relu (vision_transformer.py:22-27): NHWC, 32 groups, eps 1e-4,
    mean_close_to_zero=True => ONE-PASS moments (sufficient_statistics + normalize_moments, :196-201):
    mean = sum(x)/n, var = sum(x^2)/n - mean^2 over (h, w, channels-in-group) per (sample, group); gamma/beta per channel."""
    n, h, w, c = x.shape
    if c % num_groups != 0:
        raise ValueError(f"{c} channels is not commensurate with {num_groups} groups")  # :171-177
    xr = x.reshape(n, h, w, num_groups, c // num_groups)
    cnt = float(h * w * (c // num_groups))
    mean = xr.sum((1, 2, 4), keepdim=True) / cnt
    var = (xr * xr).sum((1, 2, 4), keepdim=True) / cnt - mean * mean
    y = ((xr - mean) * torch.rsqrt(var + eps)).reshape(n, h, w, c)
    return rnd(y * p[f"{scope}/gamma"] + p[f"{scope}/beta"])


def conv2d_fixed_padding(x: torch.Tensor, kernel: torch.Tensor, strides: int = 1, weight_standardization: bool = True,
                         rnd=_ident) -> torch.Tensor:
    """vision_transformer.py:30-66.  x NHWC, kernel HWIO, no bias.  strides > 1: explicit pad (k-1)//2 before / the rest after
    (fixed_padding :8-19) then VALID; strides == 1: SAME.  Weight standardisation (:56-60): per OUTPUT channel, moments over
    (kh, kw, cin), biased variance, eps 1e-5."""
    k = kernel.shape[0]
    if weight_standardization:
        mean = kernel.mean((0, 1, 2), keepdim=True)
        var = ((kernel - mean) ** 2).mean((0, 1, 2), keepdim=True)
        kernel = (kernel - mean) * torch.rsqrt(var + 1e-5)
    kernel = rnd(kernel)
    xn = x.permute(0, 3, 1, 2)
    if strides > 1:
        beg = (k - 1) // 2
        xn = F.pad(xn, (beg, k - 1 - beg, beg, k - 1 - beg))
        y = F.conv2d(xn, kernel.permute(3, 2, 0, 1), stride=strides)
    else:
        assert k % 2 == 1
        y = F.conv2d(xn, kernel.permute(3, 2, 0, 1), padding=k // 2)
    return rnd(y.permute(0, 2, 3, 1))


def avg_pool_same(x: torch.Tensor, s: int, rnd=_ident) -> torch.Tensor:
    """tf.nn.avg_pool2d(ksize=s, strides=s, padding='SAME') on NHWC: ceil(h/s) outputs, padding at the bottom/right only,
    padded cells excluded from the average."""
    return rnd(F.avg_pool2d(x.permute(0, 3, 1, 2), s, s, ceil_mode=True, count_include_pad=False).permute(0, 2, 3, 1))


class _ScopeNames:
    """tf.layers / variable_scope default-name uniquification inside ONE variable scope: conv2d, conv2d_1, ... and
    GroupNorm, GroupNorm_1, ... in creation order (SURVEY.md Appendix A)."""

    def __init__(self, scope: str):
        self.scope, self.nconv, self.ngn = scope, 0, 0

    def conv(self) -> str:
        n = "conv2d" if self.nconv == 0 else f"conv2d_{self.nconv}"
        self.nconv += 1
        return f"{self.scope}/{n}/kernel"

    def gn(self, name: Optional[str] = None) -> str:
        if name is not None:
            return f"{self.scope}/GroupNorm_{name}"
        n = "GroupNorm" if self.ngn == 0 else f"GroupNorm_{self.ngn}"
        self.ngn += 1
        return f"{self.scope}/{n}"


def bottleneck_block(x: torch.Tensor, p: Params, names: _ScopeNames, filters: int, strides: int, use_projection: bool,
                     rnd=_ident) -> torch.Tensor:
    """vision_transformer.py:69-96.  Striding is done by average pooling: the shortcut pools BEFORE its 1x1 (:79-83), the main
    path pools AFTER the 3x3 (:92-93).  Variable creation order: [shortcut conv, GN], 1x1, GN, 3x3, GN, 1x1, GN."""
    shortcut = x
    if use_projection:
        sc_in = avg_pool_same(x, strides, rnd) if strides > 1 else x
        shortcut = group_norm(conv2d_fixed_padding(sc_in, p[names.conv()], rnd=rnd), p, names.gn(), rnd=rnd)  # skip_relu=True
    y = torch.relu(group_norm(conv2d_fixed_padding(x, p[names.conv()], rnd=rnd), p, names.gn(), rnd=rnd))
    y = torch.relu(group_norm(conv2d_fixed_padding(y, p[names.conv()], rnd=rnd), p, names.gn(), rnd=rnd))
    if strides > 1:
        y = avg_pool_same(y, strides, rnd)
    y = group_norm(conv2d_fixed_padding(y, p[names.conv()], rnd=rnd), p, names.gn(), rnd=rnd)  # skip_relu=True
    return torch.relu(rnd(y + shortcut))


def lite_resnet50(x: torch.Tensor, p: Params, scope: str, layers, width: int = 64, rnd=_ident) -> torch.Tensor:
    """vision_transformer.py:118-170: 3-conv stem (3x3 s2, 3x3, 3x3; GN+ReLU each) -> avg-pool 2 -> len(layers) block groups
    with filters width*2^i, stride 1 for the first group and 2 after."""
    st = _ScopeNames(f"{scope}/stem")
    x = rnd(x)
    x0 = torch.relu(group_norm(conv2d_fixed_padding(x, p[st.conv()], strides=2, rnd=rnd), p, st.gn("stem0"), rnd=rnd))
    x1 = torch.relu(group_norm(conv2d_fixed_padding(x0, p[st.conv()], rnd=rnd), p, st.gn("stem1"), rnd=rnd))
    x2 = torch.relu(group_norm(conv2d_fixed_padding(x1, p[st.conv()], rnd=rnd), p, st.gn("stem2"), rnd=rnd))
    c = avg_pool_same(x2, 2, rnd)
    for i, blocks in enumerate(layers):
        names = _ScopeNames(f"{scope}/block_group{i + 1}")
        c = bottleneck_block(c, p, names, width * (2 ** i), 1 if i == 0 else 2, True, rnd)  # :109-110
        for _ in range(1, blocks):
            c = bottleneck_block(c, p, names, width * (2 ** i), 1, False, rnd)
    return c


def resnet_param_shapes(scope: str, layers, width: int = 64, hidden_size: int = 768) -> Dict[str, tuple]:
    """Variables of the hybrid stem in creation order (names per SURVEY.md Appendix A; unverifiable against a checkpoint here)."""
    s: Dict[str, tuple] = {}

    def gn(name, c):
        s[f"{name}/gamma"] = (c,)
        s[f"{name}/beta"] = (c,)

    st = _ScopeNames(f"{scope}/resnet50lite/stem")
    for (cin, cout), nm in zip(((3, width // 2), (width // 2, width // 2), (width // 2, width)), ("stem0", "stem1", "stem2")):
        s[st.conv()] = (3, 3, cin, cout)
        gn(st.gn(nm), cout)
    cin = width
    for i, blocks in enumerate(layers):
        f = width * (2 ** i)
        names = _ScopeNames(f"{scope}/resnet50lite/block_group{i + 1}")
        for b in range(blocks):
            if b == 0:
                s[names.conv()] = (1, 1, cin, 4 * f)
                gn(names.gn(), 4 * f)
            s[names.conv()] = (1, 1, cin, f)
            gn(names.gn(), f)
            s[names.conv()] = (3, 3, f, f)
            gn(names.gn(), f)
            s[names.conv()] = (1, 1, f, 4 * f)
            gn(names.gn(), 4 * f)
            cin = 4 * f
    s[f"{scope}/conv_postresnet_proj/kernel"] = (1, 1, cin, hidden_size)
    s[f"{scope}/conv_postresnet_proj/bias"] = (hidden_size,)
    return s


# ------------------------------------------------------------------------------------------------------------
# ViT backbone (utils/vision_transformer.py:173-274): patch-embed stem (resnet_layers == []) or the hybrid stem
# ------------------------------------------------------------------------------------------------------------
def vision_transformer_backbone(image: torch.Tensor, cfg: dict, p: Params, dropout=None):
    """dropout: None or the model's dropout hook; the ViT stack calls it with keys ("vit", layer, "attn" | "ffn").  The hook
    applies vit_hidden_dropout_prob there when the config sets it (:243-244)."""
    P = cfg["patch_size"]
    H = cfg["hidden_size"]
    num_cls = cfg.get("num_cls_emb", 2)
    resnet_layers = cfg.get("resnet_layers", [])
    n, h0, w0, c = image.shape
    assert h0 % P == 0 and w0 % P == 0  # :189-190
    scope = "vision_backbone/vision_transformer"
    x = image - 0.5  # :193
    h1, w1 = h0 // P, w0 // P
    if len(resnet_layers) == 0:
        # conv2d k=P, s=P, VALID == non-overlapping im2col GEMM; kernel HWIO [P,P,3,H] flattened (kh, kw, c)
        patches = x.reshape(n, h1, P, w1, P, c).permute(0, 1, 3, 2, 4, 5).reshape(n * h1 * w1, P * P * c)
        x = patches @ p[f"{scope}/conv2d/kernel"].reshape(P * P * c, H) + p[f"{scope}/conv2d/bias"]  # :196-205
    else:
        assert P == 16  # :208
        rc = lite_resnet50(x, p, f"{scope}/resnet50lite", resnet_layers, width=64)  # :209-210
        assert rc.shape[1] == h1 and rc.shape[2] == w1, "the stem reduces by 16 (2 * 2 * 2 * 2)"
        k = p[f"{scope}/conv_postresnet_proj/kernel"]  # 1x1 SAME with bias, not standardised (:213-223)
        x = rc.reshape(n * h1 * w1, k.shape[2]) @ k.reshape(k.shape[2], H) + p[f"{scope}/conv_postresnet_proj/bias"]
    x = x.reshape(n, h1 * w1, H)
    x = torch.cat([torch.zeros(n, num_cls, H, dtype=x.dtype), x], 1)  # :231
    x = layer_norm(x + position_embedder2d(p, f"{scope}/pos_embs", h1, w1, num_cls), p,
                   f"{scope}/LayerNorm_ctx_patches_pre_ln")  # :232-234
    S = h1 * w1 + num_cls
    mask = torch.ones(n, S, S, dtype=x.dtype)  # :239
    info = transformer(x, mask, p, scope, cfg.get("num_vision_transformer_hidden_layers", cfg["num_hidden_layers"]),
                       cfg["num_attention_heads"], dropout=_scoped(dropout, "vit"))
    info["cls"] = info["hidden_state"][:, :num_cls]
    seq = info["hidden_state"][:, num_cls:]
    sp = cfg["spatial_pool_size"]
    if sp > 1:  # :255-267, avg_pool2d VALID
        seq = seq.reshape(n, h1, w1, H)
        h2, w2 = h1 // sp, w1 // sp
        seq = seq[:, :h2 * sp, :w2 * sp].reshape(n, h2, sp, w2, sp, H).mean((2, 4)).reshape(n, h2 * w2, H)
    else:
        h2, w2 = h1, w1
    info["seq"] = seq
    info["num_h"], info["num_w"] = h2, w2
    return info


# ------------------------------------------------------------------------------------------------------------
# mask_inputs with injected random draws (model/modeling.py:381-489)
# ------------------------------------------------------------------------------------------------------------
def make_mask_draws(B: int, L: int, num_to_mask: int, vocab_size: int, seed: int,
                    spanbert_len_probs=(0.625, 0.25, 0.125)) -> Dict[str, torch.Tensor]:
    """The five random tensors the reference draws with tf.random.* inside mask_inputs, generated from a seed.
    `gumbel` is z = -log(-log(U)) itself (model_utils.py:647) so that no transcendental sits between draw and compare."""
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(B, L, generator=g).clamp_(1e-9, 1.0 - 1e-7)
    probs = torch.tensor(spanbert_len_probs)
    return {
        "gumbel": (-torch.log(-torch.log(u))).float(),
        "span_lower": torch.multinomial(probs, B * num_to_mask, True, generator=g).reshape(B, num_to_mask).int(),
        "span_upper": torch.multinomial(probs, B * num_to_mask, True, generator=g).reshape(B, num_to_mask).int(),
        "option": torch.multinomial(torch.tensor([0.1, 0.8, 0.1]), B * L, True, generator=g).int(),
        "rand_ids": torch.randint(100, vocab_size, (B * L,), generator=g).int(),
    }


def mask_inputs(input_ids_2d: torch.Tensor, attention_summs: Optional[torch.Tensor], cfg: dict,
                draws: Dict[str, torch.Tensor]):
    """model/modeling.py:381-489.  input_ids_2d [B,L] int; attention_summs [B,L] fp32 = sum over (layers, queries) of the
    head-mean language-only attention probabilities (:428-431).  Returns masked_ids [B,L] and sorted masked_idx [B,n]."""
    B, L = input_ids_2d.shape
    topk_perc = cfg.get("masking_use_topk_from_attn_perc", 0.20)
    choose_topk_prob = cfg.get("masking_choose_topk_prob", 0.5)
    masking_rate = cfg.get("masking_rate", 0.2)
    do_spanbert = cfg.get("masking_do_spanbert", True)
    use_attn = cfg.get("masking_use_attn", True)
    num_topk = int(L * topk_perc)
    num_to_mask = int(L * masking_rate)
    nontopk_val = 0.01
    topk_val = nontopk_val * choose_topk_prob * (1.0 - topk_perc) / (topk_perc * (1.0 - choose_topk_prob))  # :418-419

    sentinel = torch.arange(L)
    is_special = (input_ids_2d < 100).float()  # :423
    if use_attn:
        summ = attention_summs.float().reshape(B, L) * (1.0 - is_special)  # :428-433
        _, top_inds = top_k_tf(summ, num_topk)  # :435
        is_important = (top_inds[..., None] == sentinel[None, None]).any(1)  # :436
        mask_weight = is_important.float() * np.float32(topk_val - nontopk_val) + np.float32(nontopk_val)  # :437
    else:
        mask_weight = torch.ones(B, L)
    log_mask = torch.log(mask_weight) - np.float32(1e8) * is_special  # :442
    _, idx = top_k_tf(log_mask + draws["gumbel"], num_to_mask)  # model_utils.py:640-649
    idx = idx.flip(-1)  # [:, ::-1] :445
    if do_spanbert:
        start = idx - draws["span_lower"].long()  # :457
        end = idx + draws["span_upper"].long()  # :458
        does_match = (sentinel[None, None] >= start[..., None]) & (sentinel[None, None] <= end[..., None])  # :461-464
        m_idx = torch.arange(num_to_mask)[None, :, None].expand_as(does_match)
        first = torch.where(does_match, m_idx, torch.full_like(m_idx, num_to_mask)).min(1).values
        which_match = torch.where(first == num_to_mask, torch.zeros_like(first), first).float()  # argmax: first, 0 if none
        which_match = which_match * (1.0 - is_special)  # :466
        which_match = which_match + np.float32(0.5) * mask_weight / mask_weight.max()  # :468
        _, mask_idx = top_k_tf(which_match, num_to_mask)  # :469
    else:
        mask_idx = idx
    mask_idx = torch.sort(mask_idx, 1).values  # :473
    ids_flat = input_ids_2d.reshape(-1).long()
    all_options = torch.stack([ids_flat, torch.full_like(ids_flat, MASK), draws["rand_ids"].long()], 1)  # :474-478
    do_mask = (mask_idx[..., None] == sentinel[None, None]).any(1).reshape(-1)  # :482-483
    option = draws["option"].long() * do_mask.long()  # :484-485
    masked_ids = all_options.gather(1, option[:, None]).reshape(B, L)  # :486
    return {"masked_ids": masked_ids.int(), "masked_idx": mask_idx.int(), "mask_weight": mask_weight,
            "topk_val": topk_val}


# ------------------------------------------------------------------------------------------------------------
# MerlotModel (model/modeling.py:47-668)
# ------------------------------------------------------------------------------------------------------------
class MerlotOracle:
    """Functional mirror of MerlotModel.__init__ + loss heads, single replica, fp32 (or fp64) throughout.

    image: [batch*num_chunks, h, w, 3] float in [0,1]; input_ids: int [batch, num_chunks, Lc] or [batch, Lc].
    mask_draws: dict from make_mask_draws (required when mask_input=True) or
    mask_override: {'masked_ids','masked_idx'} to bypass mask selection (used to feed the GPU-chosen mask).
    dropout: None (dropout 0, the eval model) or a callable dropout(key, x [rows, H]) -> x, applied wherever the reference
    applies hidden dropout: keys ("vit" | "langonly" | "joint", layer, "attn" | "ffn") inside the three stacks and
    ("embed", "langonly" | "joint") after the two embedding LayerNorms (oracle/dropout_mask.py builds the training one).
    """

    def __init__(self, config: dict, params: Params, image, input_ids, mask_input=False, shuffled_idx_img=None,
                 mask_draws=None, mask_override=None, log_attention_probs=True, dropout=None):
        self.config = copy.deepcopy(config)
        self.p = params
        cfg = self.config
        if cfg.get("num_imgs", 1) != 1:
            raise NotImplementedError("oracle: num_imgs > 1 (modeling.py:111-122) not restated (no shipped config sets it)")
        self.num_texts = cfg.get("num_texts", 1)
        if input_ids.dim() == 2:  # :72-77
            self.num_chunks = 1
            self.num_chunks_in_group = 1
            self.batch_size, self.lang_chunk_length = input_ids.shape
            self.input_ids = input_ids[:, None]
        else:
            self.input_ids = input_ids
            self.batch_size, self.num_chunks, self.lang_chunk_length = input_ids.shape
            self.num_chunks_in_group = cfg.get("num_chunks_in_group", self.num_chunks)
            assert self.num_chunks % self.num_chunks_in_group == 0  # :82
        self.hidden_size = cfg["hidden_size"]
        self.vocab_size = cfg["vocab_size"]
        H = self.hidden_size
        dt = image.dtype

        # ---- vision backbone (:95-133) ----
        self.vision_transformer_info = vit = vision_transformer_backbone(image, cfg, params, dropout)
        self.img_trg_h = vit["cls"][:, 1]  # :99
        feats = torch.cat([vit["cls"][:, 0, None], vit["seq"]], 1)  # :101-104
        self.viz_chunk_length = vit["num_h"] * vit["num_w"] + 1
        if self.num_texts > 1:  # VCR: every image is paired with num_texts candidate texts (:111-119): features tiled per text
            assert shuffled_idx_img is None  # :319-320
            feats = feats.reshape(self.B // self.num_texts, 1, self.P, H).expand(-1, self.num_texts, -1, -1)
        feats = feats.reshape(self.B, self.P, H)  # :121
        feats = feats + self.vision_pos_emb(shuffled_idx_img)  # :125
        feats = layer_norm(feats, params, "vision_backbone/LayerNorm_final_ln")  # :126
        viz_valid = torch.ones(self.B, self.P, dtype=torch.bool)
        pieces = [{"name": "viz", "x": feats, "is_valid": viz_valid}]

        # ---- language side ----
        if mask_input:  # :135-139
            self.lang_trg_h, self.lang_transformer_info = self.langonly_reps(dropout)
            if mask_override is not None:
                self.lang_mask_info = {k: torch.as_tensor(v) for k, v in mask_override.items()}
            else:
                summ = self.lang_transformer_info["self_attn_probs"].sum((1, 2))  # :428
                self.attention_summs = summ.reshape(self.B, self.L)
                self.lang_mask_info = mask_inputs(self.input_ids.reshape(self.B, self.L), self.attention_summs, cfg,
                                                  mask_draws)
            ids_to_use = self.lang_mask_info["masked_ids"]
        else:
            ids_to_use = self.input_ids
        ids_to_use = ids_to_use.reshape(self.B, self.L)  # :143
        pieces.append({"name": "lang", "x": self.embed_words(ids_to_use, dropout=dropout), "is_valid": ids_to_use != 0})  # :145-149

        enc_in = torch.cat([x["x"] for x in pieces], 1)  # :151
        is_valid = torch.cat([x["is_valid"] for x in pieces], 1)  # :152
        attn_mask = is_valid[:, None] & is_valid[:, :, None]  # :158
        if cfg.get("disable_pairwise_lang_attn", False):  # :160-168: segment 0 = vision tokens, 1 + c = language chunk c
            segment_idx = torch.cat([torch.zeros(self.P, dtype=torch.int64),
                                     1 + torch.div(torch.arange(self.L), self.lang_chunk_length, rounding_mode="floor")])
            can_attend = segment_idx[:, None] == segment_idx[None]
            can_attend = can_attend | (segment_idx == 0)[None] | (segment_idx == 0)[:, None]
            attn_mask = attn_mask & can_attend[None]
        attn_mask = attn_mask.to(dt)  # :170
        self.encoder_info = transformer(enc_in, attn_mask, params, "encoder", cfg["num_hidden_layers"],
                                        cfg["num_attention_heads"], return_attn_probs=log_attention_probs,
                                        dropout=_scoped(dropout, "joint"))  # :171-174
        self.encoder_hidden_states = {}
        cur = 0
        for x in pieces:  # :176-184
            x["start"], x["end"] = cur, cur + x["x"].shape[1]
            cur = x["end"]
            self.encoder_hidden_states[x["name"]] = self.encoder_info["hidden_state"][:, x["start"]:x["end"]]
        self.encoder_pieces = pieces
        if log_attention_probs:  # :186-203
            sap = self.encoder_info["self_attn_probs"].mean(1)
            vf = is_valid.to(dt)
            sap = sap * (vf[:, None] * vf[:, :, None])
            sap = sap.mean(0)
            sap = sap / sap.sum()
            attns = {}
            for x_to in pieces:
                for x_from in pieces:
                    attns[f"{x_from['name']}2{x_to['name']}"] = sap[x_to["start"]:x_to["end"],
                                                                    x_from["start"]:x_from["end"]].sum()
            self.attention_log = {f"encoder/{k}": v for k, v in sorted(attns.items())}

    # shapes (:226-248)
    @property
    def B(self):
        return self.batch_size * (self.num_chunks // self.num_chunks_in_group)

    @property
    def L(self):
        return self.lang_chunk_length * self.num_chunks_in_group

    @property
    def P(self):
        return self.viz_chunk_length * self.num_chunks_in_group

    def embed_words(self, ids_2d, norm_scope_name="position_embeddings", dropout=None):
        """:262-297 -- E[ids] + Pos[0:L] -> LN embed_norm -> dropout (:294; key ("embed", "joint") for position_embeddings,
        ("embed", "langonly") for langonly_embeddings, on the [B*L, H] rows)."""
        p = self.p
        L = ids_2d.shape[1]
        assert L <= self.config["max_position_embeddings"]  # model_utils.py:282
        assert int(ids_2d.min()) >= 0 and int(ids_2d.max()) <= self.vocab_size - 1  # model_utils.py:256-257
        emb = p["word_embeddings/word_embeddings"][ids_2d.long()]
        pos = p[f"{norm_scope_name}/position_embeddings"][:L][None]
        y = layer_norm(emb + pos, p, f"{norm_scope_name}/LayerNorm_embed_norm")
        if dropout is not None:
            name = {"position_embeddings": "joint", "langonly_embeddings": "langonly"}[norm_scope_name]
            y = dropout(("embed", name), y.reshape(-1, y.shape[-1])).reshape(y.shape)
        return y

    def vision_pos_emb(self, shuffled_idx_img=None):
        """:299-337."""
        p = self.p
        n = self.num_chunks_in_group
        table = p["vision_backbone/img_idx_pe"]
        if shuffled_idx_img is None:
            my_pe = table[:n][:, None].expand(n, self.viz_chunk_length, -1).reshape(1, self.P, -1)  # :314-315
        else:
            my_pe = table[shuffled_idx_img.reshape(-1).long()]  # :321
            my_pe = my_pe[:, None].expand(-1, self.viz_chunk_length, -1).reshape(self.B, self.P, -1)  # :322-323
        pe2d = position_embedder2d(p, "vision_backbone/final_pe", self.vision_transformer_info["num_h"],
                                   self.vision_transformer_info["num_w"], 1)  # :327-335
        return my_pe + pe2d.repeat(n, 1)[None]  # :336

    def langonly_reps(self, dropout=None):
        """:339-379.  dropout: None or the model's dropout hook (keys ("embed", "langonly") and ("langonly", layer, kind))."""
        cfg = self.config
        if "langonly_num_chunks_in_group" in cfg:
            g = cfg["langonly_num_chunks_in_group"]
            ng = self.num_chunks // g
            assert ng > 0 and self.num_chunks % g == 0
            ids = self.input_ids.reshape(self.batch_size * ng, self.lang_chunk_length * g)
        else:
            ids = self.input_ids.reshape(self.batch_size, self.lang_chunk_length * self.num_chunks)
        emb = self.embed_words(ids, "langonly_embeddings", dropout)
        valid = ids != 0
        mask = (valid[:, None] & valid[:, :, None]).to(emb.dtype)
        info = transformer(emb, mask, self.p, "encoder", cfg["num_lang_transformer_hidden_layers"],
                           cfg["num_attention_heads"], return_attn_probs=True, dropout=_scoped(dropout, "langonly"))
        pool = info["_hidden_state_flat"].reshape(self.batch_size * self.num_chunks, self.lang_chunk_length, -1)[:, 0]
        return pool, info

    def lm_head(self, h):
        """:205-224."""
        p, cfg = self.p, self.config
        if cfg.get("do_projection", False):
            h = layer_norm(dense(h, p, "lm_head/projection", gelu), p, "lm_head/LayerNorm")
        logits = h @ p["word_embeddings/word_embeddings"].t()
        if cfg.get("do_bias", False):
            logits = logits + p["lm_head/output_bias"]
        return logits

    def mask_loss(self):
        """:528-551."""
        hs = self.encoder_hidden_states["lang"].reshape(self.B * self.L, -1)
        idx = (self.lang_mask_info["masked_idx"].long() + torch.arange(self.B)[:, None] * self.L).reshape(-1)  # :534
        pooled = hs[idx]
        targets = self.input_ids.reshape(-1)[idx].long()
        logits = self.lm_head(pooled)
        raw = raw_cross_entropy_with_logits(logits, targets)
        valid = (targets != 0).to(raw.dtype)
        denom = valid.sum() + 1e-5  # :543
        loss = (valid * raw).sum() / denom
        acc = (valid * (logits.argmax(-1) == targets).to(raw.dtype)).sum() / denom
        return loss, {"loss": loss, "acc": acc}

    def project_and_norm(self, x, name, add_intermediate):
        """:18-44 under scope 'contrastive'."""
        p = self.p
        if add_intermediate:
            x = layer_norm(dense(x, p, f"contrastive/{name}_intermediate", gelu), p, f"contrastive/LayerNorm_{name}_ln")
        return l2_normalize(dense(x, p, f"contrastive/{name}"))

    def contrastive_loss(self):
        """:491-526, single replica (tpu_cross_replica_stack returns (tensor[None], 0), model_utils.py:682-683)."""
        cfg = self.config
        inter = cfg.get("do_projection", False)
        lx = self.project_and_norm(self.lang_trg_h, "lang_proj", inter)
        vx = self.project_and_norm(self.img_trg_h, "viz_proj", inter)
        temp = cfg.get("contrast_temp", 0.05)
        labels = torch.arange(lx.shape[0])
        losses = {}
        for name, x, y in (("lang_to_viz", lx, vx), ("viz_to_lang", vx, lx)):
            losses[name] = raw_cross_entropy_with_logits(x @ y.t() / temp, labels).mean()
        losses["loss_all"] = cfg.get("contrast_coef", 1.0) * (losses["lang_to_viz"] + losses["viz_to_lang"]) / 2  # :525
        self.contrastive_feats = {"lang": lx, "viz": vx}
        return losses["loss_all"], losses

    def allpairs_temporal_logits(self, xa, xb, scope_name):
        """:553-596 -- row i*n+j pairs xa_i with xb_j."""
        p = self.p
        B, n, H = xa.shape
        xa_t = xa[:, :, None].expand(B, n, n, H).reshape(B, n * n, H)
        xb_t = xb[:, None].expand(B, n, n, H).reshape(B, n * n, H)
        hj = torch.cat([xa_t, xb_t], 2).reshape(B * n * n, 2 * H)
        h0 = layer_norm(dense(hj, p, f"{scope_name}/intermediate", gelu), p, f"{scope_name}/LayerNorm_ln0")
        return dense(h0, p, f"{scope_name}/logits")

    def allpairs_temporal_labels(self, video_src_ids):
        """:598-620."""
        n = self.num_chunks_in_group
        xa = torch.arange(n)[:, None].expand(n, n)
        xb = torch.arange(n)[None].expand(n, n)
        lab = (xa == xb).int() + 2 * (xa < xb).int() + 3 * (xa > xb).int()
        v = video_src_ids.reshape(self.B, n)
        same = v[:, None] == v[:, :, None]
        return torch.where(same, lab[None].expand(self.B, n, n), torch.zeros(1, dtype=torch.int32)).reshape(-1)

    def temporal_loss(self, shuffled_idx_img, video_src_ids):
        """:622-668."""
        cfg = self.config
        n, H = self.num_chunks_in_group, self.hidden_size
        h_lang = self.encoder_hidden_states["lang"].reshape(self.B, n, self.lang_chunk_length, H)[:, :, 0]
        h_viz = self.encoder_hidden_states["viz"].reshape(self.B, n, self.viz_chunk_length, H)[:, :, 0]
        is_easy = (shuffled_idx_img < 64).reshape(self.B, n)  # :635
        labels = self.allpairs_temporal_labels(video_src_ids).long()
        info = {}
        for name, xa, xb in (("lang_viz", h_lang, h_viz), ("viz_viz", h_viz, h_viz)):
            logits = self.allpairs_temporal_logits(xa, xb, f"{name}_temporal")
            easy = is_easy[:, :, None] & is_easy[:, None]
            w = ((~easy).to(logits.dtype) * 0.99 + 0.01).reshape(-1)  # :649-652
            raw = raw_cross_entropy_with_logits(logits, labels) * w
            info[f"{name}_loss"] = raw.mean()
            right = (logits.argmax(-1) == labels).to(logits.dtype)
            info[f"{name}_acc"] = (right * w).sum() / (w.sum() + 1e-5)
            info[f"{name}_logits"] = logits
        info["loss"] = info["lang_viz_loss"]
        if cfg.get("image_shuffle_prob", 0) > 0:  # :664-665
            info["loss"] = info["loss"] + info["viz_viz_loss"]
        return info["loss"] * cfg.get("temporal_coef", 1.0), info


def vcr_cls_head_val(model: "MerlotOracle", p: Params, mode: str = "answer") -> torch.Tensor:
    """downstream/vcr/modeling.py:57-77: first language token -> dense(H/2, gelu) -> dense(1) -> [img_batch, 4]."""
    first = model.encoder_hidden_states["lang"][:, 0, :]
    h = dense(first, p, f"{mode}_cls/classifier_mlp0", gelu)
    return dense(h, p, f"{mode}_cls/classifier_mlp1").reshape(-1, 4)


def contrastive_loss_replicas(models, rank: int):
    """contrastive_loss of replica `rank` when `models` holds EVERY data-parallel replica (model/modeling.py:491-526 with
    tpu_cross_replica_stack, utils/model_utils.py:673-707: every replica scatters its features into slot `replica_id` of a
    zero tensor and cross_replica_sum fills in the others, so `all_*` = the replicas' features stacked in replica order and
    the labels are shifted by rank * batch (:519)).  Built on one autograd graph, the gradient that flows into the OTHER
    replicas' features is the cross_replica_sum's gradient (a sum over replicas = the reduce-scatter of the CUDA path)."""
    me = models[rank]
    cfg = me.config
    inter = cfg.get("do_projection", False)
    feats = []
    for m in models:
        if not hasattr(m, "_ctr_feats"):
            m._ctr_feats = (m.project_and_norm(m.lang_trg_h, "lang_proj", inter), m.project_and_norm(m.img_trg_h, "viz_proj", inter))
        feats.append(m._ctr_feats)
    lx, vx = feats[rank]
    all_l = torch.cat([f[0] for f in feats], 0)
    all_v = torch.cat([f[1] for f in feats], 0)
    temp = cfg.get("contrast_temp", 0.05)
    n = lx.shape[0]
    labels = torch.arange(n) + rank * n
    losses = {}
    for name, x, y in (("lang_to_viz", lx, all_v), ("viz_to_lang", vx, all_l)):
        losses[name] = raw_cross_entropy_with_logits(x @ y.t() / temp, labels).mean()
    losses["loss_all"] = cfg.get("contrast_coef", 1.0) * (losses["lang_to_viz"] + losses["viz_to_lang"]) / 2
    return losses["loss_all"], losses


def pretrain_losses_replicas(models, shuffled_idx_imgs, video_src_ids_list):
    """Per-replica model_fn losses (model/modeling.py:700-713) of a data-parallel step, and their MEAN -- whose gradient is what
    CrossShardOptimizer applies (utils/optimization.py:241-245: gradients averaged over replicas)."""
    per = []
    for r, m in enumerate(models):
        lang_loss, _ = m.mask_loss()
        contr_loss, _ = contrastive_loss_replicas(models, r)
        if m.config.get("temporal_coef", 1.0) > 0.0:
            temp_loss, _ = m.temporal_loss(shuffled_idx_imgs[r], video_src_ids_list[r])
        else:
            temp_loss = 0.0
        per.append(lang_loss + contr_loss + temp_loss)
    return sum(per) / len(per), per


def pretrain_losses(model: MerlotOracle, shuffled_idx_img, video_src_ids):
    """model_fn loss sum, model/modeling.py:700-713."""
    lang_loss, lang = model.mask_loss()
    contr_loss, contr = model.contrastive_loss()
    if model.config.get("temporal_coef", 1.0) > 0.0:
        temp_loss, temp = model.temporal_loss(shuffled_idx_img, video_src_ids)
    else:
        temp_loss, temp = 0.0, {}
    return lang_loss + contr_loss + temp_loss, {"lang": lang, "contr": contr, "temporal": temp}


# ------------------------------------------------------------------------------------------------------------
# parameters: names/shapes of SURVEY Appendix A; initialisers of the reference
# ------------------------------------------------------------------------------------------------------------
def _trunc_normal(shape, std, g):
    t = torch.empty(shape)
    torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=g)
    return t


def param_shapes(cfg: dict) -> Dict[str, tuple]:
    """Every trainable variable the reference creates (patch-embed stem, or the hybrid stem when resnet_layers is set)."""
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    P = cfg["patch_size"]
    s: Dict[str, tuple] = {}

    def ln(scope):
        s[f"{scope}/gamma"] = (H,)
        s[f"{scope}/beta"] = (H,)

    def lin(scope, i, o):
        s[f"{scope}/kernel"] = (i, o)
        s[f"{scope}/bias"] = (o,)

    def stack(scope, n):
        for l in range(n):
            ls = f"{scope}/layer{l:02d}"
            ln(f"{ls}/LayerNorm_attn_ln0")
            for nm in ("query_layer", "key_layer", "value_layer", "context_projection_layer"):
                lin(f"{ls}/{nm}", H, H)
            ln(f"{ls}/LayerNorm_mlp_ln0")
            lin(f"{ls}/intermediate", H, I)
            lin(f"{ls}/output", I, H)
        ln(f"{scope}/LayerNorm_ln_final")

    vt = "vision_backbone/vision_transformer"
    if len(cfg.get("resnet_layers", [])) == 0:
        s[f"{vt}/conv2d/kernel"] = (P, P, 3, H)
        s[f"{vt}/conv2d/bias"] = (H,)
    else:
        s.update(resnet_param_shapes(vt, cfg["resnet_layers"], 64, H))
    s[f"{vt}/pos_embs/pos_embs"] = (1, 64, 64, H)
    s[f"{vt}/pos_embs/cls_emb"] = (1, cfg.get("num_cls_emb", 2), H)
    ln(f"{vt}/LayerNorm_ctx_patches_pre_ln")
    stack(vt, cfg.get("num_vision_transformer_hidden_layers", cfg["num_hidden_layers"]))
    s["vision_backbone/img_idx_pe"] = (cfg.get("max_vision_pos_embeddings", 1024), H)
    s["vision_backbone/final_pe/pos_embs"] = (1, 64, 64, H)
    s["vision_backbone/final_pe/cls_emb"] = (1, 1, H)
    ln("vision_backbone/LayerNorm_final_ln")
    s["word_embeddings/word_embeddings"] = (V, H)
    for sc in ("position_embeddings", "langonly_embeddings"):
        s[f"{sc}/position_embeddings"] = (cfg["max_position_embeddings"], H)
        ln(f"{sc}/LayerNorm_embed_norm")
    stack("encoder", max(cfg["num_hidden_layers"], cfg.get("num_lang_transformer_hidden_layers", 0)))
    if cfg.get("do_projection", False):
        lin("lm_head/projection", H, H)
        ln("lm_head/LayerNorm")
    if cfg.get("do_bias", False):
        s["lm_head/output_bias"] = (V,)
    C = cfg.get("contrastive_size", H)
    for t in ("lang", "viz"):
        if cfg.get("do_projection", False):
            lin(f"contrastive/{t}_proj_intermediate", H, C)
            s[f"contrastive/LayerNorm_{t}_proj_ln/gamma"] = (C,)
            s[f"contrastive/LayerNorm_{t}_proj_ln/beta"] = (C,)
        lin(f"contrastive/{t}_proj", C if cfg.get("do_projection", False) else H, C)
    for t in ("lang_viz", "viz_viz"):
        lin(f"{t}_temporal/intermediate", 2 * H, H)
        ln(f"{t}_temporal/LayerNorm_ln0")
        lin(f"{t}_temporal/logits", H, 4)
    return s


def init_params(cfg: dict, seed: int = 0, dtype=torch.float32, perturb: float = 0.0) -> Params:
    """Reference initialisers: truncated normal(0.02) for dense kernels / embeddings / position tables,
    variance_scaling (fan_in, truncated normal) for the patch conv (vision_transformer.py:204), LN gamma=1 beta=0,
    biases 0.  `perturb` > 0 adds N(0, perturb) to biases/betas/gammas so parity tests exercise them."""
    g = torch.Generator().manual_seed(seed)
    std = cfg.get("initializer_range", 0.02)
    out: Params = {}
    for name, shape in param_shapes(cfg).items():
        leaf = name.rsplit("/", 1)[-1]
        if leaf == "gamma":
            t = torch.ones(shape)
        elif leaf in ("beta", "bias", "output_bias"):
            t = torch.zeros(shape)
        elif re.search(r"/(conv2d(_\d+)?|conv_postresnet_proj)/kernel$", name):  # tf.variance_scaling_initializer() everywhere
            fan_in = shape[0] * shape[1] * shape[2]
            s_ = math.sqrt(1.0 / fan_in) / 0.87962566103423978
            t = _trunc_normal(shape, s_, g)
        else:
            t = _trunc_normal(shape, std, g)
        if perturb > 0 and leaf in ("gamma", "beta", "bias", "output_bias"):
            t = t + torch.randn(shape, generator=g) * perturb
        out[name] = t.to(dtype)
    return out


# ------------------------------------------------------------------------------------------------------------
# optimizer (utils/optimization.py)
# ------------------------------------------------------------------------------------------------------------
MISSING_PRECISION = np.float32(1.00390625)  # optimization.py:267


def lr_scale(step: int, num_train_steps: int, num_warmup_steps: int) -> np.float32:
    """optimization.py:85-115: warmup step/W while step<W, else base*(1 - min(step,T)/T), base = T/(T-W+1)."""
    T, W = np.float32(num_train_steps), np.float32(num_warmup_steps)
    base = np.float32(float(num_train_steps) / (float(num_train_steps) - float(num_warmup_steps) + 1.0)) \
        if num_warmup_steps else np.float32(1.0)
    if num_warmup_steps and step < num_warmup_steps:
        return np.float32(np.float32(step) / W)
    gs = np.float32(min(step, num_train_steps))
    return np.float32(base * (np.float32(1.0) - gs / T))  # polynomial_decay(power=1, end=0)


def decode_v(stored_v: torch.Tensor) -> torch.Tensor:
    """optimization.py:268-281: |v| if sign>0 else |v|*1.00390625 (sign==0 is multiplied too)."""
    v_abs = stored_v.abs().float()
    return torch.where(torch.sign(stored_v.float()) > 0, v_abs, v_abs * float(MISSING_PRECISION))


def encode_v(v: torch.Tensor) -> torch.Tensor:
    """optimization.py:283-288."""
    enc = v.to(torch.bfloat16)
    enc_f = enc.float()
    err0 = (enc_f - v).abs()
    err1 = (enc_f * float(MISSING_PRECISION) - v).abs()
    return torch.where(err0 <= err1, enc, -enc)


def weight_decay_for(name: str, optimizer_cfg: dict) -> float:
    """optimization.py:125-147: regex param_overrides (re.search on the variable name)."""
    import re
    wd = optimizer_cfg.get("weight_decay_rate", 1e-4)
    for regexes, over in optimizer_cfg.get("param_overrides", None) or []:
        for k in over:
            if k not in ("learning_rate", "weight_decay_rate", "beta_1", "beta_2", "epsilon", "do_factor"):
                raise ValueError(f"Regex rule {regexes} -> {over} isn't OK because {k} isn't a changable optimization parameter")
        if "weight_decay_rate" in over and any(re.search(r, name) is not None for r in regexes):
            wd = over["weight_decay_rate"]
    return wd


class AdamOracle:
    """optimization.py:290-416 with use_bfloat16_adam moment storage, per tensor, fp32 math."""

    def __init__(self, params: Params, optimizer_cfg: dict):
        self.cfg = optimizer_cfg
        self.use_bf16 = optimizer_cfg.get("use_bfloat16_adam", False)
        dt = torch.bfloat16 if self.use_bf16 else torch.float32
        self.m = {k: torch.zeros_like(v, dtype=dt) for k, v in params.items()}
        self.v = {k: torch.zeros_like(v, dtype=dt) for k, v in params.items()}
        self.global_step = 0

    @classmethod
    def from_state(cls, params: Params, optimizer_cfg: dict, m: Params, v: Params, global_step: int):
        """The optimizer of a run that has taken `global_step` steps: moments `m` and `v` per parameter, stored as
        use_bfloat16_adam stores them (bf16 m and sign-packed bf16 v, or fp32).  The tensors are copied."""
        opt = cls(params, optimizer_cfg)
        for name, p in params.items():
            for slot, src in ((opt.m, m), (opt.v, v)):
                t = src[name]
                if t.dtype != slot[name].dtype or tuple(t.shape) != tuple(p.shape):
                    raise ValueError(f"{name}: moment {t.dtype} {tuple(t.shape)}, expected {slot[name].dtype} {tuple(p.shape)}")
                slot[name] = t.detach().cpu().clone().contiguous()
        opt.global_step = int(global_step)
        return opt

    def step_scalars(self):
        c = self.cfg
        beta1, beta2 = np.float32(0.9), np.float32(c.get("beta_2", 0.98))
        scale = lr_scale(self.global_step, c["num_train_steps"], c["num_warmup_steps"])
        t = np.float32(self.global_step) + np.float32(1.0)  # :355
        bc1 = np.float32(1.0) - np.power(beta1, t, dtype=np.float32)
        bc2 = np.float32(1.0) - np.power(beta2, t, dtype=np.float32)
        lr = np.float32(np.float32(c["learning_rate"]) * scale)
        lr_t = np.float32(lr * np.sqrt(bc2, dtype=np.float32) / bc1)  # :358
        return dict(beta1=beta1, beta2=beta2, lr_t=lr_t, eps=np.float32(c.get("epsilon", 1e-6)), lr=lr)

    @torch.no_grad()
    def apply_gradients(self, params: Params, grads: Params):
        s = self.step_scalars()
        b1, b2, lr_t, eps = float(s["beta1"]), float(s["beta2"]), float(s["lr_t"]), float(s["eps"])
        for name, p in params.items():
            g = grads.get(name)
            if g is None:  # :343-344
                continue
            g = g.float()
            wd = weight_decay_for(name, self.cfg)
            g2 = g * g + 1e-30  # :360
            m = self.m[name].float()
            v = decode_v(self.v[name]) if self.use_bf16 else self.v[name]
            next_m = b1 * m + (1.0 - b1) * g  # :389
            next_v = b2 * v + (1.0 - b2) * g2  # :390
            update = next_m / (torch.sqrt(next_v) + eps)  # :392
            if wd > 0:
                update = update + wd * p  # :401-402
            p.copy_(p - lr_t * update)  # :404-406
            if self.use_bf16:
                self.m[name] = next_m.to(torch.bfloat16)
                self.v[name] = encode_v(next_v)
            else:
                self.m[name], self.v[name] = next_m, next_v
        self.global_step += 1  # :251-253
