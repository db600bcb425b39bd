"""TEST INFRASTRUCTURE ONLY.  Attention-probability dropout (attention_probs_dropout_prob, utils/transformer.py:114-115) for
the oracle: the mask of the CUDA kernels restated in NumPy from its definition, the hook that applies it, and the wrapper
that lets oracle/merlot_oracle.py's transformer drop its softmax probabilities.

The fused attention kernels (merlot_b200/csrc/ptx.cuh `attn_dropout_words`) never write the probabilities [B, heads, S, S]
to memory, so each of them regenerates the mask for the elements it holds.  The mask is a function of (seed, site, b, h,
q, k) alone, laid out so that each Philox call serves the 2 x 2 block {q, q+8} x {k, k+8} (q % 16 < 8, k % 16 < 8) that one
thread owns of a wgmma accumulator with either queries or keys on its rows:
  * n16 = ceil(S / 16); blk = ((((b * heads + h) * n16 + q // 16) * 8 + q % 8) * n16 + k // 16) * 8 + k % 8 (64 bits).
  * Philox4x32-7 (oracle/dropout_mask.py `philox4x32`) with counter = (blk & 0xffffffff, blk >> 32, site, 0x4154544e
    "ATTN") and key = (seed & 0xffffffff, seed >> 32).
  * word 2 * ((q >> 3) & 1) + ((k >> 3) & 1) decides (q, k): keep <=> (word >> 16) >= thresh16(p); kept probabilities are
    scaled by dropout_scale(p) -- the quantisation and scale of hidden dropout.
  * The fourth counter word keeps this stream disjoint from the hidden-dropout one ("MERL") at the same seed and site.
  * Layer l of a stack draws site base + l, base = the stack's hidden-dropout base site (merlot_b200/modeling.py _SITE_*).
"""
from __future__ import annotations

import functools

import numpy as np
import torch

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O

ATTN_COUNTER_TAG = 0x4154544E  # fourth counter word ("ATTN")
_U32 = np.uint64(0xFFFFFFFF)


def attention_keep(seed: int, site: int, B: int, heads: int, S: int, p: float) -> np.ndarray:
    """bool [B, heads, S, S]: the keep mask of attention-probability dropout at (seed, site), element [b, h, q, k]."""
    seed, n16 = int(seed), (S + 15) // 16
    th = np.uint64(DM.thresh16(p))
    r8 = np.arange(n16 * 8, dtype=np.uint64)
    blk16, off8 = r8 // np.uint64(8), r8 % np.uint64(8)  # q // 16 and q % 8 of a block's first query (or key)
    out = np.empty((B, heads, n16, 2, 8, n16, 2, 8), dtype=bool)  # [b, h, q // 16, (q >> 3) & 1, q % 8, k ...]
    for b in range(B):
        for h in range(heads):
            row = ((np.uint64(b * heads + h) * np.uint64(n16) + blk16) * np.uint64(8) + off8) * np.uint64(n16)
            blk = (row[:, None] + blk16[None, :]) * np.uint64(8) + off8[None, :]  # [query block row, key block row]
            words = DM.philox4x32((blk & _U32, blk >> np.uint64(32), site, ATTN_COUNTER_TAG), (seed & 0xFFFFFFFF, seed >> 32),
                                  DM.DROPOUT_ROUNDS)
            for qh in range(2):
                for kh in range(2):
                    keep = (words[2 * qh + kh] >> np.uint64(16)) >= th
                    out[b, h, :, qh, :, :, kh, :] = keep.reshape(n16, 8, n16, 8)
    return out.reshape(B, heads, n16 * 16, n16 * 16)[:, :, :S, :S]


def kernel_site(key) -> int:
    """(stack, layer, "probs") -> the site under which merlot_stack_forward / _backward draw that layer's mask."""
    from merlot_b200 import modeling as M
    stack, layer, kind = key
    assert kind == "probs", key
    return {"vit": M._SITE_VIT, "langonly": M._SITE_LANGONLY, "joint": M._SITE_JOINT}[stack] + int(layer)


@functools.lru_cache(maxsize=64)
def _keep_tensor(seed: int, site: int, B: int, heads: int, S: int, p: float) -> torch.Tensor:
    return torch.from_numpy(attention_keep(seed, site, B, heads, S, p))


def drop_probs(probs: torch.Tensor, seed: int, site: int, p: float) -> torch.Tensor:
    """probs [B, heads, S, S] * keep * 1/(1-p) under the mask of (seed, site), on probs' device; probs itself when p = 0."""
    if p == 0.0:
        return probs
    B, heads, S, _ = probs.shape
    keep = _keep_tensor(int(seed), int(site), B, heads, S, float(p)).to(probs.device)
    return probs * (keep.to(probs.dtype) * float(DM.dropout_scale(p)))


def dropout_hook(seed: int, p: float, p_vit: float = None, p_attn: float = 0.0):
    """oracle/dropout_mask.py's training hook for dropout_seed=seed (hidden_dropout_prob p, vit_hidden_dropout_prob p_vit),
    extended by attention_probs_dropout_prob p_attn in all three stacks (the ViT copies the model config,
    utils/vision_transformer.py:240) under keys (stack, layer, "probs") on x [B, heads, S, S]."""
    hidden = DM.dropout_hook(seed, p, p_vit)

    def hook(key, x):
        if key[-1] == "probs":
            return drop_probs(x, seed, kernel_site(key), p_attn)
        return hidden(key, x)
    return hook


_oracle_attention_core = O.attention_core
_oracle_transformer = O.transformer


def attention_core(q, k, v, mask, drop=None):
    """oracle attention_core (utils/transformer.py:98-120) with the probabilities passed through drop(probs) before
    probs @ v (:114-115).  Returns (dropped probs, dropped probs @ v)."""
    probs, ctx = _oracle_attention_core(q, k, v, mask)
    if drop is None:
        return probs, ctx
    probs = drop(probs)
    return probs, probs @ v


def transformer(hidden, mask, p, scope, num_layers, heads, return_attn_probs=False, dropout=None):
    """oracle transformer (utils/transformer.py:171-247) that also calls its dropout hook on each layer's probabilities, key
    (layer, "probs"), after the softmax and before probs @ v; self_attn_probs are built from what the hook returns (:138).
    Install it with `monkeypatch.setattr(merlot_oracle, "transformer", transformer)`; the hooks handed to the oracle then
    have to accept "probs" keys (dropout_hook above does)."""
    if dropout is None:
        return _oracle_transformer(hidden, mask, p, scope, num_layers, heads, return_attn_probs, dropout)
    layers = iter(range(num_layers))  # the oracle's transformer calls attention_core once per layer, bottom-up

    def core(q, k, v, m):
        return attention_core(q, k, v, m, lambda probs: dropout((next(layers), "probs"), probs))
    O.attention_core = core
    try:
        return _oracle_transformer(hidden, mask, p, scope, num_layers, heads, return_attn_probs, dropout)
    finally:
        O.attention_core = _oracle_attention_core
