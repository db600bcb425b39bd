"""ORACLE -- TEST INFRASTRUCTURE ONLY.  The counter-based hidden dropout of the CUDA path, restated in NumPy from its definition,
and the hook that applies it where the reference calls dropout (utils/model_utils.py:335-349).

The reference draws its masks with tf.nn.dropout, which no restatement can reproduce.  The CUDA kernels instead derive every
mask bit from (seed, site, element index) so that the forward and the backward regenerate the same bits.  That definition
(merlot_b200/csrc/ptx.cuh `dropout_keep8`, and `thresh16` in rowwise.cu / gemm.cu) is restated here, so that tests can hand
the oracle the very mask a training step used and compare the step with it.

  * RNG: Philox4x32 with 7 rounds (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11).
    counter = (idx8 & 0xffffffff, idx8 >> 32, site, 0x4d45524c), key = (seed & 0xffffffff, seed >> 32).
  * Element index of [rows, N] element (row, col): lin = row * N + col, idx8 = lin >> 3.  Output word i of the call at idx8
    decides elements 8*idx8 + 2i (its low 16 bits) and 8*idx8 + 2i + 1 (its high 16 bits): keep <=> lane16 >= thresh16.
  * thresh16 = uint32(float32(p) * 65536 + 0.5) and scale = 1 / (1 - p), both in float32.

Only tests/ may import this module.
"""
from __future__ import annotations

import functools

import numpy as np
import torch

PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57  # round multipliers
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85  # key schedule (Weyl) increments
COUNTER_TAG = 0x4D45524C  # fourth counter word ("MERL")
DROPOUT_ROUNDS = 7
_U32 = np.uint64(0xFFFFFFFF)


def philox4x32(ctr, key, rounds: int):
    """Philox4x32-`rounds` on uint64 arrays holding 32-bit words (broadcast against each other).  ctr: 4 words, key: 2 words.
    Each round: (c0, c1, c2, c3) <- (hi(M1*c2) ^ c1 ^ k0, lo(M1*c2), hi(M0*c0) ^ c3 ^ k1, lo(M0*c0)); then k += (W0, W1)."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _U32 for c in ctr)
    k0, k1 = (np.asarray(k, dtype=np.uint64) & _U32 for k in key)
    for _ in range(rounds):
        p0 = c0 * np.uint64(PHILOX_M0)  # 32 x 32 -> 64 bits: exact in uint64
        p1 = c2 * np.uint64(PHILOX_M1)
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _U32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _U32
        k0 = (k0 + np.uint64(PHILOX_W0)) & _U32
        k1 = (k1 + np.uint64(PHILOX_W1)) & _U32
    return c0, c1, c2, c3


def thresh16(p: float) -> int:
    """Drop threshold on a 16-bit lane, computed in float32 as the host code does."""
    return int(np.uint32(np.float32(p) * np.float32(65536.0) + np.float32(0.5)))


def dropout_scale(p: float) -> np.float32:
    """Inverted-dropout scale of the kept elements (tf.nn.dropout), in float32."""
    return np.float32(1.0) / (np.float32(1.0) - np.float32(p))


def counter_dropout_keep(seed: int, site: int, rows: int, N: int, p: float) -> np.ndarray:
    """bool [rows, N]: the keep mask of a [rows, N] tensor with row-major element index lin = row * N + col."""
    if N % 8 != 0:
        raise ValueError(f"the mask is drawn 8 elements at a time: N = {N} is not a multiple of 8")
    seed = int(seed)
    idx8 = np.arange(rows * N // 8, dtype=np.uint64)
    words = philox4x32((idx8 & _U32, idx8 >> np.uint64(32), site, COUNTER_TAG), (seed & 0xFFFFFFFF, seed >> 32),
                       DROPOUT_ROUNDS)
    lanes = np.empty((idx8.size, 8), dtype=np.uint64)
    for i, w in enumerate(words):
        lanes[:, 2 * i] = w & np.uint64(0xFFFF)
        lanes[:, 2 * i + 1] = w >> np.uint64(16)
    return (lanes >= np.uint64(thresh16(p))).reshape(rows, N)


# ------------------------------------------------------------------------------------------------------------
# the oracle's dropout hook
# ------------------------------------------------------------------------------------------------------------
def kernel_site(key) -> int:
    """The `site` under which the CUDA path draws the mask of the dropout the oracle names `key`:
    ("embed", "langonly" | "joint") -> the embedding LayerNorm sites of merlot_b200/modeling.py;
    (stack, layer, "attn" | "ffn") -> the stack's base site + 2 * layer for the attention output projection and
    + 2 * layer + 1 for the FFN output (merlot_stack_forward in merlot_b200/csrc/stack.cu)."""
    from merlot_b200 import modeling as M
    if key[0] == "embed":
        return {"langonly": M._SITE_EMB_LO, "joint": M._SITE_EMB_J}[key[1]]
    stack, layer, kind = key
    base = {"vit": M._SITE_VIT, "langonly": M._SITE_LANGONLY, "joint": M._SITE_JOINT}[stack]
    return base + 2 * int(layer) + {"attn": 0, "ffn": 1}[kind]


@functools.lru_cache(maxsize=64)
def _keep_tensor(seed: int, site: int, rows: int, N: int, p: float) -> torch.Tensor:
    return torch.from_numpy(counter_dropout_keep(seed, site, rows, N, p))


def dropout_hook(seed: int, p: float, p_vit: float = None):
    """The oracle's `dropout(key, x_flat)` callable for a training step run with `dropout_seed=seed`: hidden_dropout_prob `p`
    everywhere and vit_hidden_dropout_prob `p_vit` (default: p, utils/vision_transformer.py:243-244) in the ViT.
    x_flat is [rows, H] in the model's logical row order; the result is x * keep * scale, differentiable in x."""
    p_vit = p if p_vit is None else p_vit

    def hook(key, x):
        prob = p_vit if key[0] == "vit" else p
        if prob == 0.0:
            return x
        rows, N = x.shape
        keep = _keep_tensor(int(seed), kernel_site(key), rows, N, float(prob))
        return x * (keep.to(x.dtype) * float(dropout_scale(prob)))

    return hook
