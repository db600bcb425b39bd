"""ctypes binding of include/merlot_b200.h (the C-ABI drop-in boundary).

The library is the product path: if it cannot be loaded this module raises -- there is no CPU or PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libmerlot_b200.so"

MERLOT_OK = 0
MERLOT_EINVAL = -1
MERLOT_ESHAPE = -2
MERLOT_ECUDA = -3
MERLOT_ENOTIMPL = -4

GEMM_OUT_F32 = 1
GEMM_ATOMIC = 2
GEMM_GELU = 4
GEMM_MUL_DGELU = 8
GEMM_DROPOUT = 16
GEMM_GELU_GRAD_OUT = 32
GEMM_MUL_AUX = 64


class MerlotError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"merlot_b200 error {code}: {msg}")
        self.code = code


class MerlotShapeError(MerlotError, ValueError):
    """Mirrors the ValueError / assert the reference raises at graph-build time (utils/model_utils.py:29-56)."""


class GemmDesc(C.Structure):
    _fields_ = [
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("a", C.c_void_p), ("lda", C.c_int), ("a_mn_major", C.c_int),
        ("b", C.c_void_p), ("ldb", C.c_int), ("b_mn_major", C.c_int),
        ("out", C.c_void_p), ("ld_out", C.c_int),
        ("out2", C.c_void_p), ("ld_out2", C.c_int),
        ("bias", C.c_void_p),
        ("resid", C.c_void_p), ("ld_resid", C.c_int),
        ("aux", C.c_void_p), ("ld_aux", C.c_int),
        ("alpha", C.c_float),
        ("flags", C.c_uint32),
        ("dropout_p", C.c_float), ("dropout_seed", C.c_uint64), ("dropout_site", C.c_uint32),
        ("splits", C.c_int),
        ("block_n", C.c_int),
    ]


_lib = None


def lib() -> C.CDLL:
    """Load libmerlot_b200.so (built in-tree by merlot_b200.build). Raises if missing -- no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} not found: run `python -m merlot_b200.build` (or __graft_entry__.build()). "
            "merlot_b200 has no CPU/PyTorch fallback path.")
    l = C.CDLL(str(LIB_PATH), mode=os.RTLD_GLOBAL if hasattr(os, "RTLD_GLOBAL") else 0)
    l.merlot_last_error.restype = C.c_char_p
    l.merlot_abi_version.restype = C.c_int
    l.merlot_launch_count.restype = C.c_longlong
    l.merlot_reset_launch_count.restype = None
    for fn in ("merlot_stack_activation_bytes", "merlot_stack_scratch_bytes", "merlot_layernorm_bwd_workspace_bytes",
               "merlot_attention_bwd_workspace_bytes"):
        getattr(l, fn).restype = C.c_size_t
    _lib = l
    return l


def check(rc: int) -> None:
    if rc == MERLOT_OK:
        return
    msg = lib().merlot_last_error().decode("utf-8", "replace")
    if rc == MERLOT_ESHAPE:
        raise MerlotShapeError(rc, msg)
    if rc == MERLOT_ENOTIMPL:
        raise NotImplementedError(msg)
    raise MerlotError(rc, msg)


def exported_symbols_from_header() -> list[str]:
    """Every function name declared in include/merlot_b200.h (used by the CPU test that checks the .so exports them)."""
    import re
    hdr = (_HERE.parent / "include" / "merlot_b200.h").read_text()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(merlot_[a-z0-9_]+)\s*\(", hdr)))


class AttnDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("S", C.c_int), ("heads", C.c_int), ("head_dim", C.c_int),
        ("qkv", C.c_void_p), ("ld_qkv", C.c_int),
        ("valid", C.c_void_p),
        ("scale", C.c_float),
        ("ctx", C.c_void_p), ("ld_ctx", C.c_int),
        ("lse", C.c_void_p),
        ("d_ctx", C.c_void_p),
        ("dsum", C.c_void_p),
        ("dq_accum", C.c_void_p), ("ld_dq", C.c_int),
        ("dqkv", C.c_void_p), ("ld_dqkv", C.c_int),
        ("colsum", C.c_void_p),
        ("d_bias_qkv", C.c_void_p),
        ("colsum2", C.c_void_p), ("colsum_split", C.c_int), ("colsum_valid_q", C.c_int),
        ("pair_viz_len", C.c_int), ("pair_chunk_len", C.c_int),
        ("dropout_p", C.c_float), ("dropout_seed", C.c_uint64), ("dropout_site", C.c_uint32),
    ]


class LnDesc(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("x_f32", C.c_int), ("ld_x", C.c_int),
        ("y", C.c_void_p), ("y_f32", C.c_int), ("ld_y", C.c_int),
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("mean", C.c_void_p), ("rstd", C.c_void_p),
        ("rows", C.c_longlong), ("H", C.c_int), ("eps", C.c_float),
        ("map_per", C.c_int), ("map_stride", C.c_int), ("map_off", C.c_int),
        ("dropout_p", C.c_float), ("dropout_seed", C.c_uint64), ("dropout_site", C.c_uint32),
    ]


class LnBwdDesc(C.Structure):
    _fields_ = [
        ("dy", C.c_void_p), ("dy_f32", C.c_int), ("ld_dy", C.c_int),
        ("x", C.c_void_p), ("x_f32", C.c_int), ("ld_x", C.c_int),
        ("mean", C.c_void_p), ("rstd", C.c_void_p), ("gamma", C.c_void_p),
        ("dres", C.c_void_p), ("ld_dres", C.c_int),
        ("dx", C.c_void_p), ("dx_f32", C.c_int), ("ld_dx", C.c_int),
        ("dgamma", C.c_void_p), ("dbeta", C.c_void_p),
        ("workspace", C.c_void_p),
        ("rows", C.c_longlong), ("H", C.c_int),
        ("map_per", C.c_int), ("map_stride", C.c_int), ("map_off", C.c_int),
        ("dropout_p", C.c_float), ("dropout_seed", C.c_uint64), ("dropout_site", C.c_uint32),
    ]


class LayerParams(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "ln1_gamma", "ln1_beta", "w_qkv", "b_qkv", "w_o", "b_o", "ln2_gamma", "ln2_beta", "w_1", "b_1", "w_2", "b_2",
        "g_ln1_gamma", "g_ln1_beta", "g_w_qkv", "g_b_qkv", "g_w_o", "g_b_o", "g_ln2_gamma", "g_ln2_beta", "g_w_1", "g_b_1",
        "g_w_2", "g_b_2")]


class StackDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("S", C.c_int), ("H", C.c_int), ("I", C.c_int), ("heads", C.c_int), ("layers", C.c_int),
        ("layer_params", C.POINTER(LayerParams)),
        ("final_gamma", C.c_void_p), ("final_beta", C.c_void_p),
        ("d_final_gamma", C.c_void_p), ("d_final_beta", C.c_void_p),
        ("valid", C.c_void_p),
        ("h_in", C.c_void_p),
        ("y", C.c_void_p),
        ("act_arena", C.c_void_p),
        ("save_for_backward", C.c_int),
        ("hidden_dropout_p", C.c_float), ("attention_dropout_p", C.c_float), ("dropout_seed", C.c_uint64),
        ("dropout_site_base", C.c_uint32),
        ("attn_colsum", C.c_void_p),
        ("attn_colsum2", C.c_void_p), ("attn_colsum_split", C.c_int), ("attn_colsum_valid_q", C.c_int),
        ("attn_probs", C.c_void_p),
        ("dy", C.c_void_p),
        ("dh_in", C.c_void_p),
        ("scratch", C.c_void_p),
        ("bwd_lo", C.c_int), ("bwd_hi", C.c_int),
        ("pair_viz_len", C.c_int), ("pair_chunk_len", C.c_int),
    ]


class MaskDesc(C.Structure):
    _fields_ = [
        ("ids", C.c_void_p), ("attn_summ", C.c_void_p), ("gumbel", C.c_void_p), ("span_lower", C.c_void_p),
        ("span_upper", C.c_void_p), ("option", C.c_void_p), ("rand_ids", C.c_void_p),
        ("masked_ids", C.c_void_p), ("masked_idx", C.c_void_p), ("valid_out", C.c_void_p),
        ("B", C.c_int), ("L", C.c_int), ("num_topk", C.c_int), ("num_to_mask", C.c_int), ("do_spanbert", C.c_int),
        ("mask_token", C.c_int),
        ("w_delta", C.c_float), ("w_non", C.c_float), ("logw_top", C.c_float), ("logw_non", C.c_float), ("w_max", C.c_float),
    ]


class WsItem(C.Structure):
    _fields_ = [("w", C.c_void_p), ("out", C.c_void_p), ("dws", C.c_void_p), ("dw", C.c_void_p),
                ("rows", C.c_int), ("rows_pad", C.c_int), ("cout", C.c_int), ("ld_dws", C.c_int), ("block0", C.c_int),
                ("reserved", C.c_int)]


class AdamDesc(C.Structure):
    _fields_ = [
        ("p", C.c_void_p), ("g", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p), ("p_bf16", C.c_void_p),
        ("n", C.c_longlong),
        ("beta1", C.c_float), ("one_minus_beta1", C.c_float), ("beta2", C.c_float), ("one_minus_beta2", C.c_float),
        ("epsilon", C.c_float), ("lr_t", C.c_float), ("weight_decay", C.c_float), ("grad_scale", C.c_float),
        ("zero_grad", C.c_int),
    ]
