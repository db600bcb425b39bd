"""Torch-tensor front end of the C-ABI operators (device memory + stream plumbing only; all math is in the .so)."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib as L


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _require_cuda(*ts: Optional[torch.Tensor]) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise L.MerlotError(L.MERLOT_EINVAL, "merlot_b200 operators take CUDA tensors only (no CPU fallback)")


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn_major: bool = False, b_mn_major: bool = False,
         out: Optional[torch.Tensor] = None, out_dtype: torch.dtype = torch.bfloat16,
         bias: Optional[torch.Tensor] = None, resid: Optional[torch.Tensor] = None,
         gelu: bool = False, out_pre: Optional[torch.Tensor] = None, dgelu_aux: Optional[torch.Tensor] = None,
         gelu_grad_out: bool = False, mul_aux: Optional[torch.Tensor] = None,
         alpha: float = 1.0, atomic: bool = False, dropout_p: float = 0.0, dropout_seed: int = 0,
         dropout_site: int = 0, splits: int = 0, block_n: int = 0, generic_epilogue: bool = False,
         M: Optional[int] = None, N: Optional[int] = None, K: Optional[int] = None) -> torch.Tensor:
    """C[M,N] = epilogue(alpha * A @ B^T) on wgmma tensor cores (see include/merlot_b200.h, K1).

    a: [M,K] (or [K,M] when a_mn_major); b: [N,K] (or [K,N] when b_mn_major); both bf16, row-major, 2-D.
    With gelu=True and out_pre given: out_pre <- pre-activation, return value <- gelu(pre).
    generic_epilogue=True forces the general epilogue path (to compare it with the fast one).
    """
    _require_cuda(a, b, out, bias, resid, out_pre, dgelu_aux, mul_aux)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.dim() == 2 and b.dim() == 2
    assert a.stride(1) == 1 and b.stride(1) == 1
    if M is None:
        M = a.shape[1] if a_mn_major else a.shape[0]
    if K is None:
        K = a.shape[0] if a_mn_major else a.shape[1]
    if N is None:
        N = b.shape[1] if b_mn_major else b.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=a.device)
    assert out.stride(1) == 1
    g = L.merlot_gemm_t()
    g.M, g.N, g.K = M, N, K
    g.a, g.lda, g.a_mn_major = a.data_ptr(), a.stride(0), int(a_mn_major)
    g.b, g.ldb, g.b_mn_major = b.data_ptr(), b.stride(0), int(b_mn_major)
    flags = 0
    if out.dtype == torch.float32:
        flags |= L.GEMM_OUT_F32
    else:
        assert out.dtype == torch.bfloat16
    if atomic:
        flags |= L.GEMM_ATOMIC
    if gelu:
        flags |= L.GEMM_GELU
    if gelu and out_pre is not None:
        # C-ABI convention: out <- pre, out2 <- gelu(pre)
        g.out, g.ld_out = out_pre.data_ptr(), out_pre.stride(0)
        g.out2, g.ld_out2 = out.data_ptr(), out.stride(0)
    else:
        g.out, g.ld_out = out.data_ptr(), out.stride(0)
        g.out2, g.ld_out2 = None, 0
    if dgelu_aux is not None:
        flags |= L.GEMM_MUL_DGELU
        g.aux, g.ld_aux = dgelu_aux.data_ptr(), dgelu_aux.stride(0)
    if gelu_grad_out:  # out_pre receives gelu'(pre) instead of pre
        assert gelu and out_pre is not None
        flags |= L.GEMM_GELU_GRAD_OUT
    if mul_aux is not None:  # v *= aux (the factor saved by gelu_grad_out)
        assert dgelu_aux is None
        flags |= L.GEMM_MUL_AUX
        g.aux, g.ld_aux = mul_aux.data_ptr(), mul_aux.stride(0)
    if bias is not None:
        assert bias.dtype == torch.float32
        g.bias = bias.data_ptr()
    if resid is not None:
        assert resid.dtype == torch.bfloat16
        g.resid, g.ld_resid = resid.data_ptr(), resid.stride(0)
    if dropout_p > 0.0:
        flags |= L.GEMM_DROPOUT
    if generic_epilogue:
        flags |= L.GEMM_GENERIC_EPILOGUE
    g.alpha = alpha
    g.flags = flags
    g.dropout_p, g.dropout_seed, g.dropout_site = dropout_p, dropout_seed, dropout_site
    g.splits, g.block_n = splits, block_n
    L.lib().merlot_gemm_bf16(C.byref(g), _stream())
    return out


def _attn_desc(qkv: torch.Tensor, B: int, S: int, heads: int, valid: Optional[torch.Tensor], pair=(0, 0),
               dropout=(0.0, 0, 0)) -> L.merlot_attn_t:
    _require_cuda(qkv, valid)
    assert qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.stride(1) == 1 and qkv.shape[0] == B * S
    a = L.merlot_attn_t()
    a.B, a.S, a.heads, a.head_dim = B, S, heads, qkv.shape[1] // (3 * heads)
    a.qkv, a.ld_qkv = qkv.data_ptr(), qkv.stride(0)
    if valid is not None:
        assert valid.dtype == torch.uint8 and valid.numel() == B * S and valid.is_contiguous()
        a.valid = valid.data_ptr()
    a.scale = 1.0 / (a.head_dim ** 0.5)
    a.pair_viz_len, a.pair_chunk_len = int(pair[0]), int(pair[1])  # disable_pairwise_lang_attn (0, 0 = off)
    # attention-probability dropout (p, seed, site); one layer's forward, backward, colsum and probs take the same triple
    a.dropout_p, a.dropout_seed, a.dropout_site = float(dropout[0]), int(dropout[1]), int(dropout[2])
    return a


def attention_fwd(qkv: torch.Tensor, B: int, S: int, heads: int, valid: Optional[torch.Tensor] = None,
                  ctx: Optional[torch.Tensor] = None, lse: Optional[torch.Tensor] = None, pair=(0, 0), dropout=(0.0, 0, 0)):
    """K2: ctx[B*S,H] = softmax(mask(q k^T / sqrt(d))) v, reading q/k/v in place from the fused qkv buffer.
    dropout=(p, seed, site): the probabilities are dropped with p before the product with v (lse stays undropped)."""
    a = _attn_desc(qkv, B, S, heads, valid, pair, dropout)
    H = heads * a.head_dim
    if ctx is None:
        ctx = torch.empty((B * S, H), dtype=torch.bfloat16, device=qkv.device)
    if lse is None:
        lse = torch.empty((B, heads, S), dtype=torch.float32, device=qkv.device)
    a.ctx, a.ld_ctx, a.lse = ctx.data_ptr(), ctx.stride(0), lse.data_ptr()
    L.lib().merlot_attention_fwd(C.byref(a), _stream())
    return ctx, lse


def attention_bwd_workspace(B: int, S: int, heads: int, device) -> torch.Tensor:
    """Zeroed fp32 dQ workspace of merlot_attention_bwd_workspace_bytes(B, S, heads) as [parts*B*S, H]."""
    H = heads * 64
    n = L.lib().merlot_attention_bwd_workspace_bytes(B, S, heads) // 4
    return torch.zeros((n // H, H), dtype=torch.float32, device=device)


def attention_bwd(qkv, ctx, d_ctx, lse, B, S, heads, valid=None, dqkv=None, dq_accum=None, dsum=None, pair=(0, 0),
                  d_bias_qkv=None, dropout=(0.0, 0, 0)):
    """K3: dqkv[B*S,3H] from d_ctx.  dq_accum: fp32 workspace of merlot_attention_bwd_workspace_bytes (see the header);
    in atomic mode (long sequences) it must be zero on entry and is returned zeroed.  d_bias_qkv: optional fp32 [3H] that
    the column sums of dqkv (the gradient of the fused q/k/v bias) are added to.  dropout: the forward's (p, seed, site)."""
    a = _attn_desc(qkv, B, S, heads, valid, pair, dropout)
    H = heads * a.head_dim
    dev = qkv.device
    if dqkv is None:
        dqkv = torch.empty((B * S, 3 * H), dtype=torch.bfloat16, device=dev)
    need = L.lib().merlot_attention_bwd_workspace_bytes(B, S, heads) // 4
    if dq_accum is None:
        dq_accum = torch.zeros((need // H, H), dtype=torch.float32, device=dev)
    assert dq_accum.numel() >= need, "dq_accum smaller than merlot_attention_bwd_workspace_bytes"
    if dsum is None:
        dsum = torch.empty((B, heads, S), dtype=torch.float32, device=dev)
    a.ctx, a.ld_ctx, a.lse = ctx.data_ptr(), ctx.stride(0), lse.data_ptr()
    assert d_ctx.stride(0) == ctx.stride(0)
    a.d_ctx, a.dsum = d_ctx.data_ptr(), dsum.data_ptr()
    a.dq_accum, a.ld_dq = dq_accum.data_ptr(), H
    a.dqkv, a.ld_dqkv = dqkv.data_ptr(), dqkv.stride(0)
    if d_bias_qkv is not None:
        _require_cuda(d_bias_qkv)
        assert d_bias_qkv.dtype == torch.float32 and d_bias_qkv.numel() == 3 * H and d_bias_qkv.is_contiguous()
        a.d_bias_qkv = d_bias_qkv.data_ptr()
    L.lib().merlot_attention_bwd(C.byref(a), _stream())
    return dqkv


def attention_probs(qkv, lse, B, S, heads, valid=None, out=None, pair=(0, 0), dropout=(0.0, 0, 0), alpha=1.0, beta=0.0):
    """Export path: out = beta * out + alpha * (head-mean probabilities [B,S,S] fp32 of one layer, one layer of
    `self_attn_probs`), after the forward's dropout=(p, seed, site).  The defaults write the layer's map; beta = 0 never
    reads `out`."""
    a = _attn_desc(qkv, B, S, heads, valid, pair, dropout)
    if out is None:
        assert beta == 0.0, "beta != 0 accumulates into an existing `out`"
        out = torch.empty((B, S, S), dtype=torch.float32, device=qkv.device)
    _require_cuda(out)
    assert out.dtype == torch.float32 and out.numel() == B * S * S and out.is_contiguous()
    a.lse = lse.data_ptr()
    L.lib().merlot_attention_probs(C.byref(a), out.data_ptr(), float(alpha), float(beta), _stream())
    return out


def attention_log_probs(probs, valid, P, out=None):
    """attention_log (model/modeling.py:186-203) of a layer-mean map probs [B,S,S] fp32 with token validity uint8 [B*S]
    and P vision positions: out[4] = {lang2lang, lang2viz, viz2lang, viz2viz} block sums over the total, in a fixed order."""
    _require_cuda(probs, valid, out)
    B, S, _ = probs.shape
    assert probs.dtype == torch.float32 and probs.is_contiguous() and probs.shape == (B, S, S)
    assert valid.dtype == torch.uint8 and valid.numel() == B * S and valid.is_contiguous()
    if out is None:
        out = torch.empty(4, dtype=torch.float32, device=probs.device)
    L.lib().merlot_attention_log_probs(probs.data_ptr(), valid.data_ptr(), B, S, int(P), out.data_ptr(), _stream())
    return out


def attention_colsum(qkv, lse, colsum, B, S, heads, valid=None, pair=(0, 0), dropout=(0.0, 0, 0), colsum2=None, split=0,
                     valid_q=False):
    """K4: colsum[B,S] += mean_h sum_q P[b,h,q,k] (recomputed from q,k,lse), P after the forward's dropout=(p, seed, site).
    With colsum2, queries >= split add into colsum2 instead; valid_q: padding queries add nothing (attention_log)."""
    a = _attn_desc(qkv, B, S, heads, valid, pair, dropout)
    assert colsum.dtype == torch.float32 and colsum.numel() == B * S
    a.lse, a.colsum = lse.data_ptr(), colsum.data_ptr()
    if colsum2 is not None:
        assert colsum2.dtype == torch.float32 and colsum2.numel() == B * S
        a.colsum2, a.colsum_split = colsum2.data_ptr(), int(split)
    a.colsum_valid_q = int(valid_q)
    L.lib().merlot_attention_colsum(C.byref(a), _stream())
    return colsum


# ---------------------------------------------------------------------------------------------------------------
# thin wrappers over the remaining C-ABI entry points (pointer plumbing only)
# ---------------------------------------------------------------------------------------------------------------
def _f32(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return 1
    assert t.dtype == torch.bfloat16, t.dtype
    return 0


def layernorm_fwd(x, y, gamma, beta, mean=None, rstd=None, rows=None, remap=(0, 0, 0), dropout=(0.0, 0, 0), eps=1e-5):
    _require_cuda(x, y, gamma, beta, mean, rstd)
    d = L.merlot_ln_t()
    H = gamma.numel()
    d.x, d.x_f32, d.ld_x = x.data_ptr(), _f32(x), x.stride(-2)
    d.y, d.y_f32, d.ld_y = y.data_ptr(), _f32(y), y.stride(-2)
    d.gamma, d.beta = gamma.data_ptr(), beta.data_ptr()
    d.mean, d.rstd = _ptr(mean), _ptr(rstd)
    d.rows = x.numel() // H if rows is None else rows
    d.H, d.eps = H, eps
    d.map_per, d.map_stride, d.map_off = remap
    d.dropout_p, d.dropout_seed, d.dropout_site = dropout
    L.lib().merlot_layernorm_fwd(C.byref(d), _stream())
    return y


_ln_ws = {}


def _ln_workspace(H: int, device) -> torch.Tensor:
    # one workspace PER STREAM: ln_bwd writes per-block partials and a second launch reads them back, so two streams that
    # run LayerNorm backwards concurrently (language-only vs joint encoder) must never share the buffer
    key = (H, str(device), int(torch.cuda.current_stream(device).cuda_stream))
    if key not in _ln_ws:
        _ln_ws[key] = torch.empty(L.lib().merlot_layernorm_bwd_workspace_bytes(H), dtype=torch.uint8, device=device)
    return _ln_ws[key]


def layernorm_bwd(dy, x, mean, rstd, gamma, dx, dgamma, dbeta, dres=None, rows=None, remap=(0, 0, 0), dropout=(0.0, 0, 0)):
    _require_cuda(dy, x, mean, rstd, gamma, dx, dgamma, dbeta, dres)
    d = L.merlot_ln_bwd_t()
    H = gamma.numel()
    d.dy, d.dy_f32, d.ld_dy = dy.data_ptr(), _f32(dy), dy.stride(-2)
    d.x, d.x_f32, d.ld_x = x.data_ptr(), _f32(x), x.stride(-2)
    d.mean, d.rstd, d.gamma = mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr()
    if dres is not None:
        d.dres, d.ld_dres = dres.data_ptr(), dres.stride(-2)
    d.dx, d.dx_f32, d.ld_dx = dx.data_ptr(), _f32(dx), dx.stride(-2)
    d.dgamma, d.dbeta = dgamma.data_ptr(), dbeta.data_ptr()
    d.workspace = _ln_workspace(H, x.device).data_ptr()
    d.rows = x.numel() // H if rows is None else rows
    d.H = H
    d.map_per, d.map_stride, d.map_off = remap
    d.dropout_p, d.dropout_seed, d.dropout_site = dropout
    L.lib().merlot_layernorm_bwd(C.byref(d), _stream())
    return dx


def layernorm_bwd_fused(dy, x, mean, rstd, gamma, dx, dgamma, dbeta, dres=None, dmask=None, dbias=None, dropout=(0.0, 0, 0)):
    """The transformer stacks' LayerNorm backward (bf16, dense rows): dx = LN'(dy) + dres, dmask = dropout_bwd(dx),
    dbias += colsum(dmask or dx), dgamma / dbeta accumulated."""
    _require_cuda(dy, x, mean, rstd, gamma, dx, dgamma, dbeta, dres, dmask, dbias)
    H = gamma.numel()
    p, seed, site = dropout
    L.lib().merlot_layernorm_bwd_fused(dy.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(),
                                       _ptr(dres), dx.data_ptr(), _ptr(dmask), dgamma.data_ptr(), dbeta.data_ptr(), _ptr(dbias),
                                       None, x.numel() // H, H, p, seed, site, _stream())
    return dx


def dropout_apply(x, y, p, seed, site):
    rows, N = x.numel() // x.shape[-1], x.shape[-1]
    L.lib().merlot_dropout_apply(x.data_ptr(), x.stride(-2), y.data_ptr(), y.stride(-2), rows, N, p, seed, site, _stream())
    return y


def bias_grad(dy, out, rows=None, N=None, dropout=(0.0, 0, 0)):
    """out[n] += sum_m dy[m, n]; with dropout=(p, seed, site), dy first goes through that forward dropout mask."""
    N = out.numel() if N is None else N
    rows = dy.numel() // dy.stride(-2) if rows is None else rows
    p, seed, site = dropout
    L.lib().merlot_bias_grad(dy.data_ptr(), _f32(dy), dy.stride(-2), rows, N, out.data_ptr(), p, seed, site, _stream())


def gather_rows(src, idx, dst, n=None, H=None):
    H = src.shape[-1] if H is None else H
    n = idx.numel() if n is None else n
    assert idx.dtype == torch.int32
    L.lib().merlot_gather_rows(src.data_ptr(), _f32(src), src.stride(-2), idx.data_ptr(), dst.data_ptr(), _f32(dst),
                               dst.stride(-2), n, H, _stream())
    return dst


def scatter_add_rows(src, idx, dst, n=None, H=None, scale=1.0):
    H = dst.shape[-1] if H is None else H
    n = idx.numel() if n is None else n
    assert idx.dtype == torch.int32
    L.lib().merlot_scatter_add_rows(src.data_ptr(), _f32(src), src.stride(-2), idx.data_ptr(), dst.data_ptr(), _f32(dst),
                                    dst.stride(-2), n, H, scale, _stream())
    return dst


def gelu_f32(x, y):
    L.lib().merlot_gelu_f32(x.data_ptr(), y.data_ptr(), x.numel(), _stream())
    return y


def gelu_bwd_f32(dy, pre, dx):
    L.lib().merlot_gelu_bwd_f32(dy.data_ptr(), pre.data_ptr(), dx.data_ptr(), dy.numel(), _stream())
    return dx


def cast_f32_to_bf16(x, y):
    assert x.dtype == torch.float32 and y.dtype == torch.bfloat16 and x.numel() == y.numel()
    L.lib().merlot_cast_f32_to_bf16(x.data_ptr(), y.data_ptr(), x.numel(), _stream())
    return y


def cast_bf16_to_f32(x, y):
    assert x.dtype == torch.bfloat16 and y.dtype == torch.float32 and x.numel() == y.numel() and x.is_contiguous()
    L.lib().merlot_cast_bf16_to_f32(x.data_ptr(), y.data_ptr(), x.numel(), _stream())
    return y


def l2norm_fwd(x, y, inv):
    L.lib().merlot_l2norm_fwd(x.data_ptr(), y.data_ptr(), inv.data_ptr(), x.shape[0], x.shape[1], _stream())


def l2norm_bwd(dy, y, inv, dx):
    L.lib().merlot_l2norm_bwd(dy.data_ptr(), y.data_ptr(), inv.data_ptr(), dx.data_ptr(), y.shape[0], y.shape[1], _stream())


def softmax_ce_fwd(logits, labels, Cn, loss, lse, correct=None):
    L.lib().merlot_softmax_ce_fwd(logits.data_ptr(), logits.stride(0), labels.data_ptr(), logits.shape[0], Cn, loss.data_ptr(),
                                  lse.data_ptr(), _ptr(correct), _stream())


def softmax_ce_bwd(logits, labels, Cn, lse, coeff, dlogits):
    L.lib().merlot_softmax_ce_bwd(logits.data_ptr(), logits.stride(0), labels.data_ptr(), logits.shape[0], Cn, lse.data_ptr(),
                                  coeff.data_ptr(), dlogits.data_ptr(), _f32(dlogits), dlogits.stride(0), _stream())


def patch_im2col(image, a, P):
    N, H0, W0, _ = image.shape
    assert image.dtype == torch.bfloat16 and image.is_contiguous()
    L.lib().merlot_patch_im2col(image.data_ptr(), a.data_ptr(), N, H0, W0, P, _stream())


def ws_weights(w2d: torch.Tensor, rows_pad: int) -> torch.Tensor:
    """K13: weight-standardised bf16 GEMM operand [rows_pad, cout] of a conv kernel stored as fp32 [kh*kw*cin, cout]."""
    rows, cout = w2d.shape
    out = torch.empty((rows_pad, cout), dtype=torch.bfloat16, device=w2d.device)
    L.lib().merlot_ws_weights(w2d.data_ptr(), rows, rows_pad, cout, out.data_ptr(), _stream())
    return out


def im2col3x3(x: torch.Tensor, N, h, w, Cin, stride, out: torch.Tensor, sub_half=False):
    L.lib().merlot_im2col3x3(x.data_ptr(), N, h, w, Cin, stride, int(sub_half), out.data_ptr(), out.stride(0), _stream())


def group_norm_fwd(x, gamma, beta, y, stats, N, HW, Cc, groups=32, eps=1e-4, relu=True, shortcut=None):
    L.lib().merlot_group_norm_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), _ptr(shortcut), y.data_ptr(), stats.data_ptr(),
                                  N, HW, Cc, groups, eps, int(relu), _stream())


def avgpool2_same(x, N, h, w, Cc, y):
    L.lib().merlot_avgpool2_same(x.data_ptr(), N, h, w, Cc, y.data_ptr(), _stream())


def group_norm_bwd(dy, x, y, stats, gamma, dx, dshortcut, dgamma, dbeta, red, N, HW, Cc, groups=32, eps=1e-4, relu=True):
    L.lib().merlot_group_norm_bwd(dy.data_ptr(), x.data_ptr(), _ptr(y), stats.data_ptr(), gamma.data_ptr(), dx.data_ptr(),
                                  _ptr(dshortcut), dgamma.data_ptr(), dbeta.data_ptr(), red.data_ptr(), N, HW, Cc, groups, eps,
                                  int(relu), _stream())


def avgpool2_same_bwd(dy, N, h, w, Cc, dx):
    L.lib().merlot_avgpool2_same_bwd(dy.data_ptr(), N, h, w, Cc, dx.data_ptr(), _stream())


def col2im3x3(dcol, N, h, w, Cin, stride, dx):
    L.lib().merlot_col2im3x3(dcol.data_ptr(), N, h, w, Cin, stride, dcol.stride(0), dx.data_ptr(), _stream())


def ws_weights_bwd(dws, w2d, dw2d):
    rows, cout = w2d.shape
    L.lib().merlot_ws_weights_bwd(dws.data_ptr(), dws.stride(0), w2d.data_ptr(), rows, cout, dw2d.data_ptr(), _stream())


class WsPlan:
    """Every conv kernel of the hybrid stem as one table for merlot_ws_weights_multi / merlot_ws_weights_bwd_multi:
    `wstd[name]` bf16 [rows_pad, cout] standardised operands, `dws[name]` fp32 [rows_pad, cout] views of ONE gradient arena
    (zeroed with a single memset before the wgrad GEMMs accumulate into it)."""

    def __init__(self, kernels, grads, device):
        # kernels / grads: {name: fp32 [rows, cout] parameter / gradient views of the arenas}, in creation order
        self.names = list(kernels)
        total, offs = 0, {}
        for n in self.names:
            rows, cout = kernels[n].shape
            kp = (rows + 7) // 8 * 8
            offs[n] = (total, kp, cout)
            total += kp * cout
        self.dws_arena = torch.zeros(total, dtype=torch.float32, device=device)
        self.wstd_arena = torch.empty(total, dtype=torch.bfloat16, device=device)
        self.wstd = {n: self.wstd_arena[o:o + kp * c].view(kp, c) for n, (o, kp, c) in offs.items()}
        self.dws = {n: self.dws_arena[o:o + kp * c].view(kp, c) for n, (o, kp, c) in offs.items()}
        items = (L.merlot_ws_item_t * len(self.names))()
        b0 = 0
        for i, n in enumerate(self.names):
            rows, cout = kernels[n].shape
            it = items[i]
            it.w, it.out, it.dws, it.dw = kernels[n].data_ptr(), self.wstd[n].data_ptr(), self.dws[n].data_ptr(), grads[n].data_ptr()
            it.rows, it.rows_pad, it.cout, it.ld_dws, it.block0 = rows, offs[n][1], cout, cout, b0
            b0 += (cout + 31) // 32
        self.n_blocks = b0
        raw = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8)
        self.items_dev = raw.to(device)
        self.key = tuple(kernels[n].data_ptr() for n in self.names)

    def standardise(self):
        L.lib().merlot_ws_weights_multi(self.items_dev.data_ptr(), len(self.names), self.n_blocks, _stream())

    def zero_grads(self):
        self.dws_arena.zero_()

    def backward(self):
        L.lib().merlot_ws_weights_bwd_multi(self.items_dev.data_ptr(), len(self.names), self.n_blocks, _stream())


FRAME_FIELDS = ("src_offset", "src_h", "src_w", "scaled_h", "scaled_w", "offset_y", "offset_x", "method", "augment")


def frame_table(plan, src_bytes: int) -> np.ndarray:
    """merlot_frame_t descriptors of a frame plan: `plan` maps every FRAME_FIELDS key to n integers and "factor" to [n, 3]
    floats.  The kernel reads the table unchecked, so every frame is checked here against the header's conditions."""
    n = len(plan["src_h"])
    t = np.zeros(n, dtype=np.dtype(L.merlot_frame_t))
    for k in FRAME_FIELDS:
        t[k] = np.asarray(plan[k], dtype=np.int64)
    fac = np.asarray(plan["factor"], dtype=np.float32).reshape(n, 3)
    t["factor_r"], t["factor_g"], t["factor_b"] = fac[:, 0], fac[:, 1], fac[:, 2]
    ok = ((t["src_h"] >= 1) & (t["src_w"] >= 1) & (t["scaled_h"] >= 1) & (t["scaled_w"] >= 1) & (t["offset_y"] >= 0) &
          (t["offset_x"] >= 0) & (t["method"] >= 0) & (t["method"] <= 3) & (t["augment"] >= 0) & (t["augment"] <= 2) &
          (t["src_offset"] >= 0) & (t["src_offset"] + 3 * t["src_h"].astype(np.int64) * t["src_w"] <= src_bytes))
    if n == 0 or not ok.all():
        bad = np.flatnonzero(~ok)[:4].tolist()
        raise L.MerlotShapeError(L.MERLOT_ESHAPE, f"frames_prepare: invalid frame descriptors {bad} (of {n})")
    return t


def frames_prepare(src: torch.Tensor, plan, out_h: int, out_w: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """K14: bf16 [n, out_h, out_w, 3] <- convert, resize_and_pad, where(isfinite), augment and cast of n uint8 HWC frames packed
    in `src` (a uint8 CUDA tensor), as `plan` (see frame_table) says.  Enqueued on the current stream."""
    _require_cuda(src, out)
    assert src.dtype == torch.uint8 and src.is_contiguous()
    table = frame_table(plan, src.numel())
    n = len(table)
    if out is None:
        out = torch.empty((n, out_h, out_w, 3), dtype=torch.bfloat16, device=src.device)
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and tuple(out.shape) == (n, out_h, out_w, 3)
    table_dev = torch.from_numpy(table.view(np.uint8)).pin_memory().to(src.device, non_blocking=True)
    mean_ws = torch.empty(n * 3, dtype=torch.float32, device=src.device)
    L.lib().merlot_frames_prepare(table_dev.data_ptr(), n, src.data_ptr(), out_h, out_w, mean_ws.data_ptr(), out.data_ptr(),
                                  _stream())
    return out


def crc32c_multi(views, out: Optional[torch.Tensor] = None):
    """K15: standard CRC-32C (unmasked) of every uint8 CUDA view in `views`, in one launch.  Views may start at any byte,
    be empty or overlap.  With `out` (an int32 CUDA tensor of len(views) entries) the CRCs stay on the device, enqueued on the
    current stream, and `out` is returned; otherwise this synchronises and returns a list of ints."""
    n = len(views)
    if n == 0:
        return out if out is not None else []
    table = np.zeros(n, dtype=np.dtype(L.merlot_crc_seg_t))
    for i, v in enumerate(views):
        _require_cuda(v)
        if v.dtype != torch.uint8 or v.dim() != 1 or (v.numel() > 1 and v.stride(0) != 1):
            raise L.MerlotShapeError(L.MERLOT_ESHAPE, f"crc32c_multi: view {i} is not a contiguous 1-D uint8 tensor")
        table["ptr"][i], table["bytes"][i] = v.data_ptr(), v.numel()
    dev = views[0].device
    result = out if out is not None else torch.empty(n, dtype=torch.int32, device=dev)
    assert result.dtype == torch.int32 and result.is_cuda and result.numel() == n and result.is_contiguous()
    table_dev = torch.from_numpy(table.view(np.uint8)).pin_memory().to(dev, non_blocking=True)
    L.lib().merlot_crc32c_multi(table_dev.data_ptr(), n, result.data_ptr(), _stream())
    if out is not None:
        return out
    return (result.cpu().numpy().view(np.uint32)).tolist()


def add_bf16(a, b, out):
    L.lib().merlot_add_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), _stream())


def vit_assemble_fwd(patch, pos_table, cls_emb, xsum, N, h1, w1, ncls, H):
    L.lib().merlot_vit_assemble_fwd(patch.data_ptr(), pos_table.data_ptr(), cls_emb.data_ptr(), xsum.data_ptr(), N, h1, w1, ncls,
                                    64, H, _stream())


def vit_assemble_bwd(dxsum, dpatch, N, np_, ncls, H):
    L.lib().merlot_vit_assemble_bwd(dxsum.data_ptr(), dpatch.data_ptr(), N, np_, ncls, H, _stream())


def viz_assemble_fwd(hv, img_idx_pe, img_idx, fpos, fcls, xsum, img_trg, N, h1, w1, ncls, sp, H):
    L.lib().merlot_viz_assemble_fwd(hv.data_ptr(), img_idx_pe.data_ptr(), img_idx.data_ptr(), fpos.data_ptr(), fcls.data_ptr(),
                                    xsum.data_ptr(), img_trg.data_ptr(), N, h1, w1, ncls, sp, 64, H, _stream())


def viz_assemble_bwd(dxsum, d_img_trg, dhv, N, h1, w1, ncls, sp, H):
    L.lib().merlot_viz_assemble_bwd(dxsum.data_ptr(), _ptr(d_img_trg), dhv.data_ptr(), N, h1, w1, ncls, sp, H, _stream())


def embed_fwd(ids, emb, pos, xsum, Lseq):
    L.lib().merlot_embed_fwd(ids.data_ptr(), emb.data_ptr(), pos.data_ptr(), xsum.data_ptr(), ids.numel(), Lseq, emb.shape[1],
                             _stream())


def group_rowsum(src, groups, per, t0, nt, idxmap, dst, H):
    L.lib().merlot_group_rowsum(src.data_ptr(), src.stride(-2), groups, per, t0, nt, _ptr(idxmap), dst.data_ptr(), dst.stride(-2),
                                H, _stream())


def segment_rowsum_scatter(src, n_seg, per, idx, dst, H):
    L.lib().merlot_segment_rowsum_scatter(src.data_ptr(), src.stride(-2), n_seg, per, idx.data_ptr(), dst.data_ptr(),
                                          dst.stride(-2), H, _stream())


def ids_valid(ids, valid):
    L.lib().merlot_ids_valid(ids.data_ptr(), valid.data_ptr(), ids.numel(), _stream())


def joint_valid(ids, valid, B, P, Lseq):
    L.lib().merlot_joint_valid(ids.data_ptr(), valid.data_ptr(), B, P, Lseq, _stream())


def joint_valid_img(ids, img_mask, valid, B, nt, ni, span, Lseq):
    """img_mask: uint8 [B // nt, ni] on the device, or None (every image valid)."""
    L.lib().merlot_joint_valid_img(ids.data_ptr(), _ptr(img_mask), valid.data_ptr(), B, nt, ni, span, Lseq, _stream())


def mlm_index(ids, masked_idx, rows, targets, B, Lseq, k, P):
    L.lib().merlot_mlm_index(ids.data_ptr(), masked_idx.data_ptr(), rows.data_ptr(), targets.data_ptr(), B, Lseq, k, P, _stream())


def temporal_labels(video_src_ids, shuffled_idx, labels, weights, B, n):
    L.lib().merlot_temporal_labels(video_src_ids.data_ptr(), shuffled_idx.data_ptr(), labels.data_ptr(), weights.data_ptr(), B, n,
                                   _stream())


def weighted_loss(per_row, correct, weights, nz_labels, denom_mode, scale, out2, coeff):
    L.lib().merlot_weighted_loss(per_row.data_ptr(), _ptr(correct), _ptr(weights), _ptr(nz_labels), per_row.numel(), denom_mode,
                                 scale, out2.data_ptr(), _ptr(coeff), _stream())


def small_gemm(A, sam, sak, B, sbn, sbk, Cm, M, N, K, alpha=1.0, beta=0.0):
    L.lib().merlot_small_gemm_f32(A.data_ptr(), sam, sak, B.data_ptr(), sbn, sbk, Cm.data_ptr(), Cm.stride(0), M, N, K, alpha,
                                  beta, _stream())


def ctr_split(x, out, ld, seg_stride, lo_mask):
    """K16: the fp32 rows of x as three bf16 segments of out (hi, or lo where bit s of lo_mask is set)."""
    assert x.dtype == torch.float32 and out.dtype == torch.bfloat16 and x.stride(1) == 1
    L.lib().merlot_ctr_split(x.data_ptr(), x.shape[0], x.shape[1], x.stride(0), out.data_ptr(), ld, seg_stride, lo_mask, _stream())


def ctr_dlogits(logits, labels, C, lse, coeff, scale, dsh, dsv):
    """K16: dS = scale * coeff * (softmax - onehot) as its bf16 hi/lo GEMM operands dsh [rows, >=3C] and dsv [3 rows, >=C]."""
    assert dsh.dtype == torch.bfloat16 and dsv.dtype == torch.bfloat16
    L.lib().merlot_ctr_dlogits(logits.data_ptr(), logits.stride(0), labels.data_ptr(), logits.shape[0], C, lse.data_ptr(),
                               coeff.data_ptr(), scale, dsh.data_ptr(), dsh.stride(0), dsv.data_ptr(), dsv.stride(0), _stream())


def rank_topk(scores, pos, k, greater=None, ties=None, topk_idx=None, topk_val=None):
    """K17: per row r of fp32 scores [rows, cols] (any row stride >= cols), with p = scores[r, pos[r]]: greater[r] (entries
    > p; -1 when p is NaN, -2 when pos[r] is outside the row), ties[r] (other entries == p) and the k largest entries by
    (score descending, index ascending) as topk_idx / topk_val [rows, k] (index -1, value NaN past the non-NaN entries).
    Returns (greater, ties, topk_idx, topk_val)."""
    _require_cuda(scores, pos, greater, ties, topk_idx, topk_val)
    assert scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1
    assert pos.dtype == torch.int32 and pos.is_contiguous() and pos.numel() == scores.shape[0]
    rows, dev = scores.shape[0], scores.device
    greater = torch.empty(rows, dtype=torch.int32, device=dev) if greater is None else greater
    ties = torch.empty(rows, dtype=torch.int32, device=dev) if ties is None else ties
    topk_idx = torch.empty((rows, k), dtype=torch.int32, device=dev) if topk_idx is None else topk_idx
    topk_val = torch.empty((rows, k), dtype=torch.float32, device=dev) if topk_val is None else topk_val
    for t, dt in ((greater, torch.int32), (ties, torch.int32), (topk_idx, torch.int32), (topk_val, torch.float32)):
        assert t.dtype == dt and t.is_contiguous() and t.numel() == rows * (1 if t.dim() == 1 else k)
    L.lib().merlot_rank_topk(scores.data_ptr(), rows, scores.shape[1], max(scores.stride(0), scores.shape[1]), pos.data_ptr(), k,
                             greater.data_ptr(), ties.data_ptr(), topk_idx.data_ptr(), topk_val.data_ptr(), _stream())
    return greater, ties, topk_idx, topk_val


def axpby(x, y, a=1.0, b=1.0):
    L.lib().merlot_axpby_f32(x.data_ptr(), y.data_ptr(), x.numel(), a, b, _stream())


def mask_draws(B, Lseq, num_to_mask, vocab_size, span_probs, seed, device, out=None):
    """The tf.random draws of mask_inputs on device (no host RNG, no host->device copy); returns the dict mask_inputs takes."""
    if out is None:
        out = {"gumbel": torch.empty((B, Lseq), dtype=torch.float32, device=device),
               "span_lower": torch.empty((B, max(num_to_mask, 1)), dtype=torch.int32, device=device),
               "span_upper": torch.empty((B, max(num_to_mask, 1)), dtype=torch.int32, device=device),
               "option": torch.empty((B * Lseq,), dtype=torch.int32, device=device),
               "rand_ids": torch.empty((B * Lseq,), dtype=torch.int32, device=device)}
    L.lib().merlot_mask_draws(out["gumbel"].data_ptr(), out["span_lower"].data_ptr(), out["span_upper"].data_ptr(),
                              out["option"].data_ptr(), out["rand_ids"].data_ptr(), B * Lseq, B * num_to_mask, int(vocab_size),
                              span_probs[0], span_probs[1], seed, _stream())
    return out


def mask_inputs(ids, attn_summ, draws, masked_ids, masked_idx, valid_out, num_topk, num_to_mask, do_spanbert, mask_token, consts):
    m = L.merlot_mask_t()
    B, Lseq = ids.shape
    m.ids, m.attn_summ, m.gumbel = ids.data_ptr(), _ptr(attn_summ), draws["gumbel"].data_ptr()
    m.span_lower, m.span_upper = _ptr(draws.get("span_lower")), _ptr(draws.get("span_upper"))
    m.option, m.rand_ids = draws["option"].data_ptr(), draws["rand_ids"].data_ptr()
    m.masked_ids, m.masked_idx, m.valid_out = masked_ids.data_ptr(), masked_idx.data_ptr(), _ptr(valid_out)
    m.B, m.L, m.num_topk, m.num_to_mask, m.do_spanbert, m.mask_token = B, Lseq, num_topk, num_to_mask, int(do_spanbert), mask_token
    m.w_delta, m.w_non, m.logw_top, m.logw_non, m.w_max = consts
    L.lib().merlot_mask_inputs(C.byref(m), _stream())


def adamw_step(p, g, m, v, p_bf16, n, beta1, omb1, beta2, omb2, eps, lr_t, wd, grad_scale, zero_grad):
    """K10 on n elements.  m and v are both float32 (use_bfloat16_adam: False) or both bfloat16 (bf16 m, sign-packed v)."""
    if m.dtype != v.dtype or m.dtype not in (torch.float32, torch.bfloat16):
        raise L.MerlotError(L.MERLOT_EINVAL, f"adamw_step: m and v must be both float32 or both bfloat16, got {m.dtype} and {v.dtype}")
    d = L.merlot_adamw_t()
    d.p, d.g, d.m, d.v, d.p_bf16, d.n = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), _ptr(p_bf16), n
    d.beta1, d.one_minus_beta1, d.beta2, d.one_minus_beta2 = beta1, omb1, beta2, omb2
    d.epsilon, d.lr_t, d.weight_decay, d.grad_scale, d.zero_grad = eps, lr_t, wd, grad_scale, int(zero_grad)
    d.moments_f32 = int(m.dtype == torch.float32)
    L.lib().merlot_adamw_step(C.byref(d), _stream())


def clip_by_global_norm(g, clip_norm, scratch_f64, norm_out):
    L.lib().merlot_clip_by_global_norm(g.data_ptr(), g.numel(), clip_norm, scratch_f64.data_ptr(), _ptr(norm_out), _stream())


def clip_accumulate(acc, g, clip_norm, scratch_f64, norm_out):
    """acc += g * clip_norm / max(||g||, clip_norm), then g = 0 (norm_out <- ||g||, on the device)."""
    _require_cuda(acc, g, scratch_f64, norm_out)
    if acc.numel() != g.numel() or acc.dtype != torch.float32 or g.dtype != torch.float32:
        raise L.MerlotError(L.MERLOT_EINVAL, f"clip_accumulate: acc and g must be float32 of one length, got {acc.dtype} "
                                             f"[{acc.numel()}] and {g.dtype} [{g.numel()}]")
    L.lib().merlot_clip_accumulate(acc.data_ptr(), g.data_ptr(), g.numel(), clip_norm, scratch_f64.data_ptr(), _ptr(norm_out),
                                   _stream())
