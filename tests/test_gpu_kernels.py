"""GPU parity tests (run on an H100: pytest -m gpu): every CUDA kernel family against the oracle on the same
seeded inputs, through the C-ABI.  Tolerances: bit-exact for integer/index work and the packed bf16 Adam moments;
bf16 tensor-core outputs compared in relative Frobenius norm against the fp32 oracle evaluated on the SAME bf16-rounded
inputs (GEMM fp32-out 1e-4; bf16-out / attention 1e-2 -- one bf16 rounding is 2^-9 = 2e-3 per element)."""
import itertools

import numpy as np
import pytest
import torch

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def keep_ref(seed, site, rows, N, p):
    """float {0, 1} [rows, N]: the restated counter-based dropout mask (oracle/dropout_mask.py)."""
    return torch.from_numpy(DM.counter_dropout_keep(seed, site, rows, N, p)).float()


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


# ---------------------------------------------------------------------------------------------------------------
# K1 GEMM: all operand-major modes, ragged shapes (every Appendix-B family incl. N = 50370 and M = 200)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K,bn", [(128, 256, 64, 256), (200, 264, 136, 0), (1024, 2304, 768, 0), (3168, 768, 3072, 128),
                                      (8, 8, 8, 0), (130, 50376, 768, 0)])
def test_gemm_modes(ops, a_mn, b_mn, M, N, K, bn):
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("MN-major operands need 16-byte aligned rows")
    g = torch.Generator().manual_seed(M + N + K)
    a = (torch.randn((K, M) if a_mn else (M, K), generator=g) * 0.5).bfloat16()
    b = (torch.randn((K, N) if b_mn else (N, K), generator=g) * 0.5).bfloat16()
    out = ops.gemm(a.to(DEV), b.to(DEV), a_mn_major=a_mn, b_mn_major=b_mn, out_dtype=torch.float32, block_n=bn)
    A = a.float().t() if a_mn else a.float()
    Bm = b.float() if b_mn else b.float().t()
    assert rel(out, A @ Bm) < 1e-4


def test_gemm_epilogues(ops):
    g = torch.Generator().manual_seed(1)
    M, N, K = 520, 768, 768
    a = (torch.randn(M, K, generator=g) * 0.3).bfloat16()
    w = (torch.randn(K, N, generator=g) * 0.05).bfloat16()
    bias = torch.randn(N, generator=g)
    resid = torch.randn(M, N, generator=g).bfloat16()
    p = {"d/kernel": w.float(), "d/bias": bias}
    base = O.dense(a.float(), p, "d")  # tf.layers.dense restatement
    ad, wd, bd, rd = a.to(DEV), w.to(DEV), bias.to(DEV), resid.to(DEV)
    assert rel(ops.gemm(ad, wd, b_mn_major=True, bias=bd), base) < 6e-3
    assert rel(ops.gemm(ad, wd, b_mn_major=True, bias=bd, resid=rd), base + resid.float()) < 6e-3
    pre = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    act = ops.gemm(ad, wd, b_mn_major=True, bias=bd, gelu=True, out_pre=pre)
    assert rel(pre, base) < 6e-3 and rel(act, O.gelu(base)) < 6e-3
    aux = torch.randn(M, N, generator=g).bfloat16()
    x = aux.float().requires_grad_(True)
    O.gelu(x).sum().backward()
    assert rel(ops.gemm(ad, wd, b_mn_major=True, dgelu_aux=aux.to(DEV)), (a.float() @ w.float()) * x.grad) < 6e-3
    # the pair the stacks use: the forward saves gelu'(pre) (GELU_GRAD_OUT), the FFN2 dgrad multiplies by it (MUL_AUX)
    for kw in (dict(), dict(block_n=128), dict(block_n=256)):
        gsave = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        act2 = ops.gemm(ad, wd, b_mn_major=True, bias=bd, gelu=True, out_pre=gsave, gelu_grad_out=True, **kw)
        xb = base.clone().requires_grad_(True)
        O.gelu(xb).sum().backward()
        assert rel(act2, O.gelu(base)) < 6e-3 and rel(gsave, xb.grad) < 6e-3
        assert rel(ops.gemm(ad, wd, b_mn_major=True, mul_aux=gsave, **kw), (a.float() @ w.float()) * gsave.float().cpu()) < 6e-3
    dy = (torch.randn(M, N, generator=g) * 0.1).bfloat16()
    dw = torch.zeros(K, N, dtype=torch.float32, device=DEV)
    for _ in range(2):  # accumulation semantics of the flat gradient arena (shared `encoder` weights get two passes)
        ops.gemm(ad, dy.to(DEV), a_mn_major=True, b_mn_major=True, out=dw, atomic=True, M=K, N=N, K=M)
    assert rel(dw, 2 * (a.float().t() @ dy.float())) < 1e-4
    o1 = ops.gemm(ad, wd, b_mn_major=True, bias=bd, dropout_p=0.1, dropout_seed=7, dropout_site=3)
    o2 = ops.gemm(ad, wd, b_mn_major=True, bias=bd, dropout_p=0.1, dropout_seed=7, dropout_site=3)
    o3 = ops.gemm(ad, wd, b_mn_major=True, bias=bd, dropout_p=0.1, dropout_seed=8, dropout_site=3)
    assert torch.equal(o1, o2) and not torch.equal(o1, o3)
    assert abs((o1 == 0).float().mean().item() - 0.1) < 0.01
    kept = (o1 != 0).cpu()
    assert rel(o1.cpu()[kept], (base / 0.9)[kept]) < 6e-3  # inverted dropout scaling (tf.nn.dropout)


@pytest.mark.parametrize("bn", [128, 192, 256])
@pytest.mark.parametrize("M,N", [(300, 264), (130, 1000), (515, 72)])
def test_gemm_epilogue_instances(ops, bn, M, N):
    """Every epilogue feature combination the model uses (plain, bias, resid, bias+resid, alpha, bias+gelu dual, gelu',
    gelu'+resid, split-K fp32 red.add) on every tile width, with ragged M and N edges (N % 64 != 0, N % 32 != 0): the
    epilogue passes each warp's rows through a per-warp fp32 smem slot and clips per 8-column group and per row."""
    g = torch.Generator().manual_seed(M * 7 + N)
    K = 200
    a = (torch.randn(M, K, generator=g) * 0.3).bfloat16()
    w = (torch.randn(K, N, generator=g) * 0.1).bfloat16()
    bias = torch.randn(N, generator=g)
    resid = torch.randn(M, N, generator=g).bfloat16()
    aux = torch.randn(M, N, generator=g).bfloat16()
    base = a.float() @ w.float()
    ad, wd, bd, rd, xd = a.to(DEV), w.to(DEV), bias.to(DEV), resid.to(DEV), aux.to(DEV)
    kw = dict(b_mn_major=True, block_n=bn)
    assert rel(ops.gemm(ad, wd, **kw), base) < 6e-3
    assert rel(ops.gemm(ad, wd, bias=bd, **kw), base + bias) < 6e-3
    assert rel(ops.gemm(ad, wd, resid=rd, **kw), base + resid.float()) < 6e-3
    assert rel(ops.gemm(ad, wd, bias=bd, resid=rd, **kw), base + bias + resid.float()) < 6e-3
    assert rel(ops.gemm(ad, wd, bias=bd, resid=rd, alpha=0.5, **kw), 0.5 * base + bias + resid.float()) < 6e-3  # generic instance
    pre = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    act = ops.gemm(ad, wd, bias=bd, gelu=True, out_pre=pre, **kw)
    assert rel(pre, base + bias) < 6e-3 and rel(act, O.gelu(base + bias)) < 6e-3
    x = aux.float().requires_grad_(True)
    O.gelu(x).sum().backward()
    assert rel(ops.gemm(ad, wd, dgelu_aux=xd, **kw), base * x.grad) < 6e-3
    assert rel(ops.gemm(ad, wd, dgelu_aux=xd, resid=rd, **kw), base * x.grad + resid.float()) < 6e-3  # gelu' + unprefetched residual
    dw = torch.zeros(K, N, dtype=torch.float32, device=DEV)  # split-K fp32 accumulation (EPI 2) with ragged N
    dy = (torch.randn(M, N, generator=g) * 0.1).bfloat16()
    ops.gemm(ad, dy.to(DEV), a_mn_major=True, b_mn_major=True, out=dw, atomic=True, M=K, N=N, K=M, block_n=bn)
    assert rel(dw, a.float().t() @ dy.float()) < 1e-4
    # operands that are not 16-byte aligned: a bias view at a float offset, fp32 outputs at a float offset (plain and red.add)
    bias_off = torch.zeros(N + 1, device=DEV)[1:]
    bias_off.copy_(bd)
    assert rel(ops.gemm(ad, wd, bias=bias_off, **kw), base + bias) < 6e-3
    o32 = torch.zeros(M * N + 1, device=DEV)[1:].view(M, N)
    ops.gemm(ad, wd, out=o32, **kw)
    assert rel(o32, base) < 1e-4
    dw2 = torch.zeros(K * N + 1, device=DEV)[1:].view(K, N)
    ops.gemm(ad, dy.to(DEV), a_mn_major=True, b_mn_major=True, out=dw2, atomic=True, M=K, N=N, K=M, block_n=bn)
    assert rel(dw2, a.float().t() @ dy.float()) < 1e-4


def test_gemm_shape_errors(ops):
    from merlot_b200._lib import MerlotShapeError
    a = torch.zeros(16, 12, dtype=torch.bfloat16, device=DEV)  # lda = 12 not a multiple of 8
    b = torch.zeros(16, 12, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(MerlotShapeError):
        ops.gemm(a, b)
    assert issubclass(MerlotShapeError, ValueError)  # the reference raises ValueError on shape mismatches


# ---------------------------------------------------------------------------------------------------------------
# K2/K3/K4 attention
# ---------------------------------------------------------------------------------------------------------------
def _attn_case(B, S, heads, masked, seed):
    """Seeded bf16 qkv [B*S, 3H] -- masked: ragged valid lengths and a hole in the last sequence -- and the fp32 reference of
    utils/transformer.py:98-120 on the same rounded values.  Returns the generator (for further draws), qkv, the uint8
    validity [B*S] or None, the reference probabilities [B, heads, S, S] and context [B*S, H], and grad(d_ctx), the
    reference dqkv [B*S, 3H] for an upstream gradient d_ctx [B*S, H]."""
    g = torch.Generator().manual_seed(seed)
    H = heads * 64
    qkv = torch.randn(B * S, 3 * H, generator=g).bfloat16()
    valid = None
    mask = None
    if masked:
        lens = torch.randint(max(1, S // 3), S + 1, (B,), generator=g)
        v2 = (torch.arange(S)[None] < lens[:, None])
        if S > 10:
            v2[-1, 5:9] = False
        valid = v2.to(torch.uint8).reshape(-1).contiguous()
        vf = v2.float()
        mask = vf[:, None, :] * vf[:, :, None]
    x = qkv.float().reshape(B, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    q, k, v = (x[i].clone().requires_grad_(True) for i in range(3))
    probs, ctx4 = O.attention_core(q, k, v, mask)
    ctx_ref = ctx4.permute(0, 2, 1, 3).reshape(B * S, H)

    def grad(d_ctx):
        gq, gk, gv = torch.autograd.grad(ctx_ref, (q, k, v), d_ctx.float(), retain_graph=True)
        return torch.stack([gq, gk, gv], 0).permute(1, 3, 0, 2, 4).reshape(B * S, 3 * H)
    return g, qkv, valid, probs.detach(), ctx_ref.detach(), grad


def _assert_dqkv(dqkv, ref, H):
    for i in range(3):
        assert rel(dqkv[:, i * H:(i + 1) * H], ref[:, i * H:(i + 1) * H]) < 1.5e-2, "qkv"[i]


@pytest.mark.parametrize("B,S,heads,masked", [(1, 128, 1, False), (2, 64, 2, True), (2, 266, 12, False), (2, 396, 12, True),
                                              (3, 93, 4, True), (1, 885, 2, True), (1, 1, 1, False)])
def test_attention_fwd_bwd_colsum(ops, B, S, heads, masked):
    g, qkv, valid, probs, ctx_ref, ref_grad = _attn_case(B, S, heads, masked, seed=S)
    H = heads * 64
    vd = valid.to(DEV) if valid is not None else None
    ctx, lse = ops.attention_fwd(qkv.to(DEV), B, S, heads, vd)
    assert rel(ctx, ctx_ref) < 1e-2
    d_ctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16()
    # padding QUERY rows get a gradient too (they never do in the model): the reference's scores*m - 1e10*(1-m) keeps their
    # uniform probabilities in dV and sends nothing into q / k (utils/transformer.py:109-112)
    dqkv = ops.attention_bwd(qkv.to(DEV), ctx, d_ctx.to(DEV), lse, B, S, heads, vd)
    _assert_dqkv(dqkv, ref_grad(d_ctx), H)
    colsum = torch.zeros(B, S, device=DEV)
    ops.attention_colsum(qkv.to(DEV), lse, colsum, B, S, heads, vd)
    assert rel(colsum, probs.mean(1).sum(1)) < 2e-3  # head-mean, summed over queries (transformer.py:208-209)


# merlot_attention_bwd reduces dQ in one of two ways, chosen by merlot_attention_bwd_dq_parts(S): up to 4 key tiles of 128
# (S <= 512) every tile stores its own fp32 slice and the finish pass adds the slices in a fixed order; longer sequences
# red.add into ONE slice that the finish pass sets back to zero for the next layer (0 = atomic mode).
DQ_MODE_CASES = [(128, 1), (129, 2), (512, 4), (513, 0), (640, 0), (1100, 0), (3968, 0)]  # (S, parts); 3968: the longest S
# Bias gradient against the fp32 reference's column sums.  The q and v column sums do not cancel and keep about the element
# error of the bf16 gradient (one bf16 rounding: 2^-9 = 2e-3); the k block, zero in exact arithmetic, is measured against
# the column sums of |dK|.  Observed on an H100 SXM 80 GB (400 W limit) over all DQ_MODE_CASES: q 3.0e-3, v 1.4e-3, k 3.2e-4.
BIAS_GRAD_BAR = 1e-2


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("S,parts", DQ_MODE_CASES)
def test_attention_bwd_dq_modes(ops, S, parts, masked):
    """Both dQ modes and their boundary (S = 512 / 513) up to the longest accepted sequence: dq / dk / dv against the fp32
    reference, and the fused q/k/v bias gradient, added to a non-zero buffer, against (a) the exact column sums of the bf16
    dqkv the finish pass wrote (only the fp32 summation order differs) and (b) the column sums of the fp32 reference
    gradient.  (b) cannot use the element bar: the k block of the bias gradient is zero in exact arithmetic (softmax is
    shift invariant), so the kernel's k block is pure rounding noise of the cancelling dK rows."""
    from merlot_b200._lib import lib
    assert lib().merlot_attention_bwd_dq_parts(S) == parts  # a changed MAX_DQ_PARTS must not move cases between modes silently
    B, heads = (1, 2) if S > 2048 else (2, 2)
    g, qkv, valid, _, ctx_ref, ref_grad = _attn_case(B, S, heads, masked, seed=2 * S + masked)
    H = heads * 64
    vd = valid.to(DEV) if valid is not None else None
    ctx, lse = ops.attention_fwd(qkv.to(DEV), B, S, heads, vd)
    assert rel(ctx, ctx_ref) < 1e-2
    d_ctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16()
    start = torch.randn(3 * H, generator=g) * 0.1
    d_bias = start.to(DEV)
    dqkv = ops.attention_bwd(qkv.to(DEV), ctx, d_ctx.to(DEV), lse, B, S, heads, vd, d_bias_qkv=d_bias)
    ref = ref_grad(d_ctx)
    _assert_dqkv(dqkv, ref, H)
    d_bias = d_bias.cpu().double()
    assert rel(d_bias, start.double() + dqkv.cpu().double().sum(0)) < 1e-5
    got, ref = d_bias - start.double(), ref.double()
    for i, name in enumerate("qkv"):
        blk = slice(i * H, (i + 1) * H)
        if name == "k":  # zero up to fp32 rounding: the error against the size of the terms that cancel
            err = float((got[blk] - ref[:, blk].sum(0)).norm() / ref[:, blk].abs().sum(0).norm())
        else:
            err = rel(got[blk], ref[:, blk].sum(0))
        assert err < BIAS_GRAD_BAR, (name, err)


@pytest.mark.parametrize("S,masked", [(640, True), (1100, False), (129, True), (512, False)])
def test_attention_bwd_workspace_contract(ops, S, masked):
    """The dQ workspace as consecutive layers of a stack use it: one buffer, several backwards.  Atomic mode (S > 512): the
    workspace starts zeroed, every call's result matches its own reference and the call hands the workspace back exactly
    zero -- a slice left dirty would pollute the dQ of every later layer.  Slices mode: NaN in the workspace before each call
    must not reach the result, so every slice is fully overwritten."""
    from merlot_b200._lib import lib
    parts = lib().merlot_attention_bwd_dq_parts(S)
    assert (parts == 0) == (S > 512)
    B, heads = 2, 2
    g, qkv, valid, _, _, ref_grad = _attn_case(B, S, heads, masked, seed=3 * S + masked)
    H = heads * 64
    vd = valid.to(DEV) if valid is not None else None
    qd = qkv.to(DEV)
    ctx, lse = ops.attention_fwd(qd, B, S, heads, vd)
    ws = ops.attention_bwd_workspace(B, S, heads, DEV)
    for rep in range(2):
        if parts:
            ws.fill_(float("nan"))
        d_ctx = (torch.randn(B * S, H, generator=g) * (0.1 if rep == 0 else 0.3)).bfloat16()
        dqkv = ops.attention_bwd(qd, ctx, d_ctx.to(DEV), lse, B, S, heads, vd, dq_accum=ws)
        assert torch.isfinite(dqkv.float()).all()
        _assert_dqkv(dqkv, ref_grad(d_ctx), H)
        if not parts:
            assert torch.equal(ws, torch.zeros_like(ws)), rep


def test_attention_rejects_sequences_past_the_validity_mask(ops):
    """The kernels keep token validity as a bitmask of 4096 positions and the host accepts sequences up to one 128-row tile
    shorter: S = 3968 is the longest (test_attention_bwd_dq_modes runs it).  S = 3969 raises MerlotShapeError in the host-side
    check of forward, backward and column sums before anything is launched: every output keeps its sentinel."""
    from merlot_b200._lib import MerlotShapeError, lib
    B, S, heads, H = 1, 3969, 1, 64
    qkv = torch.zeros(B * S, 3 * H, dtype=torch.bfloat16, device=DEV)
    zeros = torch.zeros(B * S, H, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(B, heads, S, device=DEV)
    ctx_out = torch.full((B * S, H), 7.0, dtype=torch.bfloat16, device=DEV)
    lse_out = torch.full((B, heads, S), 7.0, device=DEV)
    dqkv = torch.full((B * S, 3 * H), 7.0, dtype=torch.bfloat16, device=DEV)
    dsum = torch.full((B, heads, S), 7.0, device=DEV)  # a launched dsum pass would write rowsum(0 * 0) = 0 here
    colsum = torch.full((B, S), 7.0, device=DEV)
    torch.cuda.synchronize()
    lib().merlot_reset_launch_count()
    with pytest.raises(MerlotShapeError):
        ops.attention_fwd(qkv, B, S, heads, ctx=ctx_out, lse=lse_out)
    with pytest.raises(MerlotShapeError):
        ops.attention_bwd(qkv, zeros, zeros, lse, B, S, heads, dqkv=dqkv, dsum=dsum)
    with pytest.raises(MerlotShapeError):
        ops.attention_colsum(qkv, lse, colsum, B, S, heads)
    assert lib().merlot_launch_count() == 0
    torch.cuda.synchronize()
    for t in (ctx_out, lse_out, dqkv, dsum, colsum):
        assert bool((t.float() == 7.0).all())


@pytest.mark.parametrize("B,P,chunk,nch,heads", [(2, 13, 8, 4, 2), (2, 100, 32, 5, 4), (1, 266, 32, 4, 12), (2, 0, 16, 6, 1), (1, 70, 33, 3, 2),
                                                 (1, 56, 80, 8, 2), (1, 60, 100, 6, 2)])
def test_attention_disable_pairwise_lang_attn(ops, B, P, chunk, nch, heads):
    """model/modeling.py:160-168: segment 0 = P vision tokens, segment 1 + c = language chunk c; a pair attends iff it shares a
    segment or either side is a vision token.  K2 / K3 / K4 and the export kernel take (P, chunk) and derive the partner set of
    every row arithmetically; the oracle gets the explicit [B, S, S] mask the reference builds.  Chunk boundaries fall inside
    32-position words, inside and across the 64 / 128-wide tiles, and some tokens are padding.  S = 696 and 660 (more than 4
    key tiles) run the backward's atomic dQ mode."""
    S = P + chunk * nch
    g = torch.Generator().manual_seed(S + chunk)
    H = heads * 64
    qkv = torch.randn(B * S, 3 * H, generator=g).bfloat16()
    v2 = torch.ones(B, S, dtype=torch.bool)
    for b in range(B):  # ragged captions: the tail of some chunks is padding (ids == 0)
        for c in range(nch):
            n_pad = int(torch.randint(0, chunk // 2 + 1, (1,), generator=g))
            if n_pad:
                v2[b, P + (c + 1) * chunk - n_pad:P + (c + 1) * chunk] = False
    seg = torch.cat([torch.zeros(P, dtype=torch.int64), 1 + torch.arange(chunk * nch) // chunk])
    can = (seg[:, None] == seg[None]) | (seg == 0)[None] | (seg == 0)[:, None]
    mask = (v2[:, None, :] & v2[:, :, None] & can[None]).float()
    valid = v2.to(torch.uint8).reshape(-1).contiguous().to(DEV)
    x = qkv.float().reshape(B, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    q, k, v = (x[i].clone().requires_grad_(True) for i in range(3))
    probs, ctx4 = O.attention_core(q, k, v, mask)
    ctx_ref = ctx4.permute(0, 2, 1, 3).reshape(B * S, H)
    pair = (P, chunk)
    ctx, lse = ops.attention_fwd(qkv.to(DEV), B, S, heads, valid, pair=pair)
    assert rel(ctx, ctx_ref) < 1e-2
    # the mask did something: without it the same inputs give a different context
    ctx_nopair, _ = ops.attention_fwd(qkv.to(DEV), B, S, heads, valid)
    assert nch < 2 or rel(ctx_nopair, ctx_ref) > 1e-2
    d_ctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16()
    dqkv = ops.attention_bwd(qkv.to(DEV), ctx, d_ctx.to(DEV), lse, B, S, heads, valid, pair=pair)
    ctx_ref.backward(d_ctx.float())
    ref = torch.stack([q.grad, k.grad, v.grad], 0).permute(1, 3, 0, 2, 4).reshape(B * S, 3 * H)
    for i in range(3):
        assert rel(dqkv[:, i * H:(i + 1) * H], ref[:, i * H:(i + 1) * H]) < 1.5e-2
    colsum = torch.zeros(B, S, device=DEV)
    ops.attention_colsum(qkv.to(DEV), lse, colsum, B, S, heads, valid, pair=pair)
    assert rel(colsum, probs.detach().mean(1).sum(1)) < 2e-3
    pm = ops.attention_probs(qkv.to(DEV), lse, B, S, heads, valid, pair=pair)
    assert rel(pm, probs.detach().mean(1)) < 2e-3
    # a language token of chunk 0 puts (numerically) nothing on a language token of chunk 1
    if nch >= 2:
        assert float(pm[0, P, P + chunk].abs()) < 1e-6


# ---------------------------------------------------------------------------------------------------------------
# K5 LayerNorm, CE, l2norm
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,H", [(1, 768), (1000, 768), (37, 128), (8512, 768)])
def test_layernorm_fwd_bwd(ops, rows, H):
    g = torch.Generator().manual_seed(rows)
    x = (torch.randn(rows, H, generator=g) * 2 + 0.5).bfloat16()
    gam, bet = torch.randn(H, generator=g), torch.randn(H, generator=g)
    xr = x.float().requires_grad_(True)
    gr, br = gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
    y_ref = O.layer_norm(xr, {"l/gamma": gr, "l/beta": br}, "l")
    y = torch.empty(rows, H, dtype=torch.bfloat16, device=DEV)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    ops.layernorm_fwd(x.to(DEV), y, gam.to(DEV), bet.to(DEV), mean, rstd)
    assert rel(y, y_ref) < 4e-3
    dy = torch.randn(rows, H, generator=g).bfloat16()
    dres = torch.randn(rows, H, generator=g).bfloat16()
    y_ref.backward(dy.float())
    dx = torch.empty(rows, H, dtype=torch.bfloat16, device=DEV)
    dg, db = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    ops.layernorm_bwd(dy.to(DEV), x.to(DEV), mean, rstd, gam.to(DEV), dx, dg, db, dres=dres.to(DEV))
    assert rel(dx, xr.grad + dres.float()) < 6e-3
    assert rel(dg, gr.grad) < 2e-3 and rel(db, br.grad) < 2e-3


@pytest.mark.parametrize("rows,H,with_dres,p", [(1, 768, True, 0.1), (13, 64, False, 0.0), (1777, 768, True, 0.1), (8512, 768, True, 0.1),
                                                  (8512, 768, False, 0.0), (5000, 1024, True, 0.1), (20000, 256, True, 0.0), (3, 512, True, 0.1),
                                                  (1031, 256, True, 0.5), (640, 768, False, 0.2)])
def test_layernorm_bwd_fused(ops, rows, H, with_dres, p):
    """The stacks' fused LayerNorm backward (rows arrive through per-warp bulk-copy rings): every output against the fp32 graph
    of utils/model_utils.py:113-130, the dropout mask against merlot_dropout_apply and against the restated mask bit for bit,
    the bias gradient against the exact column sums of what the kernel wrote; row counts that leave warps without rows, with
    one row, and with many ring refills."""
    g = torch.Generator().manual_seed(rows + H)
    x = (torch.randn(rows, H, generator=g) * 2 + 0.5).bfloat16()
    gam = torch.randn(H, generator=g)
    xr, gr, br = x.float().requires_grad_(True), gam.clone().requires_grad_(True), torch.zeros(H, requires_grad=True)
    y_ref = O.layer_norm(xr, {"l/gamma": gr, "l/beta": br}, "l")
    dy = torch.randn(rows, H, generator=g).bfloat16()
    dres = torch.randn(rows, H, generator=g).bfloat16() if with_dres else None
    y_ref.backward(dy.float())
    mu = x.float().mean(-1)
    rs = torch.rsqrt(x.float().var(-1, unbiased=False) + 1e-5)
    dx = torch.full((rows, H), float("nan"), dtype=torch.bfloat16, device=DEV)
    dmask = torch.full((rows, H), float("nan"), dtype=torch.bfloat16, device=DEV)
    dg, db, dbias = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    seed, site = (2 ** 40 + 3, 223) if rows % 2 else (7, 3)  # odd row counts: a seed with a non-zero high key word
    for rep in range(2):  # twice: the accumulators add up, the ring barriers start fresh every launch
        ops.layernorm_bwd_fused(dy.to(DEV), x.to(DEV), mu.to(DEV), rs.to(DEV), gam.to(DEV), dx, dg, db,
                                dres=None if dres is None else dres.to(DEV), dmask=dmask, dbias=dbias, dropout=(p, seed, site))
    want = xr.grad + (dres.float() if with_dres else 0.0)
    assert torch.isfinite(dx.float()).all()
    assert rel(dx, want) < 6e-3
    assert rel(dg, 2 * gr.grad) < 2e-3 and rel(db, 2 * br.grad) < 2e-3
    if p > 0:
        ref_mask = torch.empty_like(dx)
        ops.dropout_apply(dx, ref_mask, p, seed, site)
        assert torch.equal(dmask, ref_mask)
        keep = keep_ref(seed, site, rows, H, p)  # dmask = bf16(bf16(dx) * keep * scale)
        assert torch.equal(dmask.cpu(), (dx.cpu().float() * keep * float(DM.dropout_scale(p))).bfloat16())
        assert rel(dbias, 2 * dmask.float().sum(0)) < 1e-5
        kept = float((dmask != 0).float().mean())
        assert abs(kept - (1 - p)) < (0.2 if rows * H < 4096 else 0.02)
    else:
        assert rel(dbias, 2 * dx.float().sum(0)) < 1e-5


def _l2norm_boundary_rows(g, H):
    """Rows whose sum of squares sits at tf.math.l2_normalize's epsilon (1e-12, compared in fp32 on the device):
    0, 0.5e-12 (clamped), exactly the fp32 epsilon, 1.001e-12 and 4e-12 (not clamped).  The `exactly` row has two non-zeros,
    in lanes 0 and 1 of the kernel's warp: its fp32 sum is fl(fl(a^2) + fl(b^2)) == float32(1e-12) in any order, while the
    float64 sum of the oracle is >= 1e-12, so both sides take Maximum's not-clamped branch (the gradient goes to sum x^2 when
    it is >= eps).  The other rows spread over all H columns; their sums are 1e-3 or more away from the epsilon."""
    rows = torch.zeros(5, H)
    for i, s2 in ((1, 0.5e-12), (3, 1.001e-12), (4, 4e-12)):
        u = torch.randn(H, generator=g, dtype=torch.float64)
        rows[i] = (u * (s2 ** 0.5 / u.norm())).float()
    a, b = np.float32(8.944272167354939e-07), np.float32(4.4721355152432807e-07)
    assert np.float32(np.float32(a * a) + np.float32(b * b)) == np.float32(1e-12) and float(a) ** 2 + float(b) ** 2 >= 1e-12
    rows[2, 0], rows[2, 1] = float(a), float(b)
    return rows


# (classes, logits row stride, dlogits dtype, argmax ties): the MLM head's vocabulary with bf16 dlogits (padded to ld 50432),
# the contrastive / temporal heads' small C
CE_CASES = [(50370, 50432, torch.float32, False), (50370, 50432, torch.bfloat16, True), (4, 4, torch.float32, True),
            (32, 32, torch.bfloat16, True), (32, 40, torch.float32, False)]


def _softmax_ce_case(ops, Cn, ld, d_dtype, ties):
    """One CE_CASES entry: raw_cross_entropy_with_logits (utils/model_utils.py:313-332) + argmax accuracy, and its backward into
    fp32 or bf16 dlogits (padded columns exactly 0; bf16 = the fp32 result rounded once).  Ties: several exact maxima in
    different warps, in the same thread and with the label on a later one -- tf.argmax keeps the first."""
    case = (Cn, ld, d_dtype, ties)
    g = torch.Generator().manual_seed(Cn + ld)
    R = 37
    logits = torch.full((R, ld), 1e4)  # padding columns are never read
    logits[:, :Cn] = torch.randn(R, Cn, generator=g) * 3
    labels = torch.randint(0, Cn, (R,), generator=g, dtype=torch.int32)
    if ties:
        spots = [[5, 1000], [37, 290, 700], [100, 356], [Cn - 1, 0]] if Cn > 1000 else [[1, Cn - 1], [0, Cn // 2], [2, 3]]
        for r, cols in enumerate(spots):
            logits[r, :Cn] = torch.randn(Cn, generator=g)
            logits[r, cols] = 9.0
            labels[r] = cols[-1] if r % 2 else cols[0]
    lr = logits[:, :Cn].clone().requires_grad_(True)
    per_ref = O.raw_cross_entropy_with_logits(lr, labels)
    per, lse, corr = (torch.empty(R, device=DEV) for _ in range(3))
    ops.softmax_ce_fwd(logits.to(DEV), labels.to(DEV), Cn, per, lse, corr)
    assert torch.allclose(per.cpu(), per_ref.detach(), rtol=1e-5, atol=1e-5), case
    assert torch.equal(corr.cpu(), (lr.argmax(-1) == labels).float()), case
    if ties:
        assert corr.cpu()[1] == 0.0 and corr.cpu()[0] == 1.0, case  # label on the second maximum / on the first
    coeff = torch.rand(R, generator=g)
    (per_ref * coeff).sum().backward()
    dlog = torch.full((R, ld), float("nan"), dtype=torch.float32, device=DEV)
    ops.softmax_ce_bwd(logits.to(DEV), labels.to(DEV), Cn, lse, coeff.to(DEV), dlog)
    assert rel(dlog[:, :Cn], lr.grad) < 1e-5 and not dlog[:, Cn:].any(), case
    if d_dtype == torch.bfloat16:
        dlb = torch.full((R, ld), float("nan"), dtype=torch.bfloat16, device=DEV)
        ops.softmax_ce_bwd(logits.to(DEV), labels.to(DEV), Cn, lse, coeff.to(DEV), dlb)
        assert torch.equal(dlb, dlog.bfloat16()), case  # padded columns included: exactly 0
        assert rel(dlb[:, :Cn], lr.grad) < 4e-3, case   # one bf16 rounding


def test_softmax_ce_and_l2norm(ops):
    """Softmax cross-entropy for every CE_CASES entry (_softmax_ce_case), then l2_normalize forward / backward on random rows
    and on the epsilon boundary rows of _l2norm_boundary_rows, dx per row against autograd of O.l2_normalize in float64."""
    for case in CE_CASES:
        _softmax_ce_case(ops, *case)
    g = torch.Generator().manual_seed(0)
    H = 768
    x = torch.cat([torch.randn(32, H, generator=g), _l2norm_boundary_rows(g, H)])
    n = x.shape[0]
    xr = x.double().requires_grad_(True)
    y_ref = O.l2_normalize(xr)
    y, inv = torch.empty(n, H, device=DEV), torch.empty(n, device=DEV)
    ops.l2norm_fwd(x.to(DEV), y, inv)
    assert rel(y, y_ref) < 1e-6
    dy = torch.randn(n, H, generator=g, dtype=torch.float64)
    dy = (dy + 30.0 * y_ref.detach()).float()  # a component along y: the clamped branch drops its projection
    y_ref.backward(dy.double())
    dx = torch.empty(n, H, device=DEV)
    ops.l2norm_bwd(dy.to(DEV), y, inv, dx)
    dxc = dx.cpu().double()
    for r in range(n):
        assert rel(dxc[r], xr.grad[r]) < 1e-5, (r, rel(dxc[r], xr.grad[r]))


# ---------------------------------------------------------------------------------------------------------------
# K12 masking: bit-exact given injected draws (integer path)
# ---------------------------------------------------------------------------------------------------------------
# L > 1024: the block's 1024 threads stride over the positions; L = 3072 is the language length of configs[4]
@pytest.mark.parametrize("B,L,spanbert,use_attn", [(8, 128, True, True), (3, 32, True, True), (4, 128, False, True),
                                                   (2, 64, True, False), (2, 1024, True, True), (2, 1500, True, True),
                                                   (2, 1500, False, True), (1, 3072, True, True), (1, 3072, False, True)])
def test_mask_inputs_bit_exact(ops, tiny_cfg, B, L, spanbert, use_attn):
    cfg = dict(tiny_cfg, masking_do_spanbert=spanbert, masking_use_attn=use_attn)
    g = torch.Generator().manual_seed(L + B)
    ids = torch.randint(100, 50370, (B, L), generator=g, dtype=torch.int32)
    ids[:, ::32] = O.START
    ids[:, -L // 8:] = 0
    summ = torch.rand(B, L, generator=g) * 12
    summ[:, 5] = summ[:, 9]  # force an exact tie: tf.math.top_k keeps the lower index
    k = int(L * 0.2)
    draws = O.make_mask_draws(B, L, k, 50370, seed=B)
    ref = O.mask_inputs(ids, summ if use_attn else None, cfg, draws)
    if use_attn:
        w = torch.tensor([1.0, 0.0]) * np.float32(ref["topk_val"] - 0.01) + np.float32(0.01)
        consts = (float(np.float32(ref["topk_val"] - 0.01)), float(np.float32(0.01)), float(torch.log(w)[0]), float(torch.log(w)[1]),
                  float(w.max()))
    else:
        consts = (0.0, 1.0, 0.0, 0.0, 1.0)
    m_ids = torch.empty(B, L, dtype=torch.int32, device=DEV)
    m_idx = torch.empty(B, k, dtype=torch.int32, device=DEV)
    ops.mask_inputs(ids.to(DEV), summ.to(DEV) if use_attn else None, {k_: v.to(DEV) for k_, v in draws.items()}, m_ids, m_idx, None,
                    int(L * 0.2), k, spanbert, O.MASK, consts)
    assert torch.equal(m_idx.cpu(), ref["masked_idx"])
    assert torch.equal(m_ids.cpu(), ref["masked_ids"])


# ---------------------------------------------------------------------------------------------------------------
# K10 AdamW: packed bf16 moments bit-exact over many steps, parameters to 1e-6
# ---------------------------------------------------------------------------------------------------------------
def test_adamw_vs_oracle(ops):
    g = torch.Generator().manual_seed(0)
    n = 100003
    cfg = dict(learning_rate=3e-4, num_train_steps=1000, num_warmup_steps=10, weight_decay_rate=0.1, beta_2=0.98, epsilon=1e-6,
               use_bfloat16_adam=True, param_overrides=[[["bias"], {"weight_decay_rate": 0}]])
    p_ref = {"w/kernel": torch.randn(n, generator=g) * 0.02, "w/bias": torch.randn(n, generator=g) * 0.02}
    opt = O.AdamOracle(p_ref, cfg)
    dev = {k: dict(p=v.clone().to(DEV), m=torch.zeros(n, dtype=torch.bfloat16, device=DEV),
                   v=torch.zeros(n, dtype=torch.bfloat16, device=DEV), pb=torch.zeros(n, dtype=torch.bfloat16, device=DEV))
           for k, v in p_ref.items()}
    for step in range(25):
        grads = {k: torch.randn(n, generator=g) * (10.0 ** float(torch.randint(-6, 1, (1,), generator=g))) for k in p_ref}
        s = opt.step_scalars()
        opt.apply_gradients(p_ref, grads)
        for k, d in dev.items():
            gd = grads[k].to(DEV)
            wd = 0.1 if "kernel" in k else 0.0
            ops.adamw_step(d["p"], gd, d["m"], d["v"], d["pb"], n, float(s["beta1"]), float(np.float32(1) - s["beta1"]),
                           float(s["beta2"]), float(np.float32(1) - s["beta2"]), float(s["eps"]), float(s["lr_t"]), wd, 1.0, True)
            assert float(gd.abs().max()) == 0.0  # zero_grad
    for k, d in dev.items():
        assert torch.equal(d["m"].cpu(), opt.m[k]), "first moment must be bit-exact"
        assert torch.equal(d["v"].cpu(), opt.v[k]), "packed second moment must be bit-exact"
        assert (d["p"].cpu() - p_ref[k]).abs().max().item() < 1e-6
        assert torch.equal(d["pb"].cpu(), d["p"].cpu().bfloat16())


def test_clip_by_global_norm(ops):
    """tf.clip_by_global_norm (utils/optimization.py:233-237): g * clip / max(norm, clip)."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1000003, generator=g) * 0.01
    x = torch.cat([x, torch.zeros(1)])  # 16-byte friendly length not required
    for clip in (0.5, 1e6):
        gd = x.clone().to(DEV)
        scratch = torch.zeros(1, dtype=torch.float64, device=DEV)
        norm = torch.zeros(1, device=DEV)
        ops.clip_by_global_norm(gd, clip, scratch, norm)
        ref_norm = x.double().norm().item()
        assert abs(float(norm) - ref_norm) < 1e-5 * ref_norm
        ref = x * (clip / max(ref_norm, clip))
        assert rel(gd, ref) < 1e-6


def test_device_mask_draws_distributions_and_bit_exact_masking(ops):
    """merlot_mask_draws: the five tf.random tensors of mask_inputs drawn on device -- right distributions, reproducible from
    the seed -- and K12 fed with them is bit-exact against the oracle fed the very same tensors."""
    from merlot_b200 import ops as o
    B, L, k, V = 64, 128, 25, 50370
    d = o.mask_draws(B, L, k, V, [0.625, 0.25, 0.125], seed=11, device=DEV)
    d2 = o.mask_draws(B, L, k, V, [0.625, 0.25, 0.125], seed=11, device=DEV)
    d3 = o.mask_draws(B, L, k, V, [0.625, 0.25, 0.125], seed=12, device=DEV)
    assert all(torch.equal(d[x], d2[x]) for x in d) and not torch.equal(d["gumbel"], d3["gumbel"])
    g = d["gumbel"].double().cpu()
    assert abs(float(g.mean()) - 0.5772) < 0.03 and abs(float(g.var()) - 1.6449) < 0.1          # Gumbel(0,1): mean gamma, var pi^2/6
    opt = torch.bincount(d["option"].cpu(), minlength=3).double() / (B * L)
    assert (opt - torch.tensor([0.1, 0.8, 0.1])).abs().max() < 0.02
    for name in ("span_lower", "span_upper"):
        f = torch.bincount(d[name].reshape(-1).cpu(), minlength=3).double() / (B * k)
        assert (f - torch.tensor([0.625, 0.25, 0.125])).abs().max() < 0.04
    r = d["rand_ids"].cpu()
    assert int(r.min()) >= 100 and int(r.max()) < V and abs(float(r.double().mean()) - (100 + V) / 2) < 300
    gen = torch.Generator().manual_seed(0)
    ids = torch.randint(100, V, (B, L), generator=gen, dtype=torch.int32)
    ids[:, 0] = 2
    ids[:, 100:] = 0
    summ = torch.rand(B, L, generator=gen)
    cfg = dict(masking_use_topk_from_attn_perc=0.2, masking_choose_topk_prob=0.5, masking_rate=0.2, masking_do_spanbert=True, masking_use_attn=True)
    ref = O.mask_inputs(ids, summ, cfg, {x: v.cpu() for x, v in d.items()})
    import numpy as np
    nontop, top = 0.01, 0.01 * 0.5 * 0.8 / (0.2 * 0.5)
    w = torch.tensor([1.0, 0.0]) * np.float32(top - nontop) + np.float32(nontop)
    consts = (float(np.float32(top - nontop)), float(np.float32(nontop)), float(torch.log(w)[0]), float(torch.log(w)[1]), float(w.max()))
    mi = torch.empty(B, L, dtype=torch.int32, device=DEV)
    mx = torch.empty(B, k, dtype=torch.int32, device=DEV)
    o.mask_inputs(ids.to(DEV), summ.to(DEV), d, mi, mx, None, 25, k, True, 1, consts)
    assert torch.equal(mi.cpu(), ref["masked_ids"]) and torch.equal(mx.cpu(), ref["masked_idx"])


# ---------------------------------------------------------------------------------------------------------------
# Training-mode hidden dropout: every kernel that draws the counter-based mask (GEMM epilogue, LayerNorm forward, both
# LayerNorm backwards, bias gradient, dropout_apply) against the NumPy restatement of its definition, bit for bit.
# Inputs are chosen so that the kernel's output reads the mask back exactly (ones, gamma = 0 / beta = 1, A = 0 / bias = 1).
# ---------------------------------------------------------------------------------------------------------------
DROP_CASES = [(0, 0, 0.1), (7, 1, 0.2), (2 ** 40 + 3, 223, 0.5), (2 ** 40 + 3, 301, 0.1)]  # (seed, site, p)


def _drop_cases(*axes):
    """The product of `axes`, each combination paired with one of DROP_CASES in turn."""
    return [(*combo, *DROP_CASES[i % len(DROP_CASES)]) for i, combo in enumerate(itertools.product(*axes))]


@pytest.mark.parametrize("seed,site,p", DROP_CASES)
@pytest.mark.parametrize("rows,N,ld_x,ld_y", [(1, 8, 8, 8), (37, 136, 136, 136), (515, 72, 96, 104), (8512, 768, 768, 768)])
def test_dropout_apply_mask(ops, rows, N, ld_x, ld_y, seed, site, p):
    """Ones in: every kept element is bf16(1/(1-p)), every dropped one 0.  Leading dimensions larger than N: the mask is
    keyed by row * N + col, not by the leading dimension, and the columns past N are neither read into the mask nor written."""
    x = torch.full((rows, ld_x), 5.0, dtype=torch.bfloat16, device=DEV)
    x[:, :N] = 1.0
    y = torch.full((rows, ld_y), float("nan"), dtype=torch.bfloat16, device=DEV)
    ops.dropout_apply(x[:, :N], y[:, :N], p, seed, site)
    keep = keep_ref(seed, site, rows, N, p)
    assert torch.equal(y[:, :N].cpu(), (keep * float(DM.dropout_scale(p))).bfloat16())
    assert torch.isnan(y[:, N:].float()).all()


@pytest.mark.parametrize("bn,M,N,seed,site,p", [(bn, M, N, *c) for bn, (M, N), *c in _drop_cases((128, 192, 256), ((300, 264), (515, 72), (8512, 768)))])
def test_gemm_dropout_epilogue_mask(ops, bn, M, N, seed, site, p):
    """A = 0, bias = 1: the epilogue's output is exactly keep * scale, and bf16(keep * scale + R) with a residual.  Every tile
    width, ragged M / N edges, and at 8512 x 768 more tiles than SMs (the persistent loop runs several tiles per CTA)."""
    g = torch.Generator().manual_seed(M + N + bn)
    K = 64
    a = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
    w = (torch.randn(K, N, generator=g) * 0.1).bfloat16().to(DEV)
    ones = torch.ones(N, device=DEV)
    resid = torch.randn(M, N, generator=g).bfloat16()
    kw = dict(b_mn_major=True, bias=ones, dropout_p=p, dropout_seed=seed, dropout_site=site, block_n=bn)
    want = keep_ref(seed, site, M, N, p) * float(DM.dropout_scale(p))
    assert torch.equal(ops.gemm(a, w, **kw).cpu(), want.bfloat16())
    assert torch.equal(ops.gemm(a, w, resid=resid.to(DEV), **kw).cpu(), (want + resid.float()).bfloat16())


def test_gemm_dropout_epilogue_values(ops):
    """Non-zero A: (A @ B + bias) * keep / (1 - p) + resid -- the mask sits after the bias and before the residual."""
    g = torch.Generator().manual_seed(3)
    M, N, K = 520, 768, 768
    seed, site, p = 2 ** 40 + 3, 223, 0.2
    a = (torch.randn(M, K, generator=g) * 0.3).bfloat16()
    w = (torch.randn(K, N, generator=g) * 0.05).bfloat16()
    bias = torch.randn(N, generator=g)
    resid = torch.randn(M, N, generator=g).bfloat16()
    out = ops.gemm(a.to(DEV), w.to(DEV), b_mn_major=True, bias=bias.to(DEV), resid=resid.to(DEV), dropout_p=p,
                   dropout_seed=seed, dropout_site=site)
    keep = keep_ref(seed, site, M, N, p)
    want = (a.float() @ w.float() + bias) * keep / (1 - p) + resid.float()
    assert rel(out, want) < 6e-3
    assert rel(out, (a.float() @ w.float()) * keep / (1 - p) + bias + resid.float()) > 6e-3  # mask before the bias: caught


def _remap_rows(rows, remap):
    per, stride, off = remap
    r = torch.arange(rows)
    return (r // per) * stride + off + r % per if per > 0 else r


@pytest.mark.parametrize("x_f32,y_f32,remap,seed,site,p", _drop_cases((False, True), (False, True), ((0, 0, 0), (29, 40, 6))))
def test_layernorm_fwd_dropout_mask(ops, x_f32, y_f32, remap, seed, site, p):
    """gamma = 0, beta = 1: y = keep * scale exactly, in all four x / y dtypes, with and without the row remap of the joint
    encoder's embedding rows.  The mask follows the LOGICAL row; rows the remap skips keep their NaN sentinel.  Then random
    gamma / beta against the fp32 LayerNorm times the mask."""
    rows, H = 203, 256
    g = torch.Generator().manual_seed(rows + int(x_f32) + 2 * int(y_f32))
    x = torch.randn(rows, H, generator=g) * 2 + 0.5
    x = x if x_f32 else x.bfloat16()
    ydt = torch.float32 if y_f32 else torch.bfloat16
    orow = _remap_rows(rows, remap)
    out_rows = int(orow.max()) + 1 + (11 if remap[0] else 0)
    keep = keep_ref(seed, site, rows, H, p)
    scale = float(DM.dropout_scale(p))
    y = torch.full((out_rows, H), float("nan"), dtype=ydt, device=DEV)
    ops.layernorm_fwd(x.to(DEV), y, torch.zeros(H, device=DEV), torch.ones(H, device=DEV), rows=rows, remap=remap,
                      dropout=(p, seed, site))
    yc = y.cpu()
    assert torch.equal(yc[orow], (keep * scale).to(ydt))
    skipped = torch.ones(out_rows, dtype=torch.bool)
    skipped[orow] = False
    assert torch.isnan(yc[skipped].float()).all() and (not remap[0] or bool(skipped.any()))
    gam, bet = torch.randn(H, generator=g), torch.randn(H, generator=g)
    y.fill_(float("nan"))
    ops.layernorm_fwd(x.to(DEV), y, gam.to(DEV), bet.to(DEV), rows=rows, remap=remap, dropout=(p, seed, site))
    want = O.layer_norm(x.float(), {"l/gamma": gam, "l/beta": bet}, "l") * keep * scale
    assert rel(y.cpu()[orow], want) < (1e-5 if y_f32 else 4e-3)


def _ln_bwd_reference(x, dy_logical, dres, gam, bet, keep, scale):
    xr, gr, br = x.float().requires_grad_(True), gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
    y = O.layer_norm(xr, {"l/gamma": gr, "l/beta": br}, "l") * keep * scale
    y.backward(dy_logical.float())
    return xr.grad + dres.float(), gr.grad, br.grad


@pytest.mark.parametrize("x_f32,dy_f32,dx_f32,remap,seed,site,p",
                         [(*d, *rest) for d, *rest in _drop_cases(((False, False, False), (True, False, True), (True, True, True),
                                                                   (False, True, False)), ((0, 0, 0), (37, 50, 5)))])
def test_layernorm_bwd_dropout(ops, x_f32, dy_f32, dx_f32, remap, seed, site, p):
    """The unfused LayerNorm backward of the embedding LayerNorms: dy is the gradient of dropout(LN(x)) (read through the row
    remap), dx / dgamma / dbeta against fp32 autograd under the restated mask; the mask of site + 1 must miss those bounds."""
    rows, H = 333, 384
    g = torch.Generator().manual_seed(rows + int(x_f32) + 2 * int(dy_f32))
    xdt = torch.float32 if x_f32 else torch.bfloat16
    dxdt = torch.float32 if dx_f32 else torch.bfloat16
    x = (torch.randn(rows, H, generator=g) * 2 + 0.5).to(xdt)
    gam, bet = torch.randn(H, generator=g), torch.randn(H, generator=g)
    orow = _remap_rows(rows, remap)
    dy_full = torch.randn(int(orow.max()) + 1, H, generator=g).to(torch.float32 if dy_f32 else torch.bfloat16)
    dres = torch.randn(rows, H, generator=g).to(dxdt)
    xf = x.float()
    mu, rs = xf.mean(-1), torch.rsqrt(xf.var(-1, unbiased=False) + 1e-5)
    dx = torch.full((rows, H), float("nan"), dtype=dxdt, device=DEV)
    dg, db = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    ops.layernorm_bwd(dy_full.to(DEV), x.to(DEV), mu.to(DEV), rs.to(DEV), gam.to(DEV), dx, dg, db, dres=dres.to(DEV), rows=rows,
                      remap=remap, dropout=(p, seed, site))
    scale = float(DM.dropout_scale(p))
    tol = 1e-5 if dx_f32 else 6e-3

    def within(keep):
        want_dx, want_g, want_b = _ln_bwd_reference(x, dy_full[orow], dres, gam, bet, keep, scale)
        return rel(dx, want_dx) < tol and rel(dg, want_g) < 2e-3 and rel(db, want_b) < 2e-3

    assert within(keep_ref(seed, site, rows, H, p))
    assert not within(keep_ref(seed, site + 1, rows, H, p))


@pytest.mark.parametrize("dy_f32,rows,N,ld,seed,site,p", [(f, *shape, *c) for f, shape, *c in _drop_cases((False, True), ((8512, 768, 768), (300, 264, 280)))])
def test_bias_grad_dropout(ops, dy_f32, rows, N, ld, seed, site, p):
    """merlot_bias_grad through the forward dropout mask: dy = 1 gives scale x (kept rows of each column) to 1e-6; random dy
    against fp64 to 1e-5.  A leading dimension larger than N leaves the mask keyed by row * N + col."""
    g = torch.Generator().manual_seed(rows + N)
    dt = torch.float32 if dy_f32 else torch.bfloat16
    keep = keep_ref(seed, site, rows, N, p).double()
    scale = float(DM.dropout_scale(p))
    ones = torch.full((rows, ld), 3.0, dtype=dt, device=DEV)
    ones[:, :N] = 1.0
    out = torch.zeros(N, device=DEV)
    ops.bias_grad(ones[:, :N], out, rows=rows, N=N, dropout=(p, seed, site))
    want = keep.sum(0) * scale
    assert ((out.cpu().double() - want).abs() <= 1e-6 * want).all()
    dy = torch.randn(rows, ld, generator=g).to(dt)
    out.zero_()
    ops.bias_grad(dy.to(DEV)[:, :N], out, rows=rows, N=N, dropout=(p, seed, site))
    assert rel(out, (dy[:, :N].double() * keep * scale).sum(0)) < 1e-5
