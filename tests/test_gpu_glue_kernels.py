"""GPU tests of the glue around the three transformer stacks (pytest -m gpu): token assembly, embedding, gather / scatter,
index and label construction, the loss-head reductions, casts and GeLU, each entry point against a float64 restatement of
the reference lines named in its docstring.  Backward kernels are checked against autograd of the very forward restatement
their forward kernel was checked against.

Two input regimes:
  * exact: small-integer / dyadic fp32 inputs and power-of-two scales, so that every fp32 sum is exact in any order.  Copies,
    gathers, sums, scatter-adds (atomic collisions included) and block sums must then equal the reference bit for bit: a
    missing, duplicated or misindexed term fails whatever the summation order.
  * random: normal inputs, relative Frobenius error against float64 under a bar; the largest value measured on an
    H100 80GB HBM3 (400 W power limit) is written beside each bar."""
import types

import numpy as np
import pytest
import torch

from oracle import merlot_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = torch.float64
TAB = 64  # the 64 x 64 position tables (vision_backbone/.../pos_embs, final_pe/pos_embs)


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return ((a - b).norm() / (b.norm() + 1e-300)).item()


def exact(shape, g, lo=-64, hi=64, den=32):
    """Dyadic fp32 values k / den, k in [lo, hi): every sum of a few thousand of them is exact in fp32 (and in bf16 for one)."""
    return torch.randint(lo, hi, shape, generator=g).float() / den


def inputs(shape, g, regime):
    return exact(shape, g) if regime == "exact" else torch.randn(shape, generator=g)


def check(got, ref, regime, bar, what):
    """exact: bit for bit; random: relative Frobenius error against the float64 reference under `bar`."""
    got = got.detach().cpu()
    if regime == "exact":
        assert torch.equal(got.double(), ref.double()), (what, float((got.double() - ref.double()).abs().max()))
    else:
        err = rel(got, ref)
        assert err <= bar, (what, err)


# Random-regime bar for the fp32 sums below (group / segment row sums, scatter-add, small GEMM, block sums): the fp32
# rounding of sums of a few to a few thousand terms.  Measured maxima per test are in the docstrings; the largest, 6.1e-7,
# is the img_idx_pe gradient (segment sums of up to N * vcl rows).
SUM_BAR = 1e-5


# ---------------------------------------------------------------------------------------------------------------
# K6/K7 token assembly (csrc/assemble.cu)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,H0,W0,P", [(2, 64, 96, 16), (3, 80, 48, 16), (1, 24, 40, 8)])
def test_patch_im2col(ops, N, H0, W0, P):
    """utils/vision_transformer.py:193-205: x - 0.5, then the non-overlapping P x P VALID conv as an im2col GEMM operand, columns
    ordered (kh, kw, c) like the flattened HWIO kernel (the oracle's reshape).  One bf16 rounding on both sides: bit-exact, for
    dyadic pixels (x - 0.5 exact) and for random bf16 pixels."""
    g = torch.Generator().manual_seed(N * H0 + W0)
    h1, w1 = H0 // P, W0 // P
    for img in (torch.randint(0, 65, (N, H0, W0, 3), generator=g).float() / 64, torch.rand(N, H0, W0, 3, generator=g)):
        img = img.bfloat16()
        x = img.float() - 0.5  # :193
        ref = x.reshape(N, h1, P, w1, P, 3).permute(0, 1, 3, 2, 4, 5).reshape(N * h1 * w1, P * P * 3).bfloat16()
        a = torch.full((N * h1 * w1, P * P * 3), float("nan"), dtype=torch.bfloat16, device=DEV)
        ops.patch_im2col(img.to(DEV), a, P)
        assert torch.equal(a.cpu(), ref)


def _vit_forward_ref(patch, pos, cls, N, h1, w1, ncls):
    """utils/vision_transformer.py:229-233: [N, ncls zero slots || patch tokens] + position_embedder2d(h1, w1, ncls)."""
    H = patch.shape[-1]
    p = {"pe/pos_embs": pos.view(1, TAB, TAB, H), "pe/cls_emb": cls.view(1, ncls, H)}
    x = torch.cat([torch.zeros(N, ncls, H, dtype=patch.dtype), patch.view(N, h1 * w1, H)], 1)  # :231
    return (x + O.position_embedder2d(p, "pe", h1, w1, ncls)[None]).reshape(N * (h1 * w1 + ncls), H)  # :232


def _grid_idxmap(nh, nw):
    """Row of grid cell (i, j) in a flattened 64 x 64 position table (MerlotModel._grid_idxmap)."""
    return (torch.arange(nh)[:, None] * TAB + torch.arange(nw)[None]).reshape(-1).to(torch.int32)


@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("N,h1,w1,ncls,H", [(2, 12, 22, 2, 128), (2, 24, 44, 2, 64), (2, 64, 64, 2, 64), (3, 5, 7, 3, 64),
                                            (2, 7, 5, 2, 128), (1, 1, 1, 3, 8)])
def test_vit_assembly_and_table_gradients(ops, N, h1, w1, ncls, H, regime):
    """merlot_vit_assemble_fwd against _vit_forward_ref; merlot_vit_assemble_bwd (patch gradient, bf16) and merlot_group_rowsum
    (cls_emb and pos_embs gradients, added to pre-filled gradient buffers) against autograd of the same restatement.  The 64 x 64
    grid uses the whole position table; pos rows outside the grid must keep their previous gradient.
    Random regime (sums of N terms), measured: cls_emb 3.5e-8, pos_embs 3.1e-8."""
    g = torch.Generator().manual_seed(h1 * 100 + w1 + ncls)
    np_, Sv = h1 * w1, h1 * w1 + ncls
    patch, pos, cls = (inputs(s, g, regime) for s in ((N * np_, H), (TAB * TAB, H), (ncls, H)))
    leaves = [t.double().requires_grad_(True) for t in (patch, pos, cls)]
    xsum_ref = _vit_forward_ref(*leaves, N, h1, w1, ncls)
    xsum = torch.full((N * Sv, H), float("nan"), device=DEV)
    ops.vit_assemble_fwd(patch.to(DEV), pos.to(DEV), cls.to(DEV), xsum, N, h1, w1, ncls, H)
    assert torch.equal(xsum.cpu().double(), xsum_ref.detach().float().double())  # one fp32 add: the rounded exact sum

    dxsum = inputs((N * Sv, H), g, regime)
    d_patch_ref, d_pos_ref, d_cls_ref = torch.autograd.grad(xsum_ref, leaves, dxsum.double())
    dpatch = torch.full((N * np_, H), float("nan"), dtype=torch.bfloat16, device=DEV)
    ops.vit_assemble_bwd(dxsum.to(DEV), dpatch, N, np_, ncls, H)
    assert torch.equal(dpatch.cpu(), d_patch_ref.float().bfloat16())
    g_pos0, g_cls0 = exact((TAB * TAB, H), g), exact((ncls, H), g)  # the gradient arena already holds something
    g_pos, g_cls = g_pos0.to(DEV), g_cls0.to(DEV)
    dx = dxsum.to(DEV)
    ops.group_rowsum(dx, N, Sv, 0, ncls, None, g_cls, H)                                # modeling.py _vit backward
    ops.group_rowsum(dx, N, Sv, ncls, np_, _grid_idxmap(h1, w1).to(DEV), g_pos, H)
    check(g_cls, g_cls0.double() + d_cls_ref, regime, SUM_BAR, "cls_emb")
    check(g_pos, g_pos0.double() + d_pos_ref, regime, SUM_BAR, "pos_embs")
    untouched = torch.ones(TAB * TAB, dtype=torch.bool)
    untouched[_grid_idxmap(h1, w1).long()] = False
    assert torch.equal(g_pos.cpu()[untouched], g_pos0[untouched])


def _viz_forward_ref(hv, img_idx_pe, img_idx, fpos, fcls, N, h1, w1, ncls, sp):
    """model/modeling.py:99-125 with :299-337 on the ViT output hv [N*Sv, H]: img_trg = cls token 1 (:99); the viz tokens are
    cls token 0 || the VALID sp x sp average pool of the patch grid (utils/vision_transformer.py:255-266, the oracle's
    vision_transformer_backbone pooling: the cropped last rows / columns are dropped), plus img_idx_pe[img_idx] (:321-323) and
    position_embedder2d(final_pe, h2, w2, 1) (:327-336).  Returns (xsum [N*vcl, H], img_trg [N, H])."""
    H = hv.shape[-1]
    hv4 = hv.view(N, h1 * w1 + ncls, H)
    cls, seq = hv4[:, :ncls], hv4[:, ncls:]
    h2, w2 = h1 // sp, w1 // sp
    if sp > 1:
        seq = seq.reshape(N, h1, w1, H)[:, :h2 * sp, :w2 * sp].reshape(N, h2, sp, w2, sp, H).mean((2, 4)).reshape(N, h2 * w2, H)
    feats = torch.cat([cls[:, 0, None], seq], 1)
    p = {"fpe/pos_embs": fpos.view(1, TAB, TAB, H), "fpe/cls_emb": fcls.view(1, 1, H)}
    pe = img_idx_pe[img_idx.long()][:, None] + O.position_embedder2d(p, "fpe", h2, w2, 1)[None]
    return (feats + pe).reshape(-1, H), cls[:, 1]


@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("N,h1,w1,sp,ncls,H,with_trg", [
    (4, 12, 22, 2, 2, 128, True), (4, 24, 24, 2, 2, 64, False), (2, 64, 64, 2, 2, 64, True), (4, 5, 7, 1, 2, 64, True),
    (4, 5, 7, 2, 3, 64, False), (4, 7, 5, 3, 2, 64, True), (4, 5, 7, 3, 3, 128, True), (2, 7, 5, 2, 2, 64, True),
    (2, 24, 44, 3, 2, 64, False)])
def test_viz_assembly_and_gradients(ops, N, h1, w1, sp, ncls, H, with_trg, regime):
    """merlot_viz_assemble_fwd against _viz_forward_ref; merlot_viz_assemble_bwd (d hv, bf16, with d_img_trg given or null),
    merlot_segment_rowsum_scatter (img_idx_pe gradient; frames share rows, so the red.add collides) and merlot_group_rowsum
    (final_pe cls / pos gradients) against autograd of it.  Odd grids crop the last row / column of patches when sp > 1:
    their gradient, and that of CLS tokens >= 2 (and of token 1 without d_img_trg), is exactly zero.
    sp = 3 averages with the fp32 factor 1/9, which is not a power of two: the pooled values and their gradients are held to
    two fp32 ulps and one bf16 ulp instead of bit equality.  Random regime, measured: xsum 3.8e-8, img_idx_pe 6.1e-7,
    final_pe cls_emb 4.6e-8, final_pe pos_embs 2.1e-8."""
    g = torch.Generator().manual_seed(h1 * 1000 + w1 * 10 + sp + ncls)
    Sv, h2, w2 = h1 * w1 + ncls, h1 // sp, w1 // sp
    vcl = h2 * w2 + 1
    n_pe = 6
    hv = inputs((N * Sv, H), g, regime).bfloat16()
    img_idx_pe, fpos, fcls = (inputs(s, g, regime) for s in ((n_pe, H), (TAB * TAB, H), (1, H)))
    img_idx = torch.tensor([(3 * i) % 4 for i in range(N)], dtype=torch.int32)  # repeated rows, row n_pe - 1 never used
    img_idx[-1] = n_pe - 2
    leaves = [t.double().requires_grad_(True) for t in (hv.float(), img_idx_pe, fpos, fcls)]
    xsum_ref, trg_ref = _viz_forward_ref(leaves[0], leaves[1], img_idx, leaves[2], leaves[3], N, h1, w1, ncls, sp)
    xsum = torch.full((N * vcl, H), float("nan"), device=DEV)
    trg = torch.full((N, H), float("nan"), device=DEV)
    ops.viz_assemble_fwd(hv.to(DEV), img_idx_pe.to(DEV), img_idx.to(DEV), fpos.to(DEV), fcls.to(DEV), xsum, trg, N, h1, w1, ncls,
                         sp, H)
    assert torch.equal(trg.cpu(), hv.view(N, Sv, H)[:, 1].float())
    if regime == "random":
        check(xsum, xsum_ref.detach(), regime, SUM_BAR, "xsum")
    elif sp == 3:  # two fp32 roundings (the 1/9 factor, the product) on values of magnitude >= 2^-5
        d = (xsum.cpu().double() - xsum_ref.detach()).abs()
        assert bool((d <= 2.0 ** -21 * xsum_ref.detach().abs().clamp(min=1.0)).all()), float(d.max())
    else:
        assert torch.equal(xsum.cpu().double(), xsum_ref.detach())

    dxsum = inputs((N * vcl, H), g, regime)
    d_trg = inputs((N, H), g, regime) if with_trg else None
    outs = [xsum_ref] + ([trg_ref] if with_trg else [])
    grads = [dxsum.double()] + ([d_trg.double()] if with_trg else [])
    d_hv_ref, d_pe_ref, d_fpos_ref, d_fcls_ref = torch.autograd.grad(outs, leaves, grads)
    dhv = torch.full((N * Sv, H), float("nan"), dtype=torch.bfloat16, device=DEV)
    dx = dxsum.to(DEV)
    ops.viz_assemble_bwd(dx, d_trg.to(DEV) if with_trg else None, dhv, N, h1, w1, ncls, sp, H)
    got = dhv.cpu().float().double()
    if sp == 3:  # bf16(fp32(v * fl(1/9))) against v / 9: within one bf16 ulp
        ulp = 2.0 ** (torch.floor(torch.log2(d_hv_ref.abs().clamp(min=2.0 ** -120))) - 7)
        assert bool(((got - d_hv_ref).abs() <= ulp).all())
    else:
        assert torch.equal(dhv.cpu(), d_hv_ref.float().bfloat16())
    dz = got.view(N, Sv, H)
    grid = dz[:, ncls:].reshape(N, h1, w1, H)
    assert not grid[:, h2 * sp:].any() and not grid[:, :, w2 * sp:].any()  # cropped patches
    assert not dz[:, 2:ncls].any() and (with_trg or not dz[:, 1].any())     # unused CLS tokens

    g_pe0, g_fpos0, g_fcls0 = exact((n_pe, H), g), exact((TAB * TAB, H), g), exact((1, H), g)
    g_pe, g_fpos, g_fcls = g_pe0.to(DEV), g_fpos0.to(DEV), g_fcls0.to(DEV)
    ops.segment_rowsum_scatter(dx, N, vcl, img_idx.to(DEV), g_pe, H)                   # modeling.py viz backward
    ops.group_rowsum(dx, N, vcl, 0, 1, None, g_fcls, H)
    ops.group_rowsum(dx, N, vcl, 1, h2 * w2, _grid_idxmap(h2, w2).to(DEV), g_fpos, H)
    check(g_pe, g_pe0.double() + d_pe_ref, regime, SUM_BAR, "img_idx_pe")
    check(g_fcls, g_fcls0.double() + d_fcls_ref, regime, SUM_BAR, "final_pe/cls_emb")
    check(g_fpos, g_fpos0.double() + d_fpos_ref, regime, SUM_BAR, "final_pe/pos_embs")


@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("R,L,V,H,ids_kind", [(3 * 40, 40, 1000, 128, "spread"), (100, 32, 1000, 64, "spread"),
                                              (4096, 64, 50370, 64, "three"), (1, 1, 2, 8, "spread")])
def test_embedding_and_gradients(ops, R, L, V, H, ids_kind, regime):
    """model/modeling.py:262-292 via utils/model_utils.py:238-310 (the oracle's embed_words before its LayerNorm):
    xsum[r] = E[ids[r]] + Pos[r % L].  R = 100, L = 32: the last sequence is partial.  Ids include 0 and V - 1.  When R is a
    whole number of sequences, the word-embedding gradient (merlot_scatter_add_rows, fp32 red.add) and the position-table
    gradient (merlot_group_rowsum) against autograd of the same restatement; "three": 4096 rows land on 3 ids.
    The forward is one fp32 add, bit-exact in both regimes.  Random regime, measured: word_embeddings 1.7e-7,
    position_embeddings 1.4e-7."""
    g = torch.Generator().manual_seed(R + L + V)
    if ids_kind == "three":
        ids = torch.tensor([0, 7, V - 1], dtype=torch.int32)[torch.randint(0, 3, (R,), generator=g)]
    else:
        ids = torch.randint(0, V, (R,), generator=g, dtype=torch.int32)
        ids[0], ids[-1] = 0, V - 1
    emb, pos = inputs((V, H), g, regime), inputs((L, H), g, regime)
    E, Pt = emb.double().requires_grad_(True), pos.double().requires_grad_(True)
    ref = E[ids.long()] + Pt[torch.arange(R) % L]
    xsum = torch.full((R, H), float("nan"), device=DEV)
    ops.embed_fwd(ids.to(DEV), emb.to(DEV), pos.to(DEV), xsum, L)
    assert torch.equal(xsum.cpu().double(), ref.detach().float().double())
    if R % L:
        return
    dx = inputs((R, H), g, regime)
    dE_ref, dP_ref = torch.autograd.grad(ref, (E, Pt), dx.double())
    gE0, gP0 = exact((V, H), g), exact((L, H), g)
    gE, gP = gE0.to(DEV), gP0.to(DEV)
    ops.scatter_add_rows(dx.to(DEV), ids.to(DEV), gE)                   # MerlotModel._embed_bwd
    ops.group_rowsum(dx.to(DEV), R // L, L, 0, L, None, gP, H)
    check(gE, gE0.double() + dE_ref, regime, SUM_BAR, "word_embeddings")
    check(gP, gP0.double() + dP_ref, regime, SUM_BAR, "position_embeddings")


# ---------------------------------------------------------------------------------------------------------------
# gather / scatter-add (csrc/rowwise.cu)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("src_dt,dst_dt", [(torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32),
                                           (torch.float32, torch.float32), (torch.float32, torch.bfloat16)])
def test_gather_rows_dtypes_and_strided_views(ops, src_dt, dst_dt):
    """one_hot_gather (utils/model_utils.py:225-235) as a row gather, all four dtype pairs: dst[i] = src[idx[i]] converted (exact
    widening, or one RNE rounding).  Source and destination are column views of wider matrices, as the temporal head's
    hj[:, :H] / hj[:, H:] halves (modeling.py _temporal): the other half and the rows past n are left alone."""
    g = torch.Generator().manual_seed(int(src_dt == torch.float32) + 2 * int(dst_dt == torch.float32))
    V, H, n = 300, 96, 1000
    src_full = torch.randn(V, 3 * H, generator=g).to(src_dt)
    src = src_full.to(DEV)[:, H:2 * H]
    idx = torch.randint(0, V, (n,), generator=g, dtype=torch.int32)
    idx[:2] = torch.tensor([0, V - 1])
    dst_full = torch.full((n + 3, 2 * H), 5.0, dtype=dst_dt, device=DEV)
    ops.gather_rows(src, idx.to(DEV), dst_full[:, H:], n=n, H=H)
    want = src_full[:, H:2 * H][idx.long()].float().to(dst_dt)
    got = dst_full.cpu()
    assert torch.equal(got[:n, H:], want)
    assert bool((got[:, :H].float() == 5.0).all()) and bool((got[n:].float() == 5.0).all())


@pytest.mark.parametrize("src_dt,scale,n,V", [(torch.float32, 1.0, 4000, 5), (torch.bfloat16, 1.0, 999, 300),
                                              (torch.float32, 0.5, 2500, 1000), (torch.bfloat16, 4.0, 64, 64)])
def test_scatter_add_rows_fp32_collisions(ops, src_dt, scale, n, V):
    """The transpose of the gather: dst[idx[i]] += scale * src[i] with fp32 red.add, every row colliding many times (word
    embedding, MLM rows, pooling gradients).  Dyadic values and power-of-two scales: exact in any order, so equal to the float64
    reference bit for bit; the source is a column view with a leading dimension larger than H."""
    g = torch.Generator().manual_seed(n + V)
    H = 64
    src_full = exact((n, 2 * H), g).to(src_dt)
    idx = torch.randint(0, V, (n,), generator=g, dtype=torch.int32)
    dst0 = exact((V, H), g)
    dst = dst0.to(DEV)
    ops.scatter_add_rows(src_full.to(DEV)[:, H:], idx.to(DEV), dst, scale=scale)
    ref = dst0.double().index_add(0, idx.long(), scale * src_full[:, H:].double())
    assert torch.equal(dst.cpu().double(), ref)


def test_scatter_add_rows_bf16_unique(ops):
    """bf16 destination (unique indices, fp32 source, scale 1): dst[idx[i]] = bf16(dst + src), bit for bit; rows not indexed
    are unchanged.  Random values: one fp32 add and one bf16 rounding on both sides."""
    g = torch.Generator().manual_seed(5)
    V, H, n = 500, 128, 300
    idx = torch.randperm(V, generator=g)[:n].to(torch.int32)
    src = torch.randn(n, 2 * H, generator=g)
    dst0 = torch.randn(V, H, generator=g).bfloat16()
    dst = dst0.to(DEV)
    ops.scatter_add_rows(src.to(DEV)[:, :H], idx.to(DEV), dst)
    want = dst0.clone()
    want[idx.long()] = (dst0[idx.long()].float() + src[:, :H]).bfloat16()
    assert torch.equal(dst.cpu(), want)


# ---------------------------------------------------------------------------------------------------------------
# casts (bfloat16_getter, utils/model_utils.py:572-602)
# ---------------------------------------------------------------------------------------------------------------
def _bits_equal_or_both_nan(got, want):
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan].view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32),
                       want[~nan].view(torch.int16 if want.dtype == torch.bfloat16 else torch.int32))


def test_casts_bit_exact(ops):
    """fp32 -> bf16 against torch's round-to-nearest-even and bf16 -> fp32 against exact widening, bit for bit: +-0, fp32 and
    bf16 subnormals, +-inf, NaN (compared with isnan), exact halfway cases (to even, both directions), values that round up
    to inf, and random bit patterns.  Every bf16 bit pattern widens."""
    special = [0.0, -0.0, float("inf"), -float("inf"), float("nan"), 1e-45, -1e-45, 1e-40, 2.0 ** -126, 2.0 ** -133, -2.0 ** -134,
               1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 1.0 + 2.0 ** -8 + 2.0 ** -23, 3.3895313892515355e38,
               3.3961775292304266e38, 3.4028234663852886e38, -3.4028234663852886e38, 65504.0, 1.0 / 3.0]
    x = torch.tensor(special, dtype=torch.float32)
    halfway = (torch.arange(1, 4097, dtype=torch.int32) << 16) | 0x8000  # mantissa ...1|1000..0 / ...0|1000..0 alternately
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (100000,), generator=torch.Generator().manual_seed(0), dtype=torch.int64)
    x = torch.cat([x, halfway.view(torch.float32), -halfway.view(torch.float32), bits.to(torch.int32).view(torch.float32)])
    x = torch.cat([x, torch.zeros((-x.numel()) % 8)])
    y = torch.empty(x.numel(), dtype=torch.bfloat16, device=DEV)
    ops.cast_f32_to_bf16(x.to(DEV), y)
    _bits_equal_or_both_nan(y.cpu(), x.bfloat16())
    yc = y.cpu().float()
    assert torch.isinf(yc[16:19]).all() and bool(torch.isfinite(yc[15]))  # the bf16 maximum stays, halfway past it is inf
    b = torch.arange(-2 ** 15, 2 ** 15, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    f = torch.empty(b.numel(), device=DEV)
    ops.cast_bf16_to_f32(b.to(DEV), f)
    _bits_equal_or_both_nan(f.cpu(), b.float())


# ---------------------------------------------------------------------------------------------------------------
# loss-head glue (csrc/heads.cu, csrc/masking.cu)
# ---------------------------------------------------------------------------------------------------------------
def test_validity_and_mlm_index(ops):
    """merlot_ids_valid (ids != 0, model/modeling.py:148,363), merlot_joint_valid (viz part all valid :106-107, lang part
    ids != 0 :148) and merlot_mlm_index (modeling.py:533-536: rows of the masked positions in joint-sequence coordinates and
    the input ids there as targets), bit for bit."""
    g = torch.Generator().manual_seed(3)
    for B, P, L, k in ((2, 13, 64, 12), (3, 0, 40, 8), (1, 130, 1, 1), (8, 50, 256, 51)):
        ids = torch.randint(0, 50, (B, L), generator=g, dtype=torch.int32)
        ids[:, -1] = 0
        v = torch.full((B * L,), 7, dtype=torch.uint8, device=DEV)
        ops.ids_valid(ids.to(DEV), v)
        assert torch.equal(v.cpu(), (ids != 0).to(torch.uint8).reshape(-1))
        jv = torch.full((B * (P + L),), 7, dtype=torch.uint8, device=DEV)
        ops.joint_valid(ids.to(DEV), jv, B, P, L)
        want = torch.cat([torch.ones(B, P, dtype=torch.bool), ids != 0], 1).to(torch.uint8).reshape(-1)
        assert torch.equal(jv.cpu(), want)
        masked_idx = torch.stack([torch.randperm(L, generator=g)[:k] for _ in range(B)]).to(torch.int32)
        masked_idx[0, 0] = L - 1
        rows = torch.full((B * k,), -1, dtype=torch.int32, device=DEV)
        targets = torch.full((B * k,), -1, dtype=torch.int32, device=DEV)
        ops.mlm_index(ids.to(DEV), masked_idx.to(DEV), rows, targets, B, L, k, P)
        idx = (masked_idx.long() + torch.arange(B)[:, None] * L).reshape(-1)  # :534 (the oracle's mask_loss)
        assert torch.equal(targets.cpu().long(), ids.reshape(-1)[idx].long())  # :536
        assert torch.equal(rows.cpu().long(), (masked_idx.long() + torch.arange(B)[:, None] * (P + L) + P).reshape(-1))


@pytest.mark.parametrize("B,n", [(1, 1), (3, 4), (2, 8), (5, 7)])
def test_temporal_labels_and_weights(ops, B, n):
    """allpairs_temporal_labels (model/modeling.py:598-620, the oracle's method) and the pair weights of :635,649-652 for
    shuffled_idx_img values straddling the 64 boundary (63 is easy, 64 is not), bit for bit against
    float32(not easy) * float32(0.99) + float32(0.01)."""
    g = torch.Generator().manual_seed(B * 10 + n)
    vid = torch.randint(0, 3, (B, n), generator=g, dtype=torch.int32)
    shuf = torch.tensor([62, 63, 64, 65])[torch.randint(0, 4, (B, n), generator=g)].to(torch.int32)
    labels = torch.full((B * n * n,), -1, dtype=torch.int32, device=DEV)
    w = torch.full((B * n * n,), float("nan"), device=DEV)
    ops.temporal_labels(vid.to(DEV), shuf.to(DEV), labels, w, B, n)
    want = O.MerlotOracle.allpairs_temporal_labels(types.SimpleNamespace(num_chunks_in_group=n, B=B), vid)
    assert torch.equal(labels.cpu(), want.to(torch.int32))
    easy = (shuf < 64).numpy()
    not_easy = ~(easy[:, :, None] & easy[:, None, :])
    w_ref = not_easy.astype(np.float32) * np.float32(0.99) + np.float32(0.01)
    assert np.array_equal(w.cpu().numpy(), w_ref.reshape(-1))


# weighted_loss: sums of up to 5000 fp32 products then one division.  Measured relative error: loss 1.6e-7, accuracy 1.1e-7,
# coeff (Frobenius) 5.9e-8
WLOSS_BAR = 1e-5


@pytest.mark.parametrize("R", [1, 255, 256, 257, 5000])
@pytest.mark.parametrize("source", ["w", "nz_labels", "none", "zero_w"])
@pytest.mark.parametrize("denom_mode", [0, 1])
def test_weighted_loss(ops, R, source, denom_mode):
    """out2 = {sum(l*w)/denom, sum(correct*w)/(sum w + 1e-5)}, coeff[r] = scale*w[r]/denom with denom = R (reduce_mean,
    modeling.py:523,655) or sum w + 1e-5 (:543); w = the weights, labels != 0, or 1.  `correct` and `coeff` are also passed as
    null (the contrastive head).  All-zero weights: loss and accuracy 0, not NaN, in mode 1."""
    g = torch.Generator().manual_seed(R * 8 + denom_mode)
    l = torch.rand(R, generator=g) * 5
    corr = (torch.rand(R, generator=g) < 0.5).float()
    w = labels = None
    if source == "w":
        w = torch.where(torch.rand(R, generator=g) < 0.3, torch.tensor(0.01), torch.tensor(1.0))
        wr = w.double()
    elif source == "zero_w":
        w = torch.zeros(R)
        wr = w.double()
    elif source == "nz_labels":
        labels = torch.randint(0, 3, (R,), generator=g, dtype=torch.int32)
        wr = (labels != 0).double()
    else:
        wr = torch.ones(R, dtype=F64)
    scale = 0.125
    denom = float(R) if denom_mode == 0 else wr.sum() + 1e-5
    loss_ref = (l.double() * wr).sum() / denom
    acc_ref = (corr.double() * wr).sum() / (wr.sum() + 1e-5)
    coeff_ref = scale * wr / denom
    for with_opt in (True, False):
        out2 = torch.full((2,), float("nan"), device=DEV)
        coeff = torch.full((R,), float("nan"), device=DEV) if with_opt else None
        ops.weighted_loss(l.to(DEV), corr.to(DEV) if with_opt else None, None if w is None else w.to(DEV),
                          None if labels is None else labels.to(DEV), denom_mode, scale, out2, coeff)
        o = out2.cpu().double()
        assert abs(o[0] - loss_ref) <= WLOSS_BAR * abs(loss_ref), (float(o[0]), float(loss_ref))
        if with_opt:
            assert abs(o[1] - acc_ref) <= WLOSS_BAR * abs(acc_ref), (float(o[1]), float(acc_ref))
            assert rel(coeff, coeff_ref) <= WLOSS_BAR
        else:
            assert float(o[1]) == 0.0
    if source == "zero_w":
        assert float(o[0]) == 0.0 and torch.isfinite(o).all()


@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("M,N,K,layout,beta", [(32, 32, 128, "fwd", 0.0), (7, 40, 5, "dx", 1.0), (40, 7, 77, "dy", 0.5),
                                                (33, 65, 31, "fwd", 0.5), (2048, 2048, 8, "fwd", 1.0), (1, 1, 1, "dx", 0.0)])
def test_small_gemm(ops, M, N, K, layout, beta, regime):
    """merlot_small_gemm_f32: C = alpha * A B^T + beta * C with the element strides the contrastive head uses (modeling.py
    contrastive_loss / _contrastive_bwd): fwd A[m,k] = x[m*K + k], B[n,k] = y[n*K + k]; dx B read transposed (y[k*N + n]);
    dy both transposed.  K below, at and past the 32-lane loop, C pre-filled (NaN when beta = 0: C must not be read), ldc
    larger than N, and M*N = 4 Mi, the largest output accepted.  Random regime, measured: 7.8e-8."""
    g = torch.Generator().manual_seed(M * N + K)
    a = inputs((M * K,), g, regime)
    b = inputs((N * K,), g, regime)
    if layout == "fwd":
        A, B, sa, sb = a.view(M, K), b.view(N, K), (K, 1), (K, 1)
    elif layout == "dx":
        A, B, sa, sb = a.view(M, K), b.view(K, N).t(), (K, 1), (1, N)
    else:
        A, B, sa, sb = a.view(K, M).t(), b.view(K, N).t(), (1, M), (1, N)
    alpha = 0.5 if regime == "exact" else 1.0 / 0.05
    c0 = torch.full((M, N + 3), float("nan")) if beta == 0.0 else inputs((M, N + 3), g, regime)
    Cm = c0.to(DEV)
    ops.small_gemm(a.to(DEV), sa[0], sa[1], b.to(DEV), sb[0], sb[1], Cm[:, :N], M, N, K, alpha=alpha, beta=beta)
    ref = alpha * (A.double() @ B.double().t()) + (beta * c0[:, :N].double() if beta != 0.0 else 0.0)
    check(Cm[:, :N], ref, regime, SUM_BAR, "C")
    pad = Cm.cpu()[:, N:]  # the columns past N of every row are not written
    assert torch.equal(torch.isnan(pad), torch.isnan(c0[:, N:])) and torch.equal(pad.nan_to_num(), c0[:, N:].nan_to_num())


def test_axpby(ops):
    """y = a*x + b*y (the contrastive and temporal loss totals and gradient sums); b = 0 must not read y (NaN there stays out).
    Dyadic values and scales: bit-exact."""
    g = torch.Generator().manual_seed(9)
    for n, a, b in ((1, 0.5, 0.0), (1000, 1.0, 1.0), (4097, 0.125, 0.5), (33, -2.0, 1.0)):
        x = exact((n,), g)
        y0 = torch.full((n,), float("nan")) if b == 0.0 else exact((n,), g)
        y = y0.to(DEV)
        ops.axpby(x.to(DEV), y, a, b)
        ref = a * x.double() + (b * y0.double() if b != 0.0 else 0.0)
        assert torch.equal(y.cpu().double(), ref)


@pytest.mark.parametrize("B,S,P", [(2, 200, 60), (3, 130, 0), (2, 150, 150), (1, 5, 2), (4, 300, 100)])
def test_attention_log_blocks(ops, B, S, P):
    """attention_log (model/modeling.py:186-203, the oracle's MerlotModel lines): the layer/head-mean map masked by validity on
    both sides, averaged over the batch and normalised, summed over the {viz, lang} x {viz, lang} blocks (`from`2`to`: keys
    are `from`, queries `to`).  The kernel gets the split column sums of that map (queries in the viz / lang piece, valid
    queries only, as K4 accumulates them) and the key validity.  B*S > 256 (the single block strides), P = 0 and P = S (one
    piece empty), padding keys and queries.  Measured rel error: 4.0e-8."""
    from merlot_b200._lib import lib
    g = torch.Generator().manual_seed(B * S + P)
    sap = torch.rand(B, S, S, generator=g, dtype=F64)  # head/layer-mean probabilities [b, query, key]
    valid = torch.rand(B, S, generator=g) < 0.8
    valid[:, 0] = True
    vf = valid.double()
    c_viz = (sap * vf[:, :, None])[:, :P].sum(1).float()   # K4 column sums, valid queries of each piece
    c_lang = (sap * vf[:, :, None])[:, P:].sum(1).float()
    m = sap * (vf[:, None] * vf[:, :, None])               # :192-193, then :194-195
    m = m.mean(0)
    m = m / m.sum()
    pieces = {"viz": (0, P), "lang": (P, S)}
    ref = {f"{fr}2{to}": m[pieces[to][0]:pieces[to][1], pieces[fr][0]:pieces[fr][1]].sum() for fr in pieces for to in pieces}
    ref = torch.stack([ref["lang2lang"], ref["lang2viz"], ref["viz2lang"], ref["viz2viz"]])
    out = torch.full((4,), float("nan"), device=DEV)
    vd = valid.to(torch.uint8).reshape(-1).to(DEV)
    cv, cl = c_viz.reshape(-1).to(DEV), c_lang.reshape(-1).to(DEV)
    lib().merlot_attention_log_blocks(cv.data_ptr(), cl.data_ptr(), vd.data_ptr(), B, S, P, out.data_ptr(), ops._stream())
    assert rel(out, ref) <= SUM_BAR
    assert float(out.cpu().sum()) == pytest.approx(1.0, abs=1e-6)
    if P == 0:
        assert float(out.cpu()[1:].abs().max()) == 0.0
    if P == S:
        assert float(out.cpu()[:3].abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------------------------
# GeLU: the accurate erff kernels of the heads and the fast erf of the GEMM epilogues, on every bf16 value in [-12, 12]
# ---------------------------------------------------------------------------------------------------------------
# A result passes if it is within one bf16 ulp of the bf16-rounded float64 reference, or within 5e-7 of the reference.
# Measured maxima of |got - ref| on an H100 80GB HBM3 (400 W): in the two tests' docstrings.
GELU_ABS_BAR = 5e-7


def _all_bf16_in(lo, hi):
    x = torch.arange(-2 ** 15, 2 ** 15, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    x = x[torch.isfinite(x) & (x >= lo) & (x <= hi)]
    return torch.unique(x)  # -0 and +0 collapse


def _gelu_refs(x):
    xr = x.double().requires_grad_(True)
    y = O.gelu(xr)
    (dy,) = torch.autograd.grad(y.sum(), xr)
    return y.detach(), dy


def _gelu_bar(got, ref, what):
    """Every element within one bf16 ulp of bf16(ref), or within GELU_ABS_BAR of ref."""
    got = got.detach().cpu().double()
    r16 = ref.float().bfloat16().double()
    ulp = 2.0 ** (torch.floor(torch.log2(r16.abs().clamp(min=2.0 ** -126))) - 7)
    err = (got - ref).abs()
    ok = ((got - r16).abs() <= ulp) | (err <= GELU_ABS_BAR)
    assert bool(ok.all()), (what, got[~ok][:5].tolist(), ref[~ok][:5].tolist())


def test_gelu_heads_every_bf16_input(ops):
    """merlot_gelu_f32 / merlot_gelu_bwd_f32 (erff; the contrastive / lm_head / temporal head GeLUs) against O.gelu and its
    autograd derivative in float64, with dy = 1 and a power-of-two dy.  Measured max |got - ref|: gelu 4.8e-7 (half an
    fp32 ulp of outputs in [8, 12]), gelu' 1.3e-7."""
    x = _all_bf16_in(-12.0, 12.0)
    x = torch.cat([x, torch.zeros((-x.numel()) % 8)])
    y_ref, d_ref = _gelu_refs(x)
    y = torch.empty_like(x, device=DEV)
    ops.gelu_f32(x.to(DEV), y)
    _gelu_bar(y, y_ref, "gelu_f32")
    for s in (1.0, 0.25):
        dx = torch.empty_like(x, device=DEV)
        ops.gelu_bwd_f32(torch.full_like(x, s).to(DEV), x.to(DEV), dx)
        _gelu_bar(dx, s * d_ref, f"gelu_bwd_f32 dy={s}")


def test_gelu_gemm_epilogue_every_bf16_input(ops):
    """The K1 epilogue's fast GeLU (Abramowitz-Stegun 7.1.26 with ex2 / rcp.approx, ptx.cuh normal_cdf_fast) on every bf16
    value in [-12, 12], fed through exact GEMMs: A = identity, B = the values, so the fp32 accumulator is exactly x.
      GELU (fp32 out): gelu(x); GELU + GELU_GRAD_OUT (bf16 dual out): gelu(x) and gelu'(x); MUL_DGELU (fp32 out): A @ B = 1 and
      aux = x, so the result is gelu'(x).
    Against O.gelu and its float64 autograd derivative.  Measured max |got - ref|: GELU 3.7e-7, MUL_DGELU 2.9e-7 (fp32 outputs);
    the bf16 outputs are within one bf16 ulp of bf16(ref) wherever |got - ref| > 5e-7.  Relative error of GELU on [-5, -3)
    (|gelu| <= 3.9e-3): 1.6e-3.  Below x = -5 the float64 restatement 1 + erf(x / sqrt 2) cancels itself (it is 0 for
    x < -8.3), so only the absolute bar is meaningful there."""
    x = _all_bf16_in(-12.0, 12.0)
    K = 128
    n_cols = -(-x.numel() // K)
    n_cols += (-n_cols) % 8
    xs = torch.zeros(n_cols * K)
    xs[:x.numel()] = x
    y_ref, d_ref = _gelu_refs(xs)
    eye = torch.eye(K).bfloat16().to(DEV)
    bmat = xs.view(n_cols, K).bfloat16().to(DEV)  # B[n, k] = x[n*K + k]  ->  C[m, n] = x[n*K + m]
    to_flat = lambda c: c.t().reshape(-1)  # noqa: E731
    y32 = ops.gemm(eye, bmat, gelu=True, out_dtype=torch.float32)
    _gelu_bar(to_flat(y32), y_ref, "GELU")
    gsave = torch.empty(K, n_cols, dtype=torch.bfloat16, device=DEV)
    yb = ops.gemm(eye, bmat, gelu=True, out_pre=gsave, gelu_grad_out=True)
    _gelu_bar(to_flat(yb), y_ref, "GELU dual")
    _gelu_bar(to_flat(gsave), d_ref, "GELU_GRAD_OUT")
    ones_a = torch.zeros(K, 64, dtype=torch.bfloat16)
    ones_a[:, 0] = 1
    ones_b = torch.zeros(n_cols, 64, dtype=torch.bfloat16)
    ones_b[:, 0] = 1
    aux = xs.view(n_cols, K).t().contiguous().bfloat16().to(DEV)  # aux[m, n] = x[n*K + m]
    dg = ops.gemm(ones_a.to(DEV), ones_b.to(DEV), dgelu_aux=aux, out_dtype=torch.float32)
    _gelu_bar(to_flat(dg), d_ref, "MUL_DGELU")
