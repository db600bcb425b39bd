"""merlot_set_sm_reserve on one GPU: the grids the data-parallel step runs its ViT backward with (persistent K1 grids of
SMs - reserve CTAs, the split-K count derived from them, the fused LayerNorm backward's grid), compared with reserve 0 and
with float64.  A reserve of SMs - 9 leaves 9 K1 CTAs, each of which then walks tens of tiles: the producer's ring phase, the
fast epilogue's staging parity and its side-input prefetch carry over from tile to tile (pytest -m gpu)."""
import contextlib

import pytest
import torch

from tests import test_gpu_stack as TS
from tests.test_gpu_gemm_epilogue import SHAPES, _inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-300)).item()


def lib():
    from merlot_b200 import _lib
    return _lib.lib()


@contextlib.contextmanager
def sm_reserve(n):
    """The process-wide reserve set to n for the block, and always back to 0 after it."""
    lib().merlot_set_sm_reserve(n)
    try:
        yield
    finally:
        lib().merlot_set_sm_reserve(0)


def _reserves():
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    return [24, sms - 9]  # SMs - 9: the largest reserve num_sms() honours


@pytest.fixture(params=_reserves(), ids=lambda n: f"reserve{n}")
def reserve(request):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib().merlot_set_sm_reserve(0)
    yield request.param
    lib().merlot_set_sm_reserve(0)


@pytest.fixture(scope="module")
def ops():
    from merlot_b200 import ops as o
    return o


def _k1_outputs(ops, M, N, K, bn):
    """Every K1 epilogue kind at tile width bn: {kind: bf16 outputs}."""
    a, w, wt, bias, aux = _inputs(M, N, K, M * 7 + N + bn)
    kw = dict(block_n=bn)
    out = {"plain": [ops.gemm(a, w, b_mn_major=True, **kw)],
           "bias": [ops.gemm(a, w, b_mn_major=True, bias=bias, **kw)],
           "resid": [ops.gemm(a, w, b_mn_major=True, bias=bias, resid=aux, **kw)],
           "dropout": [ops.gemm(a, w, b_mn_major=True, bias=bias, resid=aux, dropout_p=0.1, dropout_seed=2 ** 35 + 9,
                                dropout_site=77, **kw)],
           "mul_aux_mn": [ops.gemm(a, w, b_mn_major=True, mul_aux=aux, **kw)],
           "mul_aux_k": [ops.gemm(a, wt, mul_aux=aux, **kw)],
           "mul_dgelu": [ops.gemm(a, wt, dgelu_aux=aux, **kw)],
           "generic_alpha": [ops.gemm(a, w, b_mn_major=True, bias=bias, alpha=0.37, generic_epilogue=True, **kw)]}
    for grad_out in (False, True):
        pre = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        act = ops.gemm(a, w, b_mn_major=True, bias=bias, gelu=True, out_pre=pre, gelu_grad_out=grad_out, **kw)
        out[f"gelu2_grad_out{int(grad_out)}"] = [pre, act]
    return out


@pytest.mark.parametrize("bn", [128, 192, 256])
@pytest.mark.parametrize("M,N,K", SHAPES + [(8512, 3072, 768)])
def test_k1_bitwise_under_reserve(ops, reserve, M, N, K, bn):
    """A tile's arithmetic does not depend on which CTA runs it: every bf16 output at a pinned tile width is bitwise the
    reserve-0 one."""
    want = _k1_outputs(ops, M, N, K, bn)
    with sm_reserve(reserve):
        got = _k1_outputs(ops, M, N, K, bn)
    for kind in want:
        for g, w in zip(got[kind], want[kind]):
            assert torch.equal(g, w), kind


@pytest.mark.parametrize("M,N,K", [(768, 768, 8512), (768, 3072, 8512), (3072, 768, 3168), (200, 264, 520), (768, 2304, 2128)])
def test_k1_split_k_wgrad_and_automatic_width_under_reserve(ops, reserve, M, N, K):
    """The split count of an ATOMIC wgrad and the automatic tile width follow the grid: compared with float64 (into a
    gradient that already holds a value), at the bars of test_gpu_gemm_epilogue.py / the bf16 GEMMs."""
    g = torch.Generator().manual_seed(M + N + K)
    x = (torch.randn(K, M, generator=g) * 0.3).bfloat16().to(DEV)
    dy = (torch.randn(K, N, generator=g) * 0.1).bfloat16().to(DEV)
    init = torch.randn(M, N, generator=g).to(DEV)
    ref = init.double() + x.double().t() @ dy.double()
    with sm_reserve(reserve):
        dw = init.clone()
        ops.gemm(x, dy, a_mn_major=True, b_mn_major=True, out=dw, atomic=True, M=M, N=N, K=K)
        y = ops.gemm(x.t().contiguous(), dy.t().contiguous())  # [M, N] bf16, automatic block_n
    assert rel(dw, ref) < 1e-5
    assert rel(y, x.double().t() @ dy.double()) < 6e-3


@pytest.mark.parametrize("rows,H", [(8512, 768), (20000, 256), (5000, 1024), (1777, 320), (3, 512)])
def test_layernorm_bwd_fused_under_reserve(ops, reserve, rows, H):
    """dx and the dropout-masked dmask bitwise; dgamma, dbeta and the bias gradient to fp32 reassociation."""
    g = torch.Generator().manual_seed(rows + H)
    x = (torch.randn(rows, H, generator=g) * 2 + 0.5).bfloat16().to(DEV)
    gam = torch.randn(H, generator=g).to(DEV)
    dy = torch.randn(rows, H, generator=g).bfloat16().to(DEV)
    dres = torch.randn(rows, H, generator=g).bfloat16().to(DEV)
    mu = x.float().mean(-1)
    rs = torch.rsqrt(x.float().var(-1, unbiased=False) + 1e-5)

    def run():
        dx, dmask = torch.empty_like(dy), torch.empty_like(dy)
        acc = [torch.ones(H, device=DEV) for _ in range(3)]
        ops.layernorm_bwd_fused(dy, x, mu, rs, gam, dx, acc[0], acc[1], dres=dres, dmask=dmask, dbias=acc[2],
                                dropout=(0.1, 2 ** 40 + 3, 5))
        return dx, dmask, acc
    dx0, dm0, acc0 = run()
    with sm_reserve(reserve):
        dx1, dm1, acc1 = run()
    assert torch.equal(dx1, dx0) and torch.equal(dm1, dm0)
    for a, b in zip(acc1, acc0):
        assert rel(a - 1, b - 1) < 1e-5


@pytest.mark.parametrize("name", ["tiny_odd_rows", "vit_shape", "atomic_dq", "widest"])
def test_stack_under_reserve(reserve, name):
    """y bitwise under the reserve; dh_in bitwise where dQ has no atomics (S <= 512).  The backward switches the reserve on
    after its first layer group, as the data-parallel step does, and its gradients meet the float64 reference's bars."""
    case = TS.CASES[name]
    inp = TS.make_inputs(case, seed=len(name))
    ref = TS.reference(case, inp)
    scale = [{k: float(v.std()) + 1e-6 for k, v in g.items()} for g in ref["grads"]]
    scale[-1].update(d_final_gamma=float(ref["d_final_gamma"].std()), d_final_beta=float(ref["d_final_beta"].std()))
    st = TS.Stack(case, inp, scale)
    base = st.run(backward=False)
    L = case["layers"]
    with sm_reserve(reserve):
        fwd = st.run(backward=False)
    with sm_reserve(0):
        got = st.run(groups=[(l, l + 1) for l in reversed(range(L))], on_group=lambda k: lib().merlot_set_sm_reserve(reserve))
    plain = st.run()
    assert torch.equal(fwd["y"], base["y"]) and torch.equal(got["y"], base["y"])
    if lib().merlot_attention_bwd_dq_parts(case["S"]) > 0:
        assert torch.equal(got["dh_in"], plain["dh_in"])
    e = TS.errors(got, ref)
    assert not TS.over_bar(e), TS.over_bar(e)


def _model_grads_under_reserve(cfg, n):
    """One pretraining step's forward, then two backwards of it: a plain backward() and one in the data-parallel order
    (non-ViT gradients, then the reserve, then the ViT layer groups and the stem).  Returns both gradient arenas and the
    mask of the arena that holds the hybrid stem's parameters."""
    from merlot_b200.modeling import MerlotModel
    from oracle import merlot_oracle as O
    from tests.test_gpu_model import build, synth
    image, ids, shuf, vid = synth(cfg, 2, 4, 16, 64, 96, 0)
    params, store, _ = build(cfg)
    draws = O.make_mask_draws(4, 32, 6, cfg["vocab_size"], seed=5)
    groups, _ = store.vit_buckets(4)
    m = MerlotModel(cfg, is_training=True, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                    shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, save_for_backward=True,
                    dropout_seed=2 ** 32 + 5)
    m.mask_loss(), m.contrastive_loss(), m.temporal_loss(shuf.to(DEV), vid.to(DEV))
    gs = []
    for dp in (False, True):
        store.g.zero_()
        if dp:
            with sm_reserve(0):
                m.backward(on_non_vit_grads_ready=lambda: lib().merlot_set_sm_reserve(n), vit_layer_groups=groups)
        else:
            m.backward()
        gs.append(store.g.clone())
    store.g.zero_()
    stem = torch.zeros_like(gs[0], dtype=torch.bool)
    for e in store.entries.values():
        if "/resnet50lite/" in e.name:
            stem[e.offset:e.offset + e.padded] = True
    return gs[0], gs[1], stem


# The hybrid stem's own parameter gradients are not bitwise repeatable: merlot_group_norm_bwd reduces its per-(sample, group)
# sums with fp32 atomicAdd (csrc/stem.cu), so from one call to the next a few elements of its bf16 dx round the other way
# (104 of 786432 at 8 x 32 x 48 x 64, 32 groups) and the convolutions and GroupNorms below carry that on.  Two plain
# backward() passes of one forward differ by 6.0e-3 over the stem's part of the gradient arena, by 1.1e-2 on single
# GroupNorm parameters; the data-parallel order under the reserve by 7.1e-3 (reserve 24) and 6.9e-3 (reserve 123).  Everything
# outside the stem agrees to 2.6e-8 (both models).  Measured on an H100 80GB HBM3, 700 W power limit.
STEM_BAR = 2e-2
NON_STEM_BAR = 1e-6


@pytest.mark.parametrize("stem", [False, True], ids=["plain_vit", "hybrid_stem"])
def test_model_backward_in_data_parallel_order_under_reserve(tiny_cfg, reserve, stem):
    """backward_and_apply's data-parallel ordering on one GPU: the ViT backward, the hybrid stem's included, enqueued under
    the reserve gives the gradients of a plain backward() of the same forward: within 1e-3 over the whole gradient arena,
    and within the bars above outside and inside the stem."""
    cfg = dict(tiny_cfg, num_vision_transformer_hidden_layers=4, vit_hidden_dropout_prob=0.2)
    if stem:
        cfg = dict(cfg, resnet_layers=[1, 2, 1], hidden_dropout_prob=0.0, vit_hidden_dropout_prob=0.0)
    plain, dp, in_stem = _model_grads_under_reserve(cfg, reserve)
    assert torch.isfinite(dp).all() and float(dp.abs().max()) > 0
    assert bool(in_stem.any()) == stem
    assert rel(dp, plain) < 1e-3
    assert rel(dp[~in_stem], plain[~in_stem]) < NON_STEM_BAR
    if stem:
        assert rel(dp[in_stem], plain[in_stem]) < STEM_BAR
