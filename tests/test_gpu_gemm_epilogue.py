"""K1's fast epilogue (math on the accumulator registers, TMA stores: the FFN2 dgrad x saved GeLU', the dual-output FFN1
forward, the split-K wgrads) against its generic epilogue, forced with generic_epilogue=True: bitwise equal for every bf16
output, equal up to fp32 reassociation for the reduce-add."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def _inputs(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * 0.3).bfloat16().to(DEV)
    w = (torch.randn(K, N, generator=g) * 0.1).bfloat16().to(DEV)  # MN-major (forward orientation)
    wt = w.t().contiguous()                                          # K-major (dgrad orientation)
    bias = torch.randn(N, generator=g).to(DEV)
    aux = torch.randn(M, N, generator=g).bfloat16().to(DEV)
    return a, w, wt, bias, aux


def _both(ops, *args, **kw):
    fast = ops.gemm(*args, **kw)
    slow = ops.gemm(*args, generic_epilogue=True, **kw)
    return fast, slow


SHAPES = [(300, 72, 200), (515, 264, 200), (300, 1000, 136), (3168, 768, 768), (515, 2304, 200), (8512, 3072, 256)]


@pytest.mark.parametrize("bn", [128, 192, 256])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_fast_epilogue_bitwise(ops, bn, M, N, K):
    a, w, wt, bias, aux = _inputs(M, N, K, M * 31 + N + bn)
    kw = dict(b_mn_major=True, block_n=bn)
    fast, slow = _both(ops, a, w, mul_aux=aux, **kw)
    assert torch.equal(fast, slow)
    fast, slow = _both(ops, a, wt, mul_aux=aux, block_n=bn)  # the dgrad orientation (both operands K-major)
    assert torch.equal(fast, slow)
    for grad_out in (False, True):
        pre_f = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        pre_s = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        act_f = ops.gemm(a, w, bias=bias, gelu=True, out_pre=pre_f, gelu_grad_out=grad_out, **kw)
        act_s = ops.gemm(a, w, bias=bias, gelu=True, out_pre=pre_s, gelu_grad_out=grad_out, generic_epilogue=True, **kw)
        assert torch.equal(act_f, act_s) and torch.equal(pre_f, pre_s), f"gelu grad_out={grad_out}"


@pytest.mark.parametrize("M,N,K", [(8512, 2304, 768), (8512, 768, 768), (8512, 3072, 768), (3168, 768, 3072)])
def test_fast_epilogue_step_shapes(ops, M, N, K):
    """The shapes the ViT and joint-encoder layers launch, with automatic tile width."""
    a, w, wt, bias, aux = _inputs(M, N, K, M + N + K)
    fast, slow = _both(ops, a, wt, mul_aux=aux)
    assert torch.equal(fast, slow)
    pre_f = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    pre_s = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    act_f = ops.gemm(a, w, b_mn_major=True, bias=bias, gelu=True, out_pre=pre_f, gelu_grad_out=True)
    act_s = ops.gemm(a, w, b_mn_major=True, bias=bias, gelu=True, out_pre=pre_s, gelu_grad_out=True, generic_epilogue=True)
    assert torch.equal(act_f, act_s) and torch.equal(pre_f, pre_s)


@pytest.mark.parametrize("bn", [128, 192, 256])
def test_fast_epilogue_clips_at_m_and_n(ops, bn):
    """Outputs that are views into wider, taller NaN-filled buffers: the stores write exactly [M, N), for both outputs of
    the dual-output kind."""
    M, N, K, ld = 300, 264, 200, 328
    a, w, wt, bias, aux = _inputs(M, N, K, bn)
    kw = dict(b_mn_major=True, block_n=bn, bias=bias)

    def sentinel():
        return torch.full((M + 40, ld), float("nan"), dtype=torch.bfloat16, device=DEV)

    def check(buf, ref):
        assert torch.equal(buf[:M, :N], ref)
        assert torch.isnan(buf[:, N:]).all() and torch.isnan(buf[M:, :]).all()

    buf = sentinel()
    ops.gemm(a, wt, out=buf[:M, :N], mul_aux=aux, block_n=bn)
    check(buf, ops.gemm(a, wt, mul_aux=aux, block_n=bn, generic_epilogue=True))
    pre_buf, act_buf = sentinel(), sentinel()
    ops.gemm(a, w, gelu=True, out_pre=pre_buf[:M, :N], out=act_buf[:M, :N], gelu_grad_out=True, **kw)
    pre_s = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    act_s = ops.gemm(a, w, gelu=True, out_pre=pre_s, gelu_grad_out=True, generic_epilogue=True, **kw)
    check(pre_buf, pre_s)
    check(act_buf, act_s)


@pytest.mark.parametrize("M,N,K", [(768, 768, 8512), (768, 3072, 8512), (3072, 768, 3168), (200, 264, 515)])
@pytest.mark.parametrize("splits", [0, 1])
def test_fast_epilogue_wgrad_reduce_add(ops, M, N, K, splits):
    """dW += x^T dy by TMA reduce-add, split-K on (automatic) and off, into a gradient that already holds a value."""
    g = torch.Generator().manual_seed(M + N + K)
    x = (torch.randn(K, M, generator=g) * 0.3).bfloat16().to(DEV)
    dy = (torch.randn(K, N, generator=g) * 0.1).bfloat16().to(DEV)
    init = torch.randn(M, N, generator=g).to(DEV)
    outs = []
    for generic in (False, True):
        dw = init.clone()
        ops.gemm(x, dy, a_mn_major=True, b_mn_major=True, out=dw, atomic=True, splits=splits, generic_epilogue=generic,
                 M=M, N=N, K=K)
        outs.append(dw)
    ref = init.double() + x.double().t() @ dy.double()
    for dw in outs:
        assert ((dw.double() - ref).norm() / ref.norm()).item() < 1e-5
    assert ((outs[0] - outs[1]).norm() / outs[1].norm()).item() < 1e-5
