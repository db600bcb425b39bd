"""The checks of tests/gemm_exact_oracle.py can fail: doctored K1 outputs (one element one bf16 ulp off, one 16 x 64 sub-tile
replaced, one 16-row warp slice missing one k-block, a GeLU value outside the bound in the tail) are each caught, where the
relative-Frobenius bars of test_gpu_kernels.py (1e-4 fp32, 6e-3 bf16) accept some of them.  Also: the exactness bound of the
integer operands at the largest K the GPU tests use, and the constant of the GeLU bound from the CPU restatement of the
fast GeLU over every bf16 input."""
import numpy as np
import pytest
import torch

from tests import gemm_exact_oracle as X
from tests import test_gpu_gemm_exact as G

FP32_BAR, BF16_BAR = 1e-4, 6e-3


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def small():
    """Integer operands of a 300 x 264 x 200 problem, its exact product and the bf16 output K1 should give."""
    a = X.int_operands((300, 200), 1)
    b = X.int_operands((264, 200), 2)
    acc = X.exact_product(a, b)
    return a, b, acc, X.epilogue_ref(acc)


def test_integer_bound_holds_for_the_largest_k():
    kmax = max(K for *_, K in G.MULTI_WAVE + G.SPLIT_SHAPES)
    assert kmax <= X.K_MAX
    assert X.partial_sum_bound(X.K_MAX) == 34048 < 2 ** 16
    # the split-K tests add integers of magnitude <= 64 already in the gradient
    assert X.partial_sum_bound(kmax) + 64 < 2 ** 16
    a = X.int_operands((4, X.K_MAX), 3)
    assert a.float().abs().max() <= 2 and torch.equal(a.float(), a.float().round())
    ones = torch.full((1, X.K_MAX), 2.0, dtype=torch.bfloat16)
    assert float(X.exact_product(ones, ones)) == X.partial_sum_bound(X.K_MAX)  # reached by the extreme operands


def test_one_ulp_off_is_caught(small):
    *_, want = small
    got = want.clone()
    got.view(torch.int16)[123, 45] += 1  # the next bf16 value away from zero
    assert X.bf16_ulps(got[123, 45], want[123, 45]) == 1
    with pytest.raises(AssertionError, match=r"1 of 79200 elements differ; first at \(123, 45\)"):
        X.exact_check(got, want)
    assert rel(got, want) < BF16_BAR


def test_replaced_sub_tile_is_caught(small):
    a, b, acc, want = small
    got = want.clone()
    got[16:32, 64:128] = X.epilogue_ref(X.exact_product(X.int_operands((16, 200), 9), b[64:128]))
    with pytest.raises(AssertionError, match="first at"):
        X.exact_check(got, want)


def test_missing_k_block_is_caught_where_frobenius_is_not():
    """One 16-row slice of one 128 x 256 tile of 8512 x 3072 x 768 without one of its 12 k-blocks: 3.6e-3 in relative
    Frobenius norm (bf16), under the 6e-3 bar, and thousands of wrong elements for the exact check and the bound."""
    M, N, K = 8512, 3072, 768
    g = torch.Generator().manual_seed(0)
    a = (torch.randn(M, K, generator=g) * 0.5).bfloat16()
    b = (torch.randn(N, K, generator=g) * 0.5).bfloat16()
    af, bf = a.float(), b.float()
    ref = af @ bf.t()
    rows, cols, ks = slice(4096 + 48, 4096 + 64), slice(1024, 1280), slice(320, 384)
    got = ref.clone()
    got[rows, cols] -= af[rows, ks] @ bf[cols, ks].t()
    e = rel(got.bfloat16(), ref)
    assert 2e-3 < e < BF16_BAR, e  # the bf16 bar accepts it
    # the per-element bound rejects it (on the slice, where the doctoring is, to keep the test fast)
    absprod = af[rows].abs().double() @ bf.abs().double().t()
    with pytest.raises(AssertionError, match="x the bound"):
        X.elementwise_bound_check(got[rows].bfloat16(), af[rows].double() @ bf.double().t(), absprod, K)
    # and on integer operands, the exact check
    ai, bi = X.int_operands((128, K), 5), X.int_operands((256, K), 6)
    acc = X.exact_product(ai, bi)
    doctored = acc.clone()
    doctored[48:64] -= ai[48:64, 320:384].double() @ bi[:, 320:384].double().t()
    with pytest.raises(AssertionError, match="elements differ"):
        X.exact_check(doctored.float(), acc.float())


def test_one_element_off_passes_the_fp32_frobenius_bar(small):
    *_, acc, _ = small
    got = acc.float().clone()
    got.view(torch.int32)[7, 7] += 1  # one fp32 ulp
    assert rel(got, acc) < FP32_BAR
    with pytest.raises(AssertionError):
        X.exact_check(got, acc.float())


def test_elementwise_bound_accepts_rounding_and_names_the_worst_element():
    g = torch.Generator().manual_seed(1)
    a = (torch.randn(64, 96, generator=g) * 0.3).bfloat16()
    b = (torch.randn(40, 96, generator=g) * 0.1).bfloat16()
    ref = X.exact_product(a, b)
    absprod = a.double().abs() @ b.double().abs().t()
    X.elementwise_bound_check(ref.float(), ref, absprod, 96, out_bf16=False)
    X.elementwise_bound_check(ref.bfloat16(), ref, absprod, 96)
    got = ref.bfloat16()
    got[5, 6] = got[5, 6] * 1.02
    with pytest.raises(AssertionError, match=r"element \(5, 6\)"):
        X.elementwise_bound_check(got, ref, absprod, 96)


def test_bf16_ulps():
    v = torch.tensor([1.0, 1.0078125, -0.0, 0.0, -1.0, 2.0 ** -133, -(2.0 ** -133)]).bfloat16()
    assert X.bf16_ulps(v[0], v[1]) == 1
    assert X.bf16_ulps(v[2], v[3]) == 0
    assert X.bf16_ulps(v[5], v[6]) == 2
    assert X.ulp_bf16(1.0) == 2.0 ** -7 and X.ulp_bf16(1.99) == 2.0 ** -7 and X.ulp_bf16(0.0) == 2.0 ** -133
    assert X.ulp_f32(1.0) == 2.0 ** -23


def test_epilogue_replay_rounds_once_per_step():
    acc = torch.tensor([[257.0, 3.0]], dtype=torch.float64)
    assert X.epilogue_ref(acc).tolist() == [[256.0, 3.0]]  # bf16 RNE of 257 is 256
    assert X.epilogue_ref(acc, alpha=0.5, bias=torch.tensor([0.5, 0.25])).float().tolist() == [[129.0, 1.75]]
    keep = torch.tensor([[True, False]])
    assert X.epilogue_ref(acc, keep=keep, scale=np.float32(2.0), resid=torch.tensor([[1.0, 1.0]]).bfloat16()).tolist() \
        == [[516.0, 1.0]]


# ---------------------------------------------------------------------------------------------------------------------
# GeLU
# ---------------------------------------------------------------------------------------------------------------------
def _finite_bf16():
    x = X.all_bf16().float().numpy()
    return x[np.isfinite(x)]


@pytest.mark.parametrize("kind", ["phi", "gelu", "dgelu"])
def test_fast_gelu_restatement_meets_the_bound(kind):
    """GELU_ABS comes from here: the restated fast GeLU's absolute error over every finite bf16 input, before and after
    rounding to bf16."""
    x = _finite_bf16()
    got = X.gelu_fast_np(x, kind)
    e = X.gelu_errors(x, got, kind, out="f32")
    assert e["max_abs_per_x"] <= 2.4e-7 < X.GELU_ABS
    X.gelu_bound_check(x, got, kind, out="f32")
    gb = torch.from_numpy(got).bfloat16()
    X.gelu_bound_check(x, gb, kind)
    eb = X.gelu_errors(x, gb, kind)
    assert eb["max_ulps_mid"] <= 0.55
    if kind == "gelu":
        assert eb["max_ulps_tail"] > 8  # the tail: many bf16 ulps, few absolute units


def test_gelu_outside_the_bound_is_caught():
    x = _finite_bf16()
    tail = x[(x > -12) & (x < -4)]
    got = torch.from_numpy(X.gelu_fast_np(tail, "gelu")).bfloat16().float().numpy()
    X.gelu_bound_check(tail, got, "gelu")
    i = len(tail) // 2
    bad = got.copy()
    bad[i] += 4 * X.GELU_ABS * abs(float(tail[i]))
    with pytest.raises(AssertionError, match="x the bound"):
        X.gelu_bound_check(tail, bad, "gelu")
    near0 = x[np.abs(x) < 1]
    got = torch.from_numpy(X.gelu_fast_np(near0, "dgelu")).bfloat16().float().numpy()
    got[3] = X.epilogue_ref(torch.tensor(got[3:4], dtype=torch.float64) * 1.02).float().numpy()[0]
    with pytest.raises(AssertionError):
        X.gelu_bound_check(near0, got, "dgelu")
