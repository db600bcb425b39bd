"""The attention backward for sequences of up to 512 tokens (pytest -m gpu): a dQ kernel and a dK/dV kernel, with no fp32 dQ
workspace and no atomics on dqkv.

- dqkv (dQ included) is bitwise identical across two runs on the same inputs.
- The workspace passed as dq_accum is neither read nor written: a sentinel pattern survives the call bit for bit.
- dsum still holds D = rowsum(dO o O) for every (b, h, query), within the fp32 rounding of a 64-term sum.

The shapes are the ones the model runs (language-only 128, ViT 266, joint encoder 396, VCR's joint 449) and the 512 edge,
with and without the token mask, the pair mask and attention-probability dropout."""

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [(128, 3, 2, False, False, 0.0), (266, 2, 12, False, False, 0.1), (396, 3, 2, True, False, 0.0),
         (449, 2, 2, True, True, 0.1), (512, 1, 2, True, False, 0.1), (257, 3, 1, True, True, 0.0)]


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def _inputs(B, S, heads, masked, seed):
    H = heads * 64
    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(B * S, 3 * H, generator=g) * 0.5).bfloat16().to(DEV)
    d_ctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16().to(DEV)
    valid = None
    if masked:
        lens = torch.randint(S // 2, S + 1, (B,), generator=g)
        valid = (torch.arange(S)[None, :] < lens[:, None]).to(torch.uint8).reshape(-1).contiguous().to(DEV)
    return qkv, d_ctx, valid


@pytest.mark.parametrize("S,B,heads,masked,pair,p", CASES)
def test_short_backward_is_reproducible_and_leaves_the_workspace_alone(ops, S, B, heads, masked, pair, p):
    from merlot_b200._lib import lib
    assert lib().merlot_attention_bwd_dq_parts(S) > 0  # the short-sequence kernels serve every case here
    H = heads * 64
    qkv, d_ctx, valid = _inputs(B, S, heads, masked, seed=S * 10 + B)
    pr = (S // 3, 40) if pair else (0, 0)
    drop = (p, 2 ** 33 + 7, 3)
    ctx, lse = ops.attention_fwd(qkv, B, S, heads, valid, pair=pr, dropout=drop)
    ws = ops.attention_bwd_workspace(B, S, heads, DEV)
    sentinel = (torch.arange(ws.numel(), dtype=torch.int64, device=DEV) * 40503 % (2 ** 31)).to(torch.int32).reshape(ws.shape)
    ws.view(torch.int32).copy_(sentinel)
    runs = []
    for _ in range(2):
        dsum = torch.full((B, heads, S), float("nan"), device=DEV)
        dqkv = torch.full((B * S, 3 * H), float("nan"), dtype=torch.bfloat16, device=DEV)
        ops.attention_bwd(qkv, ctx, d_ctx, lse, B, S, heads, valid, dqkv=dqkv, dq_accum=ws, dsum=dsum, pair=pr, dropout=drop)
        runs.append((dqkv.cpu(), dsum.cpu()))
    torch.cuda.synchronize()
    assert torch.equal(ws.view(torch.int32), sentinel), "the short path must not touch the dQ workspace"
    (a, da), (b, db) = runs
    assert torch.isfinite(a.float()).all(), "every element of dqkv is written"
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "dqkv (dQ included) must be bitwise reproducible"
    assert torch.equal(da, db)
    # D = rowsum(dO o O) over the 64 columns of each head: fp32 sums of 64 exact bf16 products
    o = ctx.double().cpu().reshape(B, S, heads, 64)
    go = d_ctx.double().cpu().reshape(B, S, heads, 64)
    want = (o * go).sum(-1).permute(0, 2, 1)
    bar = 64 * 2.0 ** -24 * (o * go).abs().sum(-1).permute(0, 2, 1) + 1e-30
    assert bool(((da.double() - want).abs() <= bar).all()), "dsum must hold D = rowsum(dO o O)"
