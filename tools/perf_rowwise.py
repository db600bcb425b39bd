"""Isolated timings of the non-GEMM kernels at the ViT stack's size (8512 x 768): fused LN backward, LN forward, attention."""
import ctypes as C
import sys

import torch

sys.path.insert(0, ".")
from merlot_b200 import ops  # noqa: E402
from merlot_b200._lib import check, lib  # noqa: E402

dev = "cuda"
g = torch.Generator().manual_seed(0)
M, H = 8512, 768
L = lib()


def t(name, fn, bytes_=None, flops=None, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    extra = ""
    if bytes_:
        extra += f"  {bytes_ / ms / 1e6:7.0f} GB/s"
    if flops:
        extra += f"  {flops / ms / 1e9:7.1f} TFLOP/s"
    print(f"{name:44s} {ms * 1e3:8.1f} us{extra}", flush=True)


def bf(*shape):
    return (torch.randn(*shape, generator=g) * 0.5).bfloat16().to(dev)


x, dy, dres = bf(M, H), bf(M, H), bf(M, H)
dx, dmask, y = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
mean, rstd = torch.randn(M).to(dev), (torch.rand(M) + 0.5).to(dev)
gamma, beta = torch.randn(H).to(dev), torch.randn(H).to(dev)
dgam, dbet, dbias = torch.zeros(H, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)


def lnb(rows, drop, bias, res=True):
    check(L.merlot_layernorm_bwd_fused(dy.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(),
                                       dres.data_ptr() if res else None, dx.data_ptr(), dmask.data_ptr() if drop else None,
                                       dgam.data_ptr(), dbet.data_ptr(), dbias.data_ptr() if bias else None, None, rows, H,
                                       0.1 if drop else 0.0, 1, 3, st))


t("ln_bwd_fused  dres+dropout+bias  (8512)", lambda: lnb(M, True, True), bytes_=M * H * 2 * 5)
t("ln_bwd_fused  dres+bias          (8512)", lambda: lnb(M, False, True), bytes_=M * H * 2 * 4)
t("ln_bwd_fused  dres               (8512)", lambda: lnb(M, False, False), bytes_=M * H * 2 * 4)
t("ln_bwd_fused  dres+dropout+bias  (2176)", lambda: lnb(2176, True, True), bytes_=2176 * H * 2 * 5)
t("ln_bwd_fused  dres+dropout+bias  (640)", lambda: lnb(640, True, True), bytes_=640 * H * 2 * 5)
t("ln_fwd                           (8512)", lambda: ops.layernorm_fwd(x, y, gamma, beta, mean, rstd), bytes_=M * H * 2 * 2)
cs = torch.zeros(H, device=dev)
t("bias_grad colsum bf16            (8512)", lambda: ops.bias_grad(dy, cs), bytes_=M * H * 2)

# attention at the ViT shape: 32 frames x 266 tokens, 12 heads
B, S, heads = 32, 266, 12
qkv = bf(B * S, 3 * H)
ctx, lse = ops.attention_fwd(qkv, B, S, heads)
dctx = bf(B * S, H)
fl_fwd = 4.0 * B * heads * S * S * 64
t("attention_fwd  ViT (32x266, 12 heads)", lambda: ops.attention_fwd(qkv, B, S, heads), flops=fl_fwd)
t("attention_bwd  ViT (incl. dsum, finish)", lambda: ops.attention_bwd(qkv, ctx, dctx, lse, B, S, heads), flops=2.5 * fl_fwd)
