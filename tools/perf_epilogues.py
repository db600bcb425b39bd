"""Isolated timings of the ViT-size GEMMs WITH their real epilogues (bias / gelu dual / resid+dropout / dgelu)."""
import sys

import torch

sys.path.insert(0, ".")
from merlot_b200 import ops  # noqa: E402

dev = "cuda"
g = torch.Generator().manual_seed(0)
M, H, I = 8512, 768, 3072


def t(name, fn, flops):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    print(f"{name:46s} {ms * 1e3:7.1f} us  {flops / ms / 1e9:7.1f} TFLOP/s", flush=True)


x = (torch.randn(M, H, generator=g) * 0.5).bfloat16().to(dev)
xi = (torch.randn(M, I, generator=g) * 0.5).bfloat16().to(dev)
wqkv = (torch.randn(H, 3 * H, generator=g) * 0.05).bfloat16().to(dev)
wo = (torch.randn(H, H, generator=g) * 0.05).bfloat16().to(dev)
w1 = (torch.randn(H, I, generator=g) * 0.05).bfloat16().to(dev)
w2 = (torch.randn(I, H, generator=g) * 0.05).bfloat16().to(dev)
b3, b1, bh = torch.randn(3 * H).to(dev), torch.randn(I).to(dev), torch.randn(H).to(dev)
oqkv = torch.empty(M, 3 * H, dtype=torch.bfloat16, device=dev)
oh = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
oi = torch.empty(M, I, dtype=torch.bfloat16, device=dev)
oi2 = torch.empty(M, I, dtype=torch.bfloat16, device=dev)
t("QKV plain", lambda: ops.gemm(x, wqkv, b_mn_major=True, out=oqkv), 2.0 * M * 3 * H * H)
t("QKV +bias", lambda: ops.gemm(x, wqkv, b_mn_major=True, bias=b3, out=oqkv), 2.0 * M * 3 * H * H)
t("out-proj plain", lambda: ops.gemm(x, wo, b_mn_major=True, out=oh), 2.0 * M * H * H)
t("out-proj +bias+resid", lambda: ops.gemm(x, wo, b_mn_major=True, bias=bh, resid=x, out=oh), 2.0 * M * H * H)
t("out-proj +bias+resid+dropout", lambda: ops.gemm(x, wo, b_mn_major=True, bias=bh, resid=x, out=oh, dropout_p=0.1, dropout_seed=1), 2.0 * M * H * H)
t("FFN1 plain", lambda: ops.gemm(x, w1, b_mn_major=True, out=oi), 2.0 * M * I * H)
t("FFN1 +bias+gelu (pre+act)", lambda: ops.gemm(x, w1, b_mn_major=True, bias=b1, gelu=True, out_pre=oi2, out=oi), 2.0 * M * I * H)
t("FFN2 plain", lambda: ops.gemm(xi, w2, b_mn_major=True, out=oh), 2.0 * M * I * H)
t("FFN2 +bias+resid+dropout", lambda: ops.gemm(xi, w2, b_mn_major=True, bias=bh, resid=x, out=oh, dropout_p=0.1, dropout_seed=1), 2.0 * M * I * H)
t("FFN2-dgrad plain (N=3072,K=768)", lambda: ops.gemm(x, w2, out=oi, M=M, N=I, K=H), 2.0 * M * I * H)
t("FFN2-dgrad x gelu'(pre)", lambda: ops.gemm(x, w2, out=oi, dgelu_aux=oi2, M=M, N=I, K=H), 2.0 * M * I * H)
# the pair the training step launches: the forward saves gelu'(pre), the dgrad multiplies by it
t("FFN1 +bias+gelu (gelu'+act)", lambda: ops.gemm(x, w1, b_mn_major=True, bias=b1, gelu=True, out_pre=oi2, gelu_grad_out=True, out=oi), 2.0 * M * I * H)
t("FFN2-dgrad x saved gelu'", lambda: ops.gemm(x, w2, out=oi, mul_aux=oi2, M=M, N=I, K=H), 2.0 * M * I * H)
t("FFN1-dgrad plain (N=768,K=3072)", lambda: ops.gemm(xi, w1, out=oh, M=M, N=H, K=I), 2.0 * M * I * H)
t("QKV-dgrad plain (N=768,K=2304)", lambda: ops.gemm(oqkv, wqkv, out=oh, M=M, N=H, K=3 * H), 2.0 * M * 3 * H * H)

# tile widths on the N = 768 dgrads (K-major weights)
for name, A, W, K_ in (("FFN1-dgrad K=3072", xi, w1, I), ("QKV-dgrad K=2304", oqkv, wqkv, 3 * H), ("out-proj dgrad K=768", x, wo, H)):
    for bn in (128, 192, 256):
        t(f"{name} block_n={bn}", lambda: ops.gemm(A, W, out=oh, M=M, N=H, K=K_, block_n=bn), 2.0 * M * H * K_)
