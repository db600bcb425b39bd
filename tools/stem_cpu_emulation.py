"""CPU check of the hybrid stem's ORCHESTRATION (forward tape + backward walk of merlot_b200/stem.py's HybridStem) without a GPU:
every K13 / K1 call is emulated in fp32 torch with the same formulas as the CUDA kernels, and the parameter gradients that come out
of HybridStem.backward are compared with torch autograd through the oracle's lite_resnet50.  Proves names, shapes, op
order, gradient routing and the closed-form backward formulas -- not the CUDA code itself."""
import sys

import torch

sys.path.insert(0, ".")
from merlot_b200 import ops  # noqa: E402
from merlot_b200.params import ParamStore  # noqa: E402
from merlot_b200.stem import HybridStem  # noqa: E402
from oracle import merlot_oracle as O  # noqa: E402

LAYERS = [1, 2, 1]
cfg = dict(use_bfloat16=True, hidden_size=128, vocab_size=1000, patch_size=16, spatial_pool_size=2, num_attention_heads=2,
           num_hidden_layers=1, num_vision_transformer_hidden_layers=1, num_lang_transformer_hidden_layers=1, intermediate_size=256,
           max_position_embeddings=64, num_chunks_in_group=2, resnet_layers=LAYERS)
st = ParamStore(cfg, device="cpu")
params = O.init_params(cfg, seed=0, perturb=0.05)
st.load_tf_dict(params)
st.g.zero_()


def ws_weights(w2d, kp):
    rows, cout = w2d.shape
    mean = w2d.mean(0, keepdim=True)
    var = ((w2d - mean) ** 2).mean(0, keepdim=True)
    out = torch.zeros(kp, cout)
    out[:rows] = (w2d - mean) * torch.rsqrt(var + 1e-5)
    return out


def im2col3x3(x, N, h, w, C, stride, out, sub_half=False):
    xx = x.reshape(N, h, w, C).float()
    if sub_half:
        xx = xx - 0.5
    ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
    xp = torch.nn.functional.pad(xx, (0, 0, 1, 1, 1, 1))
    out.zero_()
    for t in range(9):
        ky, kx = t // 3, t % 3
        out[:, t * C:(t + 1) * C] = xp[:, ky:ky + (ho - 1) * stride + 1:stride, kx:kx + (wo - 1) * stride + 1:stride, :].reshape(N * ho * wo, C)


def gemm(a, b, a_mn_major=False, b_mn_major=False, out=None, atomic=False, M=None, N=None, K=None, **kw):
    A = a.float().t() if a_mn_major else a.float()
    B = b.float() if b_mn_major else b.float().t()
    r = A @ B
    if atomic:
        out += r
    else:
        out.copy_(r)
    return out


def group_norm_fwd(x, gamma, beta, y, stats, N, HW, C, groups, eps, relu, shortcut):
    xr = x.reshape(N, HW, groups, C // groups).float()
    stats.zero_()
    sv = stats[:N * groups * 2].view(N, groups, 2)
    sv[..., 0] = xr.sum((1, 3))
    sv[..., 1] = (xr * xr).sum((1, 3))
    cnt = HW * (C // groups)
    mean = (sv[..., 0] / cnt)[:, None, :, None]
    var = (sv[..., 1] / cnt)[:, None, :, None] - mean * mean
    r = ((xr - mean) * torch.rsqrt(var + eps)).reshape(N * HW, C) * gamma + beta
    if shortcut is not None:
        r = r + shortcut.float()
    if relu:
        r = torch.relu(r)
    y.copy_(r)


def group_norm_bwd(dy, x, y, stats, gamma, dx, dsc, dgamma, dbeta, red, N, HW, C, groups=32, eps=1e-4, relu=True):
    cg = C // groups
    cnt = HW * cg
    sv = stats[:N * groups * 2].view(N, groups, 2)
    mean = (sv[..., 0] / cnt).repeat_interleave(cg, 1)[:, None, :]          # [N, 1, C]
    rstd = torch.rsqrt(sv[..., 1] / cnt - (sv[..., 0] / cnt) ** 2 + eps).repeat_interleave(cg, 1)[:, None, :]
    g = dy.reshape(N, HW, C).float()
    if relu:
        g = g * (y.reshape(N, HW, C) > 0)
    xh = (x.reshape(N, HW, C).float() - mean) * rstd
    gg = g * gamma
    S1 = gg.reshape(N, HW, groups, cg).sum((1, 3)) / cnt
    S2 = (gg * xh).reshape(N, HW, groups, cg).sum((1, 3)) / cnt
    dgamma += (g * xh).sum((0, 1))
    dbeta += g.sum((0, 1))
    dx.copy_((rstd * (gg - S1.repeat_interleave(cg, 1)[:, None, :] - xh * S2.repeat_interleave(cg, 1)[:, None, :])).reshape(N * HW, C))
    if dsc is not None:
        dsc.copy_(g.reshape(N * HW, C))


def avgpool2_same(x, N, h, w, C, y):
    y.copy_(O.avg_pool_same(x.reshape(N, h, w, C).float(), 2).reshape(y.shape))


def avgpool2_same_bwd(dy, N, h, w, C, dx):
    ho, wo = (h + 1) // 2, (w + 1) // 2
    d = dy.reshape(N, ho, wo, C).float()
    out = torch.zeros(N, h, w, C)
    for iy in range(h):
        for ix in range(w):
            oy, ox = iy // 2, ix // 2
            cnt = (2 if oy * 2 + 1 < h else 1) * (2 if ox * 2 + 1 < w else 1)
            out[:, iy, ix] = d[:, oy, ox] / cnt
    dx.copy_(out.reshape(dx.shape))


def col2im3x3(dcol, N, h, w, C, stride, dx):
    ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
    d = dcol.float().reshape(N, ho, wo, -1)
    out = torch.zeros(N, h, w, C)
    for iy in range(h):
        for ix in range(w):
            for ky in range(3):
                ty = iy - ky + 1
                if ty < 0 or ty % stride or ty // stride >= ho:
                    continue
                for kx in range(3):
                    tx = ix - kx + 1
                    if tx < 0 or tx % stride or tx // stride >= wo:
                        continue
                    t = ky * 3 + kx
                    out[:, iy, ix] += d[:, ty // stride, tx // stride, t * C:(t + 1) * C]
    dx.copy_(out.reshape(dx.shape))


def ws_weights_bwd(dws, w2d, dw2d):
    rows = w2d.shape[0]
    mean = w2d.mean(0, keepdim=True)
    rstd = torch.rsqrt(((w2d - mean) ** 2).mean(0, keepdim=True) + 1e-5)
    wh = (w2d - mean) * rstd
    g = dws[:rows]
    dw2d += rstd * (g - g.mean(0, keepdim=True) - wh * (g * wh).mean(0, keepdim=True))


def add_bf16(a, b, out):
    out.copy_(a.float() + b.float())


class WsPlan:  # ops.WsPlan: all conv kernels standardised up front, their gradients standardised back at the end
    def __init__(self, kernels, grads, device):
        self.names, self.k, self.g = list(kernels), kernels, grads
        self.wstd = {}
        self.dws = {n: torch.zeros((k.shape[0] + 7) // 8 * 8, k.shape[1]) for n, k in kernels.items()}
        self.key = tuple(k.data_ptr() for k in kernels.values())

    def standardise(self):
        for n, k in self.k.items():
            self.wstd[n] = ws_weights(k, (k.shape[0] + 7) // 8 * 8)

    def zero_grads(self):
        for d in self.dws.values():
            d.zero_()

    def backward(self):
        for n, k in self.k.items():
            ws_weights_bwd(self.dws[n], k, self.g[n])


ops.WsPlan = WsPlan
for name, fn in dict(ws_weights=ws_weights, im2col3x3=im2col3x3, gemm=gemm, group_norm_fwd=group_norm_fwd, group_norm_bwd=group_norm_bwd,
                     avgpool2_same=avgpool2_same, avgpool2_same_bwd=avgpool2_same_bwd, col2im3x3=col2im3x3, ws_weights_bwd=ws_weights_bwd,
                     add_bf16=add_bf16).items():
    setattr(ops, name, fn)


class Bufs:
    def __init__(self):
        self.d = {}

    def get(self, name, shape, dtype, zero=False):
        k = (name, tuple(shape), dtype)
        if k not in self.d:
            self.d[k] = torch.zeros(shape, dtype=torch.float32)
        elif zero:
            self.d[k].zero_()
        return self.d[k]


stem = HybridStem(st, Bufs(), LAYERS, save=True)
N = 2
gen = torch.Generator().manual_seed(1)
img = torch.rand(N, 64, 96, 3, generator=gen)
rc, h, w = stem.forward(img, N, 64, 96)
d_out = torch.randn(rc.shape, generator=gen) * 0.1
stem.backward(d_out.clone())

leaf = {k: v.clone().requires_grad_(True) for k, v in params.items() if "resnet50lite" in k}
ref = O.lite_resnet50(img - 0.5, leaf, "vision_backbone/vision_transformer/resnet50lite", LAYERS)
print("forward rel", ((rc - ref.reshape(rc.shape)).norm() / ref.norm()).item())
(ref.reshape(rc.shape) * d_out).sum().backward()
got = st.to_tf_dict("g")
worst = 0.0
for k, v in leaf.items():
    r = ((got[k] - v.grad).norm() / (v.grad.norm() + 1e-30)).item()
    worst = max(worst, r)
    if r > 1e-3:
        print("MISMATCH", k, r)
print(f"{len(leaf)} parameter gradients, worst rel err {worst:.2e}")
assert worst < 1e-3
