"""GPU bring-up for K2/K3/K4 against a torch fp32 restatement of utils/transformer.py:98-127."""
import sys
import time

import torch

sys.path.insert(0, ".")
from merlot_b200 import ops  # noqa: E402


def ref_attention(qkv, B, S, heads, valid):
    H = qkv.shape[1] // 3
    d = H // heads
    x = qkv.float().reshape(B, S, 3, heads, d).permute(2, 0, 3, 1, 4)
    q, k, v = x[0].clone().requires_grad_(True), x[1].clone().requires_grad_(True), x[2].clone().requires_grad_(True)
    s = (q @ k.transpose(-1, -2)) * (1.0 / d ** 0.5)
    if valid is not None:
        vf = valid.reshape(B, S).float()
        m = (vf[:, None, :] * vf[:, :, None])[:, None]
        s = s * m - 1e10 * (1 - m)
    p = torch.softmax(s, -1)
    ctx = (p @ v).permute(0, 2, 1, 3).reshape(B * S, H)
    return q, k, v, p, ctx


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def run(B, S, heads, masked, seed):
    dev = "cuda"
    g = torch.Generator().manual_seed(seed)
    H = heads * 64
    qkv = (torch.randn(B * S, 3 * H, generator=g) * 1.0).bfloat16().to(dev)
    valid = None
    if masked:
        lens = torch.randint(max(1, S // 3), S + 1, (B,), generator=g)
        valid = (torch.arange(S)[None] < lens[:, None]).to(torch.uint8)
        if B > 1:
            valid[1, 5:9] = 0  # holes in the middle
        valid = valid.reshape(-1).contiguous().to(dev)
    ctx, lse = ops.attention_fwd(qkv, B, S, heads, valid)
    torch.cuda.synchronize()
    q, k, v, p, ctx_ref = ref_attention(qkv, B, S, heads, valid)
    e_ctx = rel(ctx, ctx_ref)
    d_ctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16().to(dev)
    if valid is not None:  # padding rows carry no gradient in the real model
        d_ctx = d_ctx * valid[:, None].to(d_ctx.dtype)
    dqkv = ops.attention_bwd(qkv, ctx, d_ctx, lse, B, S, heads, valid)
    torch.cuda.synchronize()
    ctx_ref.backward(d_ctx.float())
    ref_dqkv = torch.stack([q.grad, k.grad, v.grad], 0).permute(1, 3, 0, 2, 4).reshape(B * S, 3 * H)
    e_dq, e_dk, e_dv = (rel(dqkv[:, i * H:(i + 1) * H], ref_dqkv[:, i * H:(i + 1) * H]) for i in range(3))
    colsum = torch.zeros(B, S, device=dev)
    ops.attention_colsum(qkv, lse, colsum, B, S, heads, valid)
    torch.cuda.synchronize()
    cs_ref = p.detach().mean(1).sum(1)  # mean over heads, sum over queries -> [B, S]
    e_cs = rel(colsum, cs_ref)
    ok = max(e_ctx, e_dq, e_dk, e_dv) < 2e-2 and e_cs < 5e-3 and bool(torch.isfinite(dqkv.float()).all())
    print(f"{'OK  ' if ok else 'FAIL'} B={B} S={S} heads={heads} masked={masked}: ctx={e_ctx:.3e} dq={e_dq:.3e} "
          f"dk={e_dk:.3e} dv={e_dv:.3e} colsum={e_cs:.3e}", flush=True)
    return ok


def perf():
    dev = "cuda"
    for (B, S, heads) in [(32, 266, 12), (8, 396, 12), (8, 128, 12), (16, 3608, 12)]:
        H = heads * 64
        qkv = torch.randn(B * S, 3 * H, device=dev).bfloat16()
        ctx, lse = ops.attention_fwd(qkv, B, S, heads)
        d_ctx = torch.randn_like(ctx)
        dq_acc = ops.attention_bwd_workspace(B, S, heads, dev)
        dqkv = torch.empty_like(qkv)
        for name, fn, mult in (("fwd", lambda: ops.attention_fwd(qkv, B, S, heads, ctx=ctx, lse=lse), 1.0),
                               ("bwd", lambda: ops.attention_bwd(qkv, ctx, d_ctx, lse, B, S, heads, dqkv=dqkv,
                                                                 dq_accum=dq_acc), 2.5)):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            fl = 4.0 * B * heads * S * S * 64 * mult
            print(f"perf attn {name} B={B} S={S}: {ms * 1e3:.1f} us  {fl / ms / 1e9:.1f} TFLOP/s", flush=True)


if __name__ == "__main__":
    t0 = time.time()
    if len(sys.argv) > 1 and sys.argv[1] == "perf":
        perf()
        sys.exit(0)
    ok = True
    for i, (B, S, heads, masked) in enumerate([(1, 128, 1, False), (2, 128, 2, True), (2, 64, 2, False), (2, 266, 12, False),
                                               (2, 396, 12, True), (3, 93, 4, True), (1, 885, 2, True), (2, 256, 1, False)]):
        ok &= run(B, S, heads, masked, i)
    print(f"[attn] {'PASS' if ok else 'FAIL'} in {time.time() - t0:.1f}s", flush=True)
    sys.exit(0 if ok else 1)
