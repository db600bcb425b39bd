"""GPU parity of the hybrid ResNet-lite stem's FORWARD (SURVEY.md 8(f) next-row 1): the K13 kernels one by one against the
oracle's primitives, then lite_resnet50 and the whole MerlotModel forward with `resnet_layers` set (pytest -m gpu)."""
import pytest
import torch

from oracle import merlot_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def test_weight_standardisation(ops):  # utils/vision_transformer.py:56-60
    g = torch.Generator().manual_seed(0)
    for kh, cin, cout in ((3, 3, 32), (3, 64, 64), (1, 256, 128)):
        w = torch.randn(kh, kh, cin, cout, generator=g) * 0.2 + 0.05
        rows = kh * kh * cin
        kp = (rows + 7) // 8 * 8
        out = ops.ws_weights(w.reshape(rows, cout).to(DEV), kp).float().cpu()
        mean = w.mean((0, 1, 2), keepdim=True)
        ref = ((w - mean) * torch.rsqrt(((w - mean) ** 2).mean((0, 1, 2), keepdim=True) + 1e-5)).reshape(rows, cout)
        assert rel(out[:rows], ref) < 4e-3                       # one bf16 rounding of the standardised kernel
        assert torch.all(out[rows:] == 0) and out.shape == (kp, cout)


@pytest.mark.parametrize("N,h,w,cin,cout,stride", [(2, 9, 7, 32, 64, 1), (1, 16, 24, 64, 64, 1), (2, 32, 48, 3, 32, 2), (1, 9, 7, 3, 32, 2)])
def test_conv3x3_as_im2col_gemm(ops, N, h, w, cin, cout, stride):  # conv2d_fixed_padding :30-66 (SAME / fixed_padding + VALID)
    g = torch.Generator().manual_seed(h * w + cin)
    first = cin == 3  # the image conv subtracts 0.5 before the zero padding (:193)
    x = (torch.rand(N, h, w, cin, generator=g) if first else torch.randn(N, h, w, cin, generator=g)).bfloat16()
    k = (torch.randn(3, 3, cin, cout, generator=g) * 0.2).bfloat16()
    rows = 9 * cin
    kp = (rows + 7) // 8 * 8
    ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
    col = torch.empty(N * ho * wo, kp, dtype=torch.bfloat16, device=DEV)
    ops.im2col3x3(x.to(DEV), N, h, w, cin, stride, col, sub_half=first)
    wmat = torch.zeros(kp, cout, dtype=torch.bfloat16)
    wmat[:rows] = k.reshape(rows, cout)
    y = ops.gemm(col, wmat.to(DEV), b_mn_major=True, out_dtype=torch.float32)
    xin = (x.float() - 0.5).bfloat16().float() if first else x.float()
    ref = O.conv2d_fixed_padding(xin, k.float(), strides=stride, weight_standardization=False)
    assert tuple(ref.shape) == (N, ho, wo, cout)
    assert rel(y, ref.reshape(N * ho * wo, cout)) < 2e-3


@pytest.mark.parametrize("N,HW,C", [(2, 35, 32), (3, 63, 64), (2, 24, 256), (1, 7, 1024)])
def test_group_norm_relu_shortcut(ops, N, HW, C):  # batch_norm_relu :22-27, bottleneck tail :95-96
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(N, HW, 1, C, generator=g) * 1.5 + 0.3).bfloat16()
    sc = torch.randn(N, HW, 1, C, generator=g).bfloat16()
    p = {"s/gamma": torch.randn(C, generator=g) * 0.3 + 1.0, "s/beta": torch.randn(C, generator=g) * 0.2}
    ref = O.group_norm(x.float(), p, "s")
    stats = torch.empty(N * 64, device=DEV)
    for relu, short in ((True, None), (False, None), (True, sc)):
        y = torch.empty(N * HW, C, dtype=torch.bfloat16, device=DEV)
        ops.group_norm_fwd(x.reshape(N * HW, C).to(DEV), p["s/gamma"].to(DEV), p["s/beta"].to(DEV), y, stats, N, HW, C, 32, 1e-4, relu,
                           None if short is None else short.reshape(N * HW, C).to(DEV))
        r = ref if short is None else ref.bfloat16().float() + short.float()
        r = torch.relu(r) if relu else r
        assert rel(y, r.reshape(N * HW, C)) < 6e-3


def test_avgpool_same_ragged(ops):  # tf.nn.avg_pool2d SAME, odd sizes: bottom/right cells average fewer pixels
    g = torch.Generator().manual_seed(2)
    for N, h, w, C in ((2, 9, 7, 32), (1, 12, 22, 64)):
        x = torch.randn(N, h, w, C, generator=g).bfloat16()
        ho, wo = (h + 1) // 2, (w + 1) // 2
        y = torch.empty(N * ho * wo, C, dtype=torch.bfloat16, device=DEV)
        ops.avgpool2_same(x.to(DEV), N, h, w, C, y)
        assert rel(y, O.avg_pool_same(x.float(), 2).reshape(N * ho * wo, C)) < 4e-3


def _stem_cfg(tiny_cfg):
    return dict(tiny_cfg, resnet_layers=[1, 2, 1], hidden_dropout_prob=0.0)


def test_hybrid_stem_forward_and_model_forward(tiny_cfg):
    """lite_resnet50 + conv_postresnet_proj inside the MerlotModel forward (is_training=False) against the oracle on the same
    weights (the backward has its own tests below)."""
    from merlot_b200.modeling import MerlotModel
    from tests.test_gpu_model import build, synth
    cfg = _stem_cfg(tiny_cfg)
    batch, nc, Lc = 2, 2, 16
    image, ids, shuf, vid = synth(cfg, batch, nc, Lc, 64, 96, 0)
    params, store, _ = build(cfg)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=False,
                    shuffled_idx_img=shuf.to(DEV), params=store)
    N = batch * nc
    rc, hs, ws = m._stem.forward(image.bfloat16().to(DEV).contiguous(), N, 64, 96)
    scope = "vision_backbone/vision_transformer/resnet50lite"
    ref = O.lite_resnet50(image - 0.5, params, scope, cfg["resnet_layers"])
    ref16 = O.lite_resnet50(image - 0.5, params, scope, cfg["resnet_layers"], rnd=O.bf16_round)  # the reference's own dtype policy
    assert (hs, ws) == (4, 6) and tuple(ref.shape) == (N, 4, 6, 1024)
    om = O.MerlotOracle(cfg, params, image, ids, mask_input=False, shuffled_idx_img=shuf)
    r16, r32, r1632 = rel(rc, ref16.reshape(N * 24, 1024)), rel(rc, ref.reshape(N * 24, 1024)), rel(ref16, ref)
    rh = {name: rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name]) for name in ("viz", "lang")}
    print(f"stem parity: gpu~bf16-graph {r16:.3e}  gpu~fp32 {r32:.3e}  bf16-graph~fp32 {r1632:.3e}  hidden {rh}")
    # ~20 bf16 convs + GroupNorms over 4x6 maps deep: the bf16 graph itself sits 3.9e-2 from the fp32 restatement, and two bf16
    # evaluations that differ in summation order decorrelate at the same scale, so the bars are multiples of that noise floor
    assert r1632 < 6e-2 and r32 < 1.5 * r1632 + 1e-2, (r16, r32, r1632)
    assert r16 < 1.5 * r1632 + 1e-2, (r16, r32, r1632)
    for name in ("viz", "lang"):
        assert rh[name] < 1e-1, rh


# ---------------------------------------------------------------------------------------------------------------
# backward of the stem -- a test design that CAN fail (round-1 review).
#
# Why whole-graph bars were useless: a ResNet stem's parameter gradients at random init are sums of random-sign terms; the
# bf16 graph sits ~4e-2 from fp32 in the FORWARD, which flips ~3 % of the ReLU masks, and a 3 % flip of a random-sign sum is a
# ~25-30 % relative change of that sum -- on any map size (measured on CPU: the oracle in the reference's bf16 dtype policy vs
# its fp32 self: median 0.31 at 64x96, 128x192 and batch 8 alike).  So a comparison across DIFFERENT rounding points cannot
# tell a right gradient from a subtly wrong one.  The tests below compare at IDENTICAL rounding points instead:
#   (1) op level: each backward kernel vs autograd of the same op, ReLU masks taken from the kernel's own forward output;
#   (2) in situ: the real tape of lite_resnet50 at 128x192 (maps 64x96 .. 8x12): for EVERY op the GPU's dx / d_shortcut /
#       parameter gradient vs autograd of that op on the GPU's own saved input and the GPU's own incoming gradient, plus the
#       routing identity (an op's incoming gradient = sum of its consumers' dx);
#   (3) model level: the oracle is given the GPU's stem OUTPUT as a leaf: every non-stem gradient and d(stem output) at the
#       same 4e-2 bar as the patch-embed model test.  (1)+(2)+(3) chain to the whole gradient; tools/stem_cpu_emulation.py
#       (CPU suite) proves the tape walk in fp32 to 2.4e-6.
# ---------------------------------------------------------------------------------------------------------------
OP_BAR = 2e-2   # bf16 rounding of dx (4e-3) + bf16 operands; a wrong term in a backward formula shows up at >= 1e-1


@pytest.mark.parametrize("N,HW,C,relu,short", [(2, 35, 32, True, False), (3, 63, 64, False, False), (2, 24, 256, True, True), (1, 7, 1024, True, True),
                                               (2, 96, 1024, True, True)])
def test_group_norm_backward(ops, N, HW, C, relu, short):
    g = torch.Generator().manual_seed(C + HW)
    x = (torch.randn(N, HW, 1, C, generator=g) * 1.5 + 0.3).bfloat16()
    sc = torch.randn(N, HW, 1, C, generator=g).bfloat16() if short else None
    dy = (torch.randn(N, HW, 1, C, generator=g) * 0.2).bfloat16()
    gam, bet = torch.randn(C, generator=g) * 0.3 + 1.0, torch.randn(C, generator=g) * 0.2
    dev = lambda t: t.reshape(N * HW, C).to(DEV)
    y = torch.empty(N * HW, C, dtype=torch.bfloat16, device=DEV)
    stats, red = torch.empty(N * 64, device=DEV), torch.empty(N * 64, device=DEV)
    ops.group_norm_fwd(dev(x), gam.to(DEV), bet.to(DEV), y, stats, N, HW, C, 32, 1e-4, relu, dev(sc) if short else None)
    dx = torch.empty_like(y)
    dsc = torch.empty_like(y) if short else None
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    ops.group_norm_bwd(dev(dy), dev(x), y if relu else None, stats, gam.to(DEV), dx, dsc, dg, db, red, N, HW, C, 32, 1e-4, relu)
    # reference: autograd of the same op with the ReLU mask of the kernel's own forward output (identical rounding points)
    xr, gr, br = x.float().requires_grad_(True), gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
    scr = sc.float().requires_grad_(True) if short else None
    ref = O.group_norm(xr, {"s/gamma": gr, "s/beta": br}, "s")
    if short:
        ref = ref + scr
    if relu:
        ref = ref * (y.float().cpu().reshape(N, HW, 1, C) > 0).float()
    (ref * dy.float()).sum().backward()
    assert rel(dx, xr.grad.reshape(N * HW, C)) < OP_BAR
    assert rel(dg, gr.grad) < OP_BAR and rel(db, br.grad) < OP_BAR
    if short:
        assert rel(dsc, scr.grad.reshape(N * HW, C)) < OP_BAR


def test_pool_col2im_ws_backward(ops):
    g = torch.Generator().manual_seed(7)
    for N, h, w, C in ((2, 9, 7, 32), (1, 12, 22, 64)):  # avg-pool: adjoint of the forward (ragged windows weigh 1/cnt)
        ho, wo = (h + 1) // 2, (w + 1) // 2
        x = torch.randn(N, h, w, C, generator=g, requires_grad=True)
        dy = torch.randn(N, ho, wo, C, generator=g).bfloat16()
        (O.avg_pool_same(x, 2) * dy.float()).sum().backward()
        dx = torch.empty(N * h * w, C, dtype=torch.bfloat16, device=DEV)
        ops.avgpool2_same_bwd(dy.reshape(-1, C).to(DEV), N, h, w, C, dx)
        assert rel(dx, x.grad.reshape(N * h * w, C)) < 4e-3
    for N, h, w, C, stride in ((2, 9, 7, 32, 1), (1, 8, 12, 64, 1), (2, 10, 14, 32, 2)):  # col2im = im2col^T, elementwise
        ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
        dcol = torch.randn(N * ho * wo, 9 * C, generator=g).bfloat16()
        dx = torch.empty(N * h * w, C, dtype=torch.bfloat16, device=DEV)
        ops.col2im3x3(dcol.to(DEV), N, h, w, C, stride, dx)
        # reference: the adjoint of the oracle's conv with an identity-like kernel bank = scatter of the 9 taps
        xr = torch.zeros(N, h + 2, w + 2, C)
        d4 = dcol.float().reshape(N, ho, wo, 9, C)
        for t in range(9):
            ky, kx = t // 3, t % 3
            xr[:, ky:ky + (ho - 1) * stride + 1:stride, kx:kx + (wo - 1) * stride + 1:stride] += d4[:, :, :, t]
        assert rel(dx, xr[:, 1:h + 1, 1:w + 1].reshape(N * h * w, C)) < 4e-3  # one bf16 rounding of the 9-tap sum
    for kh, cin, cout in ((3, 16, 32), (1, 64, 24)):  # weight standardisation backward vs autograd
        rows = kh * kh * cin
        w2 = (torch.randn(rows, cout, generator=g) * 0.2 + 0.05).requires_grad_(True)
        dws = torch.randn(rows, cout, generator=g)
        mean = w2.mean(0, keepdim=True)
        ws = (w2 - mean) * torch.rsqrt(((w2 - mean) ** 2).mean(0, keepdim=True) + 1e-5)
        (ws * dws).sum().backward()
        dw = torch.full((rows, cout), 0.5, device=DEV)  # accumulates
        ops.ws_weights_bwd(dws.to(DEV), w2.detach().to(DEV), dw)
        assert rel(dw - 0.5, w2.grad) < 1e-4
    a = torch.randn(4096, generator=g).bfloat16()
    b = torch.randn(4096, generator=g).bfloat16()
    out = torch.empty(4096, dtype=torch.bfloat16, device=DEV)
    ops.add_bf16(a.to(DEV), b.to(DEV), out)
    assert torch.equal(out.cpu(), (a.float() + b.float()).bfloat16())


def test_ws_weights_multi_equals_per_kernel_launches(ops):
    """merlot_ws_weights_multi / merlot_ws_weights_bwd_multi (ops.WsPlan: every conv kernel of the stem in one launch each) run
    the same per-channel code as merlot_ws_weights / merlot_ws_weights_bwd: bit for bit the per-kernel results, for kernels
    whose channel counts are not multiples of the 32-channel block (so blocks of one item end mid-way) and whose row counts
    need padding; the gradients accumulate into non-zero buffers."""
    g = torch.Generator().manual_seed(11)
    shapes = {"a": (27, 40), "b": (576, 64), "c": (64, 24), "d": (9 * 16, 100)}
    kernels = {n: (torch.randn(r, c, generator=g) * 0.2 + 0.05).to(DEV) for n, (r, c) in shapes.items()}
    grads = {n: torch.full(s, 0.5, device=DEV) for n, s in shapes.items()}
    plan = ops.WsPlan(kernels, grads, DEV)
    plan.standardise()
    for n, (r, c) in shapes.items():
        kp = (r + 7) // 8 * 8
        assert torch.equal(plan.wstd[n], ops.ws_weights(kernels[n], kp)), n
    for n, (r, c) in shapes.items():
        plan.dws[n].copy_(torch.randn(plan.dws[n].shape, generator=g))
    plan.backward()
    for n, (r, c) in shapes.items():
        dw = torch.full((r, c), 0.5, device=DEV)
        ops.ws_weights_bwd(plan.dws[n][:r], kernels[n], dw)
        assert torch.equal(grads[n], dw), n


def _stem_model(tiny_cfg, h0, w0, batch=2, nc=2, save=True):
    from merlot_b200.modeling import MerlotModel
    from tests.test_gpu_model import build, synth
    cfg = _stem_cfg(tiny_cfg)
    image, ids, shuf, vid = synth(cfg, batch, nc, 16, h0, w0, 0)
    params, store, _ = build(cfg)
    draws = O.make_mask_draws(batch, 32, 6, cfg["vocab_size"], seed=5)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                    shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, save_for_backward=save)
    return cfg, m, params, store, (image, ids, shuf, vid)


def test_hybrid_stem_backward_in_situ(tiny_cfg):
    """Every op of the real lite_resnet50 tape (128x192 input: maps 64x96, 32x48, 16x24, 8x12; 4 frames), backward vs autograd
    of that single op on the GPU's own saved input and incoming gradient; plus gradient routing."""
    cfg, m, params, store, (image, ids, shuf, vid) = _stem_model(tiny_cfg, 128, 192)
    N = image.shape[0]
    tape = m._stem.tape
    rc = tape[-1][1]["y"]
    g = torch.Generator().manual_seed(3)
    d_rc = (torch.randn(rc.shape, generator=g) * 0.1).bfloat16().to(DEV)
    store.g.zero_()
    trace = []
    m._stem.backward(d_rc.clone(), trace=trace)
    assert len(trace) == len(tape)
    f = lambda t: t.float().cpu()
    worst = {"gn": 0.0, "conv": 0.0, "pool": 0.0, "param": 0.0}
    produced = {}   # y ptr -> list of dx contributions routed to it
    for t in trace:
        r, kind = t["r"], t["kind"]
        dy = f(t["dy"])
        if t.get("dx") is not None:
            produced.setdefault(r["x"].data_ptr(), []).append(f(t["dx"]))
        if t.get("dsc") is not None:
            produced.setdefault(r["shortcut"].data_ptr(), []).append(f(t["dsc"]))
        if kind == "gn":
            hw, c = r["hw"], r["c"]
            x = f(r["x"]).reshape(N, hw, 1, c).requires_grad_(True)
            gam = store.P(f"{r['scope']}/gamma").float().cpu().clone().requires_grad_(True)
            bet = store.P(f"{r['scope']}/beta").float().cpu().clone().requires_grad_(True)
            out = O.group_norm(x, {"s/gamma": gam, "s/beta": bet}, "s")
            sc = None
            if r["shortcut"] is not None:
                sc = f(r["shortcut"]).reshape(N, hw, 1, c).requires_grad_(True)
                out = out + sc
            if r["relu"]:
                out = out * (f(r["y"]).reshape(N, hw, 1, c) > 0).float()
            (out * dy.reshape(N, hw, 1, c)).sum().backward()
            e = [rel(f(t["dx"]), x.grad.reshape(N * hw, c))]
            if sc is not None:
                e.append(rel(f(t["dsc"]), sc.grad.reshape(N * hw, c)))
            worst["gn"] = max(worst["gn"], *e)
            worst["param"] = max(worst["param"], rel(store.G(f"{r['scope']}/gamma"), gam.grad), rel(store.G(f"{r['scope']}/beta"), bet.grad))
        elif kind == "pool":
            x = f(r["x"]).reshape(N, r["h"], r["w"], r["c"]).requires_grad_(True)
            ho, wo = (r["h"] + 1) // 2, (r["w"] + 1) // 2
            (O.avg_pool_same(x, 2) * dy.reshape(N, ho, wo, r["c"])).sum().backward()
            worst["pool"] = max(worst["pool"], rel(f(t["dx"]), x.grad.reshape(-1, r["c"])))
        else:
            k, cin, cout = r["k"], r["cin"], r["cout"]
            x = f(r["x"]).reshape(N, r["h"], r["w"], cin)
            if r["sub_half"]:
                x = (x - 0.5).bfloat16().float()
            x.requires_grad_(True)
            kern = store.P(r["kname"]).float().cpu().clone().reshape(k, k, cin, cout).requires_grad_(True)
            out = O.conv2d_fixed_padding(x, kern, strides=r["stride"], weight_standardization=True)
            (out * dy.reshape(out.shape)).sum().backward()
            if t["dx"] is not None:
                worst["conv"] = max(worst["conv"], rel(f(t["dx"]), x.grad.reshape(-1, cin)))
            worst["param"] = max(worst["param"], rel(store.G(r["kname"]).float().cpu().reshape(k, k, cin, cout), kern.grad))
    # routing: the gradient each op received = sum of the dx its consumers produced (bf16 adds in between)
    route = 0.0
    for t in trace:
        key = t["r"]["y"].data_ptr()
        if key in produced:
            route = max(route, rel(f(t["dy"]), sum(produced[key])))
    print(f"stem backward in situ ({len(trace)} ops): worst rel err {worst}, routing {route:.2e}")
    assert worst["gn"] < OP_BAR and worst["conv"] < OP_BAR and worst["pool"] < 5e-3 and worst["param"] < OP_BAR, worst
    assert route < 8e-3  # one or two bf16 roundings of the sum
    store.g.zero_()


def test_training_step_through_the_hybrid_stem(tiny_cfg, monkeypatch):
    """Whole pretraining step with the hybrid stem; the oracle's lite_resnet50 is replaced by a LEAF holding the GPU's stem
    output, so the two graphs share their rounding points at the stem boundary: the three losses, every non-stem gradient and the
    gradient handed to the stem are compared at bf16 noise-floor bars (1e-3 losses; gradients 6e-2 worst tensor, 2.5e-2 median, 4e-2 at the stem boundary)."""
    cfg, m, params, store, (image, ids, shuf, vid) = _stem_model(tiny_cfg, 128, 192)
    N = image.shape[0]
    rc = m._stem.tape[-1][1]["y"]
    hs, ws = 128 // 16, 192 // 16
    leaf_rc = rc.float().cpu().reshape(N, hs, ws, rc.shape[1]).clone().requires_grad_(True)
    monkeypatch.setattr(O, "lite_resnet50", lambda x, p, scope, layers, width=64, rnd=O._ident: leaf_rc)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(2, 32), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm)
    ll, _ = m.mask_loss()
    cl, _ = m.contrastive_loss()
    tl, _ = m.temporal_loss(shuf.to(DEV), vid.to(DEV))
    total_ref, _ = O.pretrain_losses(om, shuf, vid)
    total = float(ll) + float(cl) + float(tl)
    assert abs(total - float(total_ref)) <= 1e-3 * abs(float(total_ref)), (total, float(total_ref))
    store.g.zero_()
    m.backward()
    total_ref.backward()
    grads = store.to_tf_dict("g")
    worst = {}
    for k, v in leaf.items():
        if "resnet50lite" in k or v.grad is None or float(v.grad.norm()) < 1e-7:
            continue
        worst[k] = rel(grads[k], v.grad)
    e_rc = rel(m.d_rc, leaf_rc.grad.reshape(N * hs * ws, -1))
    stem_norm = sum(float(grads[k].norm()) for k in grads if "resnet50lite" in k)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    vals = sorted(worst.values())
    print(f"stem boundary: d(stem out) rel {e_rc:.3e}; non-stem worst {max(worst.values()):.3e} median {vals[len(vals) // 2]:.3e}; "
          f"stem grad norm sum {stem_norm:.3e}; worst tensors {top}")
    # bf16 noise floor of this graph: the worst single tensor of ~115 sits at 3.7-3.9e-2 run to run (the red.add order of the
    # split-K wgrads is not fixed), so the bar on the worst tensor is 6e-2 and the tighter bar goes on the median; a wrong
    # backward shows up at O(0.1-1) (the broken stem of round 1 measured 0.39 worst / 0.26 median).
    assert max(worst.values()) < 6e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    assert vals[len(vals) // 2] < 2.5e-2, vals[len(vals) // 2]
    assert e_rc < 4e-2
    assert stem_norm > 0 and all(torch.isfinite(grads[k]).all() for k in grads)
    store.g.zero_()
