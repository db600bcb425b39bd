"""The hybrid ResNet-lite stem (utils/vision_transformer.py:118-170, 206-223): one walk of lite_resnet50 that names its
variables and orders its ops, and HybridStem, which runs that walk forward on the K1 / K13 kernels and back along a tape."""
from __future__ import annotations

import functools
from typing import NamedTuple, Optional

import torch

from . import ops


class StemOp(NamedTuple):
    """One op of lite_resnet50.  Ops read and write named registers: "x" holds the running activation (a block's input
    until its last GroupNorm), "y" a block's main path, "sc" its projection shortcut."""
    kind: str                  # "conv" | "gn" | "pool"
    tag: str                   # buffer tag: an inference forward shares one buffer between the ops of a tag and shape
    name: str = ""             # conv: kernel variable; gn: GroupNorm variable scope
    k: int = 1                 # conv: kernel size (1 or 3)
    cin: int = 0               # conv: input channels
    cout: int = 0              # conv: output channels; gn: channels
    stride: int = 1            # conv
    sub_half: bool = False     # conv on the image, which is image - 0.5 (:193)
    relu: bool = True          # gn
    add: Optional[str] = None  # gn: register of the shortcut added before the ReLU (:95-96)
    src: str = "x"
    dst: str = "x"


@functools.lru_cache(maxsize=None)
def stem_ops(scope: str, layers: tuple, width: int = 64) -> tuple:
    """lite_resnet50's ops in execution order, with the reference's variable names (SURVEY.md Appendix A: conv2d, conv2d_1,
    ... / GroupNorm, GroupNorm_1, ... uniquified inside each variable scope).  The reference creates the variables in this
    same order, the projection shortcut of a block first (:77-85), so the walk also lists the variables."""
    out = []

    def namer(s):
        count = {"conv2d": 0, "GroupNorm": 0}

        def name(base):
            i, count[base] = count[base], count[base] + 1
            return f"{s}/{base}{'_%d' % i if i else ''}"
        return name

    nm = namer(f"{scope}/resnet50lite/stem")
    for i, (cin, cout) in enumerate(((3, width // 2), (width // 2, width // 2), (width // 2, width))):  # :138-159
        out.append(StemOp("conv", f"s{i}", nm("conv2d") + "/kernel", k=3, cin=cin, cout=cout, stride=2 if i == 0 else 1,
                          sub_half=i == 0))
        out.append(StemOp("gn", f"s{i}g", f"{scope}/resnet50lite/stem/GroupNorm_stem{i}", cout=cout))
    out.append(StemOp("pool", "s2p"))
    cin = width
    for i, blocks in enumerate(layers):
        nm = namer(f"{scope}/resnet50lite/block_group{i + 1}")
        f = width * 2 ** i
        for b in range(blocks):  # bottleneck_block (:69-96); only the first block of a group projects and strides (:109-113)
            pool = b == 0 and i > 0  # striding is an average pool: before the shortcut's 1x1, after the main path's 3x3
            if b == 0:
                if pool:
                    out.append(StemOp("pool", f"g{i}sp", dst="sc"))
                out.append(StemOp("conv", f"g{i}sc", nm("conv2d") + "/kernel", cin=cin, cout=4 * f, src="sc" if pool else "x",
                                  dst="sc"))
                out.append(StemOp("gn", f"g{i}scg", nm("GroupNorm"), cout=4 * f, relu=False, src="sc", dst="sc"))
            out.append(StemOp("conv", f"g{i}a", nm("conv2d") + "/kernel", cin=cin, cout=f, dst="y"))
            out.append(StemOp("gn", f"g{i}ag", nm("GroupNorm"), cout=f, src="y", dst="y"))
            out.append(StemOp("conv", f"g{i}b", nm("conv2d") + "/kernel", k=3, cin=f, cout=f, src="y", dst="y"))
            out.append(StemOp("gn", f"g{i}bg", nm("GroupNorm"), cout=f, src="y", dst="y"))
            if pool:
                out.append(StemOp("pool", f"g{i}bp", src="y", dst="y"))
            out.append(StemOp("conv", f"g{i}c", nm("conv2d") + "/kernel", cin=f, cout=4 * f, src="y", dst="y"))
            out.append(StemOp("gn", f"g{i}out{b % 2}", nm("GroupNorm"), cout=4 * f, src="y", add="sc" if b == 0 else "x"))
            cin = 4 * f
    return tuple(out)


class HybridStem:
    """lite_resnet50 on the device: NHWC bf16 activations as [N*h*w, C] matrices, every conv a K1 GEMM on weight-standardised
    bf16 kernels (1x1: the activation matrix itself; 3x3: an im2col matrix), GroupNorm32 (+ReLU / +shortcut) and the avg-pool
    striding as K13 kernels (csrc/stem.cu).  With `save` every op keeps its own buffers and is recorded on `tape` for
    backward(); without it, ops of one tag and shape share a buffer."""

    def __init__(self, store, bufs, layers, save: bool):
        self.store, self.bufs, self.save = store, bufs, bool(save)
        self.ops = stem_ops("vision_backbone/vision_transformer", tuple(layers))
        self.tape = None

    def plan(self):
        """The stem's conv kernels as one table (ops.WsPlan), cached on the store (the arenas' addresses never change)."""
        st = self.store
        names = [n for n in st.entries if "resnet50lite" in n and n.endswith("/kernel")]
        key = tuple(st.P(n).data_ptr() for n in names)
        plan = getattr(st, "_ws_plan_cache", None)
        if plan is None or plan.key != key:
            plan = ops.WsPlan({n: st.P(n) for n in names}, {n: st.G(n) for n in names}, st.device)
            st._ws_plan_cache = plan
        return plan

    def forward(self, img, N, h0, w0):
        """img: NHWC bf16 [N, h0, w0, 3].  Returns ([N*h*w, 4*f_last] bf16, h, w)."""
        st, bf, save = self.store, self.bufs, self.save
        self.N = N
        plan = self.plan()
        plan.standardise()  # :56-60 (fp32 moments, bf16 operand) for every conv kernel of the stem in one launch
        tape = []
        reg = {"x": (img, h0, w0, 3)}
        for site, op in enumerate(self.ops, 1):
            x, h, w, c = reg[op.src]
            if op.kind == "conv":
                kp = (op.k * op.k * op.cin + 7) // 8 * 8
                if op.k == 1:
                    a, ho, wo = x, h, w
                else:
                    ho, wo = (h + 2 - 3) // op.stride + 1, (w + 2 - 3) // op.stride + 1
                    a = bf.get("stem.col", (N * ho * wo, kp), torch.bfloat16)  # recomputed in the backward pass: never per-op
                    ops.im2col3x3(x, N, h, w, op.cin, op.stride, a, sub_half=op.sub_half)
                c = op.cout
            elif op.kind == "pool":
                ho, wo = (h + 1) // 2, (w + 1) // 2
            else:
                ho, wo = h, w
            y = bf.get(f"stem.{op.tag}.{site}" if save else f"stem.{op.tag}", (N * ho * wo, c), torch.bfloat16)
            if op.kind == "conv":
                ops.gemm(a, plan.wstd[op.name], b_mn_major=True, out=y)
                rec = dict(x=x, h=h, w=w, cin=op.cin, kname=op.name, k=op.k, stride=op.stride, sub_half=op.sub_half, y=y, ho=ho,
                           wo=wo, cout=c, kp=kp)
            elif op.kind == "pool":
                ops.avgpool2_same(x, N, h, w, c, y)
                rec = dict(x=x, h=h, w=w, c=c, y=y)
            else:
                stats = bf.get(f"stem.gn_stats.{site}" if save else "stem.gn_stats", (N * 64,), torch.float32)
                shortcut = reg[op.add][0] if op.add else None
                ops.group_norm_fwd(x, st.P(f"{op.name}/gamma"), st.P(f"{op.name}/beta"), y, stats, N, h * w, c, 32, 1e-4, op.relu,
                                   shortcut)
                rec = dict(x=x, y=y, scope=op.name, hw=h * w, c=c, relu=op.relu, shortcut=shortcut, stats=stats)
            tape.append((op.kind, rec))
            reg[op.dst] = (y, ho, wo, c)
        self.tape = tape if save else None
        return reg["x"][:3]

    def backward(self, d_out, trace=None):
        """Gradient of forward(): walks the tape backwards.  d_out: bf16 gradient of the stem output.  Parameter gradients are
        ACCUMULATED into the arena (conv kernels through the weight-standardisation backward, GroupNorm gamma/beta directly);
        activation gradients meet by tensor identity (a block input feeds the first 1x1 and the shortcut).  `trace`, a list,
        receives every op's (dy, dx, d_shortcut)."""
        st, bf, N, tape = self.store, self.bufs, self.N, self.tape
        grads = {tape[-1][1]["y"].data_ptr(): d_out}
        red = bf.get("stem.gn_red", (N * 64,), torch.float32)
        ctr = [0]
        plan = self.plan()  # holds the forward's standardised operands; the wgrad GEMMs accumulate into its gradient arena
        plan.zero_grads()

        def D(rows, cols):
            ctr[0] += 1
            return bf.get(f"stem.d.{ctr[0]}", (rows, cols), torch.bfloat16)

        def acc(t, g):
            k = t.data_ptr()
            if k in grads:
                ops.add_bf16(grads[k], g, grads[k])
            else:
                grads[k] = g

        for kind, r in reversed(tape):
            dy = grads.pop(r["y"].data_ptr(), None)
            if dy is None:
                continue
            if kind == "gn":
                dx = D(*r["x"].shape)
                dsc = D(*r["y"].shape) if r["shortcut"] is not None else None
                ops.group_norm_bwd(dy, r["x"], r["y"] if r["relu"] else None, r["stats"], st.P(f"{r['scope']}/gamma"), dx, dsc,
                                   st.G(f"{r['scope']}/gamma"), st.G(f"{r['scope']}/beta"), red, N, r["hw"], r["c"], 32, 1e-4, r["relu"])
                if trace is not None:
                    trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=dx.clone(), dsc=None if dsc is None else dsc.clone()))
                acc(r["x"], dx)
                if dsc is not None:
                    acc(r["shortcut"], dsc)
            elif kind == "pool":
                dx = D(*r["x"].shape)
                ops.avgpool2_same_bwd(dy, N, r["h"], r["w"], r["c"], dx)
                if trace is not None:
                    trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=dx.clone()))
                acc(r["x"], dx)
            else:  # conv
                kp, cout, M = r["kp"], r["cout"], N * r["ho"] * r["wo"]
                if r["k"] == 1:
                    a = r["x"]
                else:
                    a = bf.get("stem.col", (M, kp), torch.bfloat16)
                    ops.im2col3x3(r["x"], N, r["h"], r["w"], r["cin"], r["stride"], a, sub_half=r["sub_half"])
                dws = plan.dws[r["kname"]]
                ops.gemm(a, dy, a_mn_major=True, b_mn_major=True, out=dws, atomic=True, M=kp, N=cout, K=M)  # d(standardised kernel)
                if r["sub_half"]:
                    if trace is not None:
                        trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=None))
                    continue  # the image itself needs no gradient
                wstd = plan.wstd[r["kname"]]
                if r["k"] == 1:
                    dx = D(M, kp)
                    ops.gemm(dy, wstd, out=dx)  # dx[M, cin] = dy[M, cout] . wstd[cin, cout]^T
                else:
                    dcol = bf.get("stem.dcol", (M, kp), torch.bfloat16)
                    ops.gemm(dy, wstd, out=dcol)
                    dx = D(N * r["h"] * r["w"], r["cin"])
                    ops.col2im3x3(dcol, N, r["h"], r["w"], r["cin"], r["stride"], dx)
                if trace is not None:
                    trace.append(dict(kind=kind, r=r, dy=dy.clone(), dx=dx.clone()))
                acc(r["x"], dx)
        plan.backward()  # weight-standardisation backward of every conv kernel: arena gradients += d(standardise)/dw . dws
