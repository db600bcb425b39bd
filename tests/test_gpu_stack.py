"""merlot_stack_forward / merlot_stack_backward called directly through the C ABI, against the float64 stack of
tests/stack_oracle.py: the output, the attention column sums and probabilities, the input gradient and every parameter
gradient of every layer, at tolerances an order below the whole-model tests'.  Also the stack's contract: forward-only mode,
the arena and scratch sizes it reports, no output that depends on what those buffers held, partial backwards over layer
groups, dh_in = NULL, and descriptors it must reject before it launches anything (pytest -m gpu)."""
import ctypes as C

import pytest
import torch

from merlot_b200._lib import MERLOT_EINVAL as EINVAL, MERLOT_ESHAPE as ESHAPE
from tests import stack_oracle as SO

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 2 ** 33 + 12345  # non-zero high key word
SITE_BASE = 1001
GUARD = 4096            # bytes of sentinel after the arena and the scratch
GUARD_BYTE = 0xA5

# name: B, S, H, heads, I, layers and features.  `valid` lists the valid prefix length of each sequence; "pair" is
# (pair_viz_len, pair_chunk_len); "split" the colsum split (with valid_q); "probs" requests attn_probs.
CASES = {
    "tiny_odd_rows": dict(B=2, S=37, H=128, heads=2, I=256, layers=3, valid=[30, 19], hidden_p=0.1, attn_p=0.1, probs=True),
    "degenerate": dict(B=3, S=1, H=64, heads=1, I=128, layers=3),                  # fewer rows than one LN block's warps
    "vit_shape": dict(B=8, S=266, H=768, heads=12, I=3072, layers=3, hidden_p=0.1),
    "joint_shape": dict(B=2, S=396, H=768, heads=12, I=3072, layers=3, valid=[390, 300], pair=(268, 32), split=268,
                        probs=True),
    "atomic_dq": dict(B=1, S=696, H=128, heads=2, I=256, layers=3, valid=[650], hidden_p=0.1, attn_p=0.1),  # > 4 key tiles
    "partial_ln_chunk": dict(B=2, S=130, H=320, heads=5, I=1000, layers=3),        # H % 256 != 0, I % 64 != 0
    "widest": dict(B=2, S=130, H=1024, heads=16, I=4096, layers=2),                # the fused LN backward's NCH = 4
}
GRAD_NAMES = ["g_" + n for n in SO.LAYER_PARAMS]

# Tolerances: rel-Frobenius error against the float64 stack (bf16 storage rounding included in the reference).  Observed on
# an H100 80GB HBM3 (700 W power limit), the largest of each and the case that sets it:
#   y              4.3e-3 tiny_odd_rows (partial_ln_chunk 4.2e-3, joint 3.9e-3, vit 3.8e-3, atomic_dq 3.6e-3, widest 2.9e-3)
#   colsum(2)      1.4e-4 tiny_odd_rows (5.0e-5 at the joint shape)
#   attn_probs     9.0e-4 tiny_odd_rows (3.7e-4 joint_shape)
#   dh_in          4.7e-3 tiny_odd_rows and atomic_dq
#   gradients      6.9e-3 g_ln1_beta of layer 1 in degenerate, 6.1e-3 g_ln1_gamma of layer 0 in vit_shape; d_final_beta 7e-8
# y is the one that cannot land far below the whole-model hidden-state bar (1e-2): the stack keeps the residual stream in
# bf16, rounding it at hmid and hout in every layer.  The reference rounds at the same points, but wherever the kernels' fp32
# value and the float64 one fall on either side of a rounding boundary they part by one bf16 ulp (2^-8 to 2^-7 relative),
# and the next layer computes on from the two different values.  After three layers the values y is rounded from differ by
# about an ulp in much of the tensor, so y's error is of the order of one bf16 ulp, whatever the kernels' arithmetic.  The
# forward is bitwise repeatable, so its bar needs no room for run-to-run spread: 1.4x the largest observed.
# The wrong references of test_wrong_references_miss_the_bars land at y 5.6e-2 (attention masks of the next site), 4.2e-1
# (dropout sites swapped) and g_ln2_gamma of the middle layer 0.5 (LN2's backward at LN1's statistics).
BARS = dict(y=6e-3, colsum=4e-4, probs=2e-3, dh_in=1e-2, grad=1.2e-2)
# Two runs of the same stack: the parameter gradients differ only by the order of fp32 atomic adds (split-K wgrads, the LN
# and bias column sums) while dQ is reduced without atomics (S <= 512): observed 6.3e-7.  Beyond, dQ's atomic fp32 sum flips
# bf16 roundings of dqkv and the layers below carry that on: observed 1.4e-4 on dh_in, 5.7e-4 on the gradients.
REPRO_BAR = 1e-5
REPRO_BAR_ATOMIC_DQ = 2e-3


def repro_bar(case):
    from merlot_b200 import _lib
    return REPRO_BAR if _lib.lib().merlot_attention_bwd_dq_parts(case["S"]) > 0 else REPRO_BAR_ATOMIC_DQ


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-300)).item()


def lib():
    from merlot_b200 import _lib
    return _lib.lib()


def make_inputs(case, seed=0):
    """CPU tensors of one case: bf16 weights in the [in, out] layout, fp32 vectors, bf16 input / output gradient, validity."""
    g = torch.Generator().manual_seed(seed)
    H, I = case["H"], case["I"]

    def w(i, o):
        return (torch.randn(i, o, generator=g) * (0.6 / i ** 0.5)).bfloat16()

    def vec(n, base=0.0, s=0.1):
        return base + s * torch.randn(n, generator=g)

    # b_o is centred at 0.5: each out-projection moves the row means of the residual stream, so that the statistics of
    # LN2's input (hmid) are not those of LN1's (h) and a backward that mixes them up shows
    layers = [dict(ln1_gamma=vec(H, 1.0), ln1_beta=vec(H), w_qkv=w(H, 3 * H), b_qkv=vec(3 * H), w_o=w(H, H), b_o=vec(H, 0.5),
                   ln2_gamma=vec(H, 1.0), ln2_beta=vec(H), w_1=w(H, I), b_1=vec(I), w_2=w(I, H), b_2=vec(H))
              for _ in range(case["layers"])]
    M = case["B"] * case["S"]
    valid = None
    if "valid" in case:
        valid = torch.zeros(case["B"], case["S"], dtype=torch.uint8)
        for b, n in enumerate(case["valid"]):
            valid[b, :n] = 1
        valid = valid.reshape(-1)
    return dict(layers=layers, final_gamma=vec(H, 1.0), final_beta=vec(H), h_in=torch.randn(M, H, generator=g).bfloat16(),
                dy=torch.randn(M, H, generator=g).bfloat16(), valid=valid)


def reference(case, inp, wrong=None):
    return SO.stack_reference(inp["layers"], inp["final_gamma"], inp["final_beta"], inp["h_in"], inp["dy"], B=case["B"],
                              S=case["S"], heads=case["heads"], valid=inp["valid"], pair=case.get("pair", (0, 0)),
                              hidden_p=case.get("hidden_p", 0.0), attn_p=case.get("attn_p", 0.0), seed=SEED,
                              site_base=SITE_BASE, colsum_split=case.get("split", 0), colsum_valid_q="split" in case,
                              wrong=wrong, device=DEV)


class Stack:
    """Device copies of one case's tensors and a merlot_stack_t over them; parameter gradients start random."""

    def __init__(self, case, inp, grad_scale):
        self.case = case
        B, S, H, L = case["B"], case["S"], case["H"], case["layers"]
        self.M = B * S
        self.w = [{k: v.to(DEV) for k, v in lp.items()} for lp in inp["layers"]]
        self.fg, self.fb = inp["final_gamma"].to(DEV), inp["final_beta"].to(DEV)
        self.h_in, self.dy = inp["h_in"].to(DEV), inp["dy"].to(DEV)
        self.valid = inp["valid"].to(DEV) if inp["valid"] is not None else None
        gen = torch.Generator(device=DEV).manual_seed(7)
        self.g = [{"g_" + k: torch.randn(v.shape, generator=gen, device=DEV) * grad_scale[l]["g_" + k]
                   for k, v in lp.items()} for l, lp in enumerate(self.w)]
        self.dfg = torch.randn(H, generator=gen, device=DEV) * grad_scale[-1]["d_final_gamma"]
        self.dfb = torch.randn(H, generator=gen, device=DEV) * grad_scale[-1]["d_final_beta"]
        self.y = torch.empty(self.M, H, dtype=torch.bfloat16, device=DEV)
        self.dh_in = torch.empty(self.M, H, dtype=torch.bfloat16, device=DEV)
        self.colsum = torch.zeros(B, S, device=DEV)
        self.colsum2 = torch.zeros(B, S, device=DEV) if "split" in case else None
        self.probs = torch.zeros(L, B, S, S, device=DEV) if case.get("probs") else None
        from merlot_b200 import _lib
        self.lp = (_lib.merlot_layer_params_t * L)()  # the descriptor's host array of device pointers
        for l in range(L):
            for n in SO.LAYER_PARAMS:
                setattr(self.lp[l], n, self.w[l][n].data_ptr())
                setattr(self.lp[l], "g_" + n, self.g[l]["g_" + n].data_ptr())

    def desc(self, save=1):
        from merlot_b200 import _lib as L
        c = self.case
        d = L.merlot_stack_t()
        d.B, d.S, d.H, d.I, d.heads, d.layers = c["B"], c["S"], c["H"], c["I"], c["heads"], c["layers"]
        d.layer_params = C.addressof(self.lp)
        d.final_gamma, d.final_beta = self.fg.data_ptr(), self.fb.data_ptr()
        d.d_final_gamma, d.d_final_beta = self.dfg.data_ptr(), self.dfb.data_ptr()
        d.valid = self.valid.data_ptr() if self.valid is not None else None
        d.h_in, d.y = self.h_in.data_ptr(), self.y.data_ptr()
        d.save_for_backward = save
        d.hidden_dropout_p, d.attention_dropout_p = c.get("hidden_p", 0.0), c.get("attn_p", 0.0)
        d.dropout_seed, d.dropout_site_base = SEED, SITE_BASE
        d.attn_colsum = self.colsum.data_ptr()
        if self.colsum2 is not None:
            d.attn_colsum2, d.attn_colsum_split, d.attn_colsum_valid_q = self.colsum2.data_ptr(), c["split"], 1
        d.attn_probs = self.probs.data_ptr() if self.probs is not None else None
        d.dy, d.dh_in = self.dy.data_ptr(), self.dh_in.data_ptr()
        d.pair_viz_len, d.pair_chunk_len = c.get("pair", (0, 0))
        return d

    def buffers(self, d, fill):
        """Arena and scratch of exactly the reported sizes, each followed by GUARD sentinel bytes, filled with `fill`."""
        n_act = lib().merlot_stack_activation_bytes(C.byref(d))
        n_scr = lib().merlot_stack_scratch_bytes(C.byref(d))
        arena = torch.full((n_act + GUARD,), fill, dtype=torch.uint8, device=DEV)
        scratch = torch.full((n_scr + GUARD,), fill, dtype=torch.uint8, device=DEV)
        arena[n_act:] = GUARD_BYTE
        scratch[n_scr:] = GUARD_BYTE
        d.act_arena, d.scratch = arena.data_ptr(), scratch.data_ptr()
        return arena, scratch

    def grads(self):
        return [{k: v.clone() for k, v in g.items()} for g in self.g], self.dfg.clone(), self.dfb.clone()

    def run(self, *, fill=0xFF, save=1, backward=True, groups=None, dh_in=True, on_group=None):
        """Forward (and backward, walked in `groups` with on_group(k) after call k) on buffers filled with `fill`.  Returns
        the outputs and the parameter-gradient increments as CPU tensors, and whether both guard tails are intact."""
        from merlot_b200 import ops
        d = self.desc(save)
        arena, scratch = self.buffers(d, fill)
        self.colsum.zero_()
        if self.colsum2 is not None:
            self.colsum2.zero_()
        if self.probs is not None:
            self.probs.fill_(float("nan"))
        self.y.fill_(float("nan"))
        self.dh_in.fill_(float("nan"))
        g0, dfg0, dfb0 = self.grads()
        st = ops._stream()
        lib().merlot_stack_forward(C.byref(d), st)
        out = dict(y=self.y.cpu(), colsum=self.colsum.cpu(), colsum2=None if self.colsum2 is None else self.colsum2.cpu(),
                   probs=None if self.probs is None else self.probs.cpu())
        if backward:
            if not dh_in:
                d.dh_in = None
            for k, (lo, hi) in enumerate(groups or [(0, 0)]):
                d.bwd_lo, d.bwd_hi = lo, hi
                lib().merlot_stack_backward(C.byref(d), st)
                if on_group is not None:
                    on_group(k)
            g1, dfg1, dfb1 = self.grads()
            out.update(dh_in=self.dh_in.cpu() if dh_in else None,
                       grads=[{k: (g1[l][k] - g0[l][k]).cpu() for k in GRAD_NAMES} for l in range(len(g1))],
                       d_final_gamma=(dfg1 - dfg0).cpu(), d_final_beta=(dfb1 - dfb0).cpu())
        torch.cuda.synchronize()
        n_act, n_scr = arena.numel() - GUARD, scratch.numel() - GUARD
        out["guard_ok"] = bool((arena[n_act:] == GUARD_BYTE).all()) and bool((scratch[n_scr:] == GUARD_BYTE).all())
        return out


def errors(out, ref):
    """{tensor name: rel error} of every compared output; gradients per layer as '<name>[l]'."""
    e = {"y": rel(out["y"], ref["y"]), "colsum": rel(out["colsum"], ref["colsum"])}
    if out.get("colsum2") is not None:
        e["colsum2"] = rel(out["colsum2"], ref["colsum2"])
    if out.get("probs") is not None:
        e["probs"] = rel(out["probs"], ref["probs"])
    if "grads" in out:
        if out["dh_in"] is not None:
            e["dh_in"] = rel(out["dh_in"], ref["dh_in"])
        e["d_final_gamma"] = rel(out["d_final_gamma"], ref["d_final_gamma"])
        e["d_final_beta"] = rel(out["d_final_beta"], ref["d_final_beta"])
        for l, (go, gr) in enumerate(zip(out["grads"], ref["grads"])):
            for k in GRAD_NAMES:
                e[f"{k}[{l}]"] = rel(go[k], gr[k])
    return e


def bar(name):
    if name in ("y", "dh_in", "probs"):
        return BARS[name]
    if name.startswith("colsum"):
        return BARS["colsum"]
    return BARS["grad"]


def over_bar(e):
    return {k: v for k, v in e.items() if v >= bar(k)}


@pytest.fixture(scope="module", params=list(CASES))
def setup(request):
    """(case, inputs, float64 reference, Stack, result of one full forward + backward on 0xFF-filled buffers)."""
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    case = CASES[request.param]
    inp = make_inputs(case, seed=len(request.param))
    ref = reference(case, inp)
    scale = [{k: float(v.std()) + 1e-6 for k, v in g.items()} for g in ref["grads"]]
    scale[-1].update(d_final_gamma=float(ref["d_final_gamma"].std()), d_final_beta=float(ref["d_final_beta"].std()))
    st = Stack(case, inp, scale)
    out = st.run()
    return request.param, case, inp, ref, st, out


def test_stack_against_float64_reference(setup):
    name, case, inp, ref, st, out = setup
    e = errors(out, ref)
    assert torch.isfinite(out["y"].float()).all() and torch.isfinite(out["dh_in"].float()).all()
    assert not over_bar(e), over_bar(e)


def test_wrong_references_miss_the_bars(setup):
    """Each bar is tight enough to see one wrong detail: dropout sites, attention-mask sites, LN2 backward statistics."""
    name, case, inp, ref, st, out = setup
    wrongs = ["ln2_stats"]
    if case.get("hidden_p"):
        wrongs.append("sites_swapped")
    if case.get("attn_p"):
        wrongs.append("attn_next_site")
    for w in wrongs:
        e = errors(out, reference(case, inp, wrong=w))
        assert over_bar(e), w


def test_forward_only_mode_matches_saved_mode(setup):
    """save_for_backward = 0 (one layer in the arena, hmid / hout as ping-pong buffers) gives y bitwise."""
    name, case, inp, ref, st, out = setup
    fo = st.run(save=0, backward=False)
    assert torch.equal(fo["y"], out["y"])
    assert fo["guard_ok"]


def test_reported_sizes_suffice_and_old_contents_are_not_read(setup):
    """Arena and scratch of exactly the reported sizes: the guard bytes after them survive forward and backward.  Buffers
    filled with 0xFF (bf16 / fp32 NaN) give the same y, bitwise, as zeroed ones; dh_in too where dQ has no atomics (S <= 512),
    and to fp32 reassociation beyond; the parameter gradients to fp32 reassociation."""
    name, case, inp, ref, st, out = setup
    assert out["guard_ok"]
    z = st.run(fill=0)
    assert z["guard_ok"]
    assert torch.isfinite(out["y"].float()).all() and torch.equal(out["y"], z["y"])
    assert torch.isfinite(out["dh_in"].float()).all()
    if lib().merlot_attention_bwd_dq_parts(case["S"]) > 0:
        assert torch.equal(out["dh_in"], z["dh_in"])
    else:
        assert rel(out["dh_in"], z["dh_in"]) < REPRO_BAR_ATOMIC_DQ
    worst = max(rel(out["grads"][l][k], z["grads"][l][k]) for l in range(case["layers"]) for k in GRAD_NAMES)
    assert worst < repro_bar(case)


def test_layer_groups_and_null_dh_in(setup):
    """Partial backwards over [(3,2),(2,1),(1,0)] and [(3,1),(1,0)] give the gradients of one full call; dh_in = NULL leaves
    every parameter gradient as it is with dh_in set."""
    name, case, inp, ref, st, out = setup
    L = case["layers"]
    bar_ = repro_bar(case)
    for groups in ([(l, l + 1) for l in reversed(range(L))], [(1, L), (0, 1)]):
        p = st.run(groups=groups)
        assert torch.equal(p["y"], out["y"])
        if lib().merlot_attention_bwd_dq_parts(case["S"]) > 0:
            assert torch.equal(p["dh_in"], out["dh_in"]), groups
        else:
            assert rel(p["dh_in"], out["dh_in"]) < REPRO_BAR_ATOMIC_DQ, groups
        for l in range(L):
            for k in GRAD_NAMES:
                assert rel(p["grads"][l][k], out["grads"][l][k]) < bar_, (groups, l, k)
    n = st.run(dh_in=False)
    for l in range(L):
        for k in GRAD_NAMES:
            assert rel(n["grads"][l][k], out["grads"][l][k]) < bar_, ("dh_in=NULL", l, k)


# (name, case, which calls, change to a valid descriptor): each is rejected with its code before anything is launched
REJECT_BASE = dict(B=1, S=696, H=128, heads=2, I=256, layers=3, valid=[650], probs=True)


def _set(**kw):
    return lambda d: [setattr(d, k, v) for k, v in kw.items()]


REJECTIONS = [
    ("bwd_range_inverted", REJECT_BASE, "bwd", _set(bwd_lo=2, bwd_hi=1), EINVAL),
    ("bwd_range_past_top", REJECT_BASE, "bwd", _set(bwd_lo=1, bwd_hi=4), EINVAL),
    ("bwd_range_negative", REJECT_BASE, "bwd", _set(bwd_lo=-1, bwd_hi=2), EINVAL),
    ("backward_without_saved_forward", REJECT_BASE, "bwd", _set(save_for_backward=0), EINVAL),
    ("hidden_not_heads_x_64", REJECT_BASE, "both", _set(heads=3), ESHAPE),
    ("intermediate_zero", dict(REJECT_BASE, S=130), "both", _set(I=0), ESHAPE),
    ("sequence_past_validity_mask", dict(B=1, S=3969, H=64, heads=1, I=128, layers=1, valid=[3000]), "both", _set(), ESHAPE),
    ("pair_mode_without_valid", dict(B=1, S=130, H=64, heads=1, I=128, layers=2), "both",
     _set(pair_viz_len=34, pair_chunk_len=32), EINVAL),
    ("attention_dropout_one", dict(REJECT_BASE, S=130), "both", _set(attention_dropout_p=1.0), EINVAL),
    ("dh_in_misaligned", REJECT_BASE, "bwd", lambda d: setattr(d, "dh_in", d.dh_in + 2), EINVAL),
    ("dy_misaligned", REJECT_BASE, "bwd", lambda d: setattr(d, "dy", d.dy + 2), EINVAL),
]


@pytest.mark.parametrize("name,case,which,change,code", REJECTIONS, ids=[r[0] for r in REJECTIONS])
def test_stack_rejects_before_launching(name, case, which, change, code):
    """A descriptor the stack cannot run returns its error code from the host checks: merlot_launch_count() stays 0 and every
    output, the gradients, the arena and the scratch keep their sentinels (atomic dQ mode's workspace memset included)."""
    from merlot_b200._lib import MerlotError
    inp = make_inputs(case)
    st = Stack(case, inp, [{"g_" + n: 1.0 for n in SO.LAYER_PARAMS} | {"d_final_gamma": 1.0, "d_final_beta": 1.0}
                           for _ in range(case["layers"])])
    d = st.desc(save=1)
    change(d)
    arena, scratch = st.buffers(d, 0x5A)  # sized for the descriptor as changed: a launch would stay inside them
    outs = [t for t in (st.y, st.dh_in, st.colsum, st.probs, st.dfg, st.dfb) if t is not None]
    outs += [t for g in st.g for t in g.values()]
    for t in outs:
        t.fill_(7.0)
    before = [t.clone() for t in outs] + [arena.clone(), scratch.clone()]
    torch.cuda.synchronize()
    lib().merlot_reset_launch_count()
    calls = {"fwd": [lib().merlot_stack_forward], "bwd": [lib().merlot_stack_backward]}.get(
        which, [lib().merlot_stack_forward, lib().merlot_stack_backward])
    for f in calls:
        with pytest.raises(MerlotError) as e:
            f(C.byref(d), torch.cuda.current_stream().cuda_stream)
        assert e.value.code == code, (f.__name__, e.value)
    assert lib().merlot_launch_count() == 0
    torch.cuda.synchronize()
    for t, b in zip(outs + [arena, scratch], before):
        assert torch.equal(t, b)
