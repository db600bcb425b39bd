"""Attention-probability dropout in the fused attention kernels (pytest -m gpu; utils/transformer.py:114-115).

K2 (forward), K3 (backward), K4 (column sums) and the export kernel each regenerate the mask for the elements they hold.
These tests read each kernel's mask back bit for bit and compare it with the restatement in tests/attn_dropout_oracle.py, check
values against fp32 autograd under that mask, and run the training step with attention dropout on against the oracle."""
import pytest
import torch

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O
from tests import attn_dropout_oracle as AD
from tests.test_gpu_model import _partial_backward_equals_full, _step_parity, build, synth

pytestmark = pytest.mark.gpu

DEV = "cuda"
SEED = 2 ** 32 + 12345  # non-zero high word of the Philox key
SITE = 7
P = 0.1
DROP = (P, SEED, SITE)


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def _validity(B, S, masked, g):
    """bool [B, S] (ragged lengths and a hole in the last sequence, as test_gpu_kernels._attn_case) or None."""
    if not masked:
        return None
    lens = torch.randint(max(1, S // 3), S + 1, (B,), generator=g)
    v2 = torch.arange(S)[None] < lens[:, None]
    if S > 10:
        v2[-1, 5:9] = False
    return v2


def _u8(v2):
    return None if v2 is None else v2.to(torch.uint8).reshape(-1).contiguous().to(DEV)


def _nonzero(v2, B, S):
    """bool [B, S, S]: where the undropped probability is positive.  A padding query row is uniform over all keys."""
    if v2 is None:
        return torch.ones(B, S, S, dtype=torch.bool)
    return (v2[:, :, None] & v2[:, None, :]) | ~v2[:, :, None]


# ---------------------------------------------------------------------------------------------------------------
# the mask, bit for bit, in every orientation
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("S", [64, 266, 513, 1100])
def test_attention_dropout_mask_bits(ops, S, masked):
    """q = k = 0 makes P uniform.  Forward: V is a one-hot identity over a 64-key window, so ctx[q, c] > 0 <=> keep(q, k0 + c).
    Backward: dO is a one-hot identity over a 64-query window, so dV[k, c] > 0 <=> keep(q0 + c, k) (keys on the rows).
    Export (heads = 1): probs[q, k] > 0 <=> keep(q, k)."""
    B, heads = 2, 2
    H = heads * 64
    v2 = _validity(B, S, masked, torch.Generator().manual_seed(S + masked))
    vd = _u8(v2)
    nz = _nonzero(v2, B, S)
    want = torch.from_numpy(AD.attention_keep(SEED, SITE, B, heads, S, P)) & nz[:, None]
    eye = torch.eye(64, dtype=torch.bfloat16, device=DEV)
    qkv = torch.zeros(B * S, 3 * H, dtype=torch.bfloat16, device=DEV)
    v = qkv.view(B, S, 3, heads, 64)[:, :, 2]
    got_f = torch.zeros(B, heads, S, S, dtype=torch.bool)
    got_b = torch.zeros(B, heads, S, S, dtype=torch.bool)
    for w0 in range(0, S, 64):
        n = min(64, S - w0)
        v.zero_()
        v[:, w0:w0 + n] = eye[:n, None, :]
        ctx, lse = ops.attention_fwd(qkv, B, S, heads, vd, dropout=DROP)
        got_f[..., w0:w0 + n] = (ctx.view(B, S, heads, 64)[..., :n].permute(0, 2, 1, 3).float() > 0).cpu()
        d_ctx = torch.zeros(B * S, H, dtype=torch.bfloat16, device=DEV)
        d_ctx.view(B, S, heads, 64)[:, w0:w0 + n] = eye[:n, None, :]
        dqkv = ops.attention_bwd(qkv, ctx, d_ctx, lse, B, S, heads, vd, dropout=DROP)
        dv = dqkv.view(B, S, 3, heads, 64)[:, :, 2, :, :n]  # [B, key, head, query - w0]
        got_b[:, :, w0:w0 + n, :] = (dv.permute(0, 2, 3, 1).float() > 0).cpu()
    assert torch.equal(got_f, want)
    assert torch.equal(got_b, want)
    q1 = torch.zeros(B * S, 3 * 64, dtype=torch.bfloat16, device=DEV)
    _, lse1 = ops.attention_fwd(q1, B, S, 1, vd, dropout=DROP)
    pm = ops.attention_probs(q1, lse1, B, S, 1, vd, dropout=DROP)
    want1 = torch.from_numpy(AD.attention_keep(SEED, SITE, B, 1, S, P))[:, 0] & nz
    assert torch.equal((pm > 0).cpu(), want1)
    # the mask really is the one of this (seed, site): another site disagrees somewhere
    assert not torch.equal(want1, torch.from_numpy(AD.attention_keep(SEED, SITE + 1, B, 1, S, P))[:, 0] & nz)


# ---------------------------------------------------------------------------------------------------------------
# values against fp32 autograd under the restated mask
# ---------------------------------------------------------------------------------------------------------------
def _drop_case(B, S, heads, v2, seed, pair=None):
    """Seeded bf16 qkv and the fp32 reference of utils/transformer.py:98-120 with the probabilities dropped by the restated
    mask (x keep / (1 - p)).  Returns generator, qkv, dropped probabilities [B, heads, S, S], ctx [B*S, H], grad(d_ctx)."""
    g = torch.Generator().manual_seed(seed)
    H = heads * 64
    qkv = torch.randn(B * S, 3 * H, generator=g).bfloat16()
    mask = None
    if v2 is not None:
        mask = (v2[:, None, :] & v2[:, :, None]).float()
        if pair is not None:
            P_, chunk = pair
            seg = torch.cat([torch.zeros(P_, dtype=torch.int64), 1 + torch.arange(S - P_) // chunk])
            can = (seg[:, None] == seg[None]) | (seg == 0)[None] | (seg == 0)[:, None]
            mask = mask * can[None].float()
    factor = torch.from_numpy(AD.attention_keep(SEED, SITE, B, heads, S, P)).float() * float(DM.dropout_scale(P))
    x = qkv.float().reshape(B, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    q, k, v = (x[i].clone().requires_grad_(True) for i in range(3))
    probs, ctx4 = AD.attention_core(q, k, v, mask, lambda pr: pr * factor)
    ctx_ref = ctx4.permute(0, 2, 1, 3).reshape(B * S, H)

    def grad(d_ctx):
        gq, gk, gv = torch.autograd.grad(ctx_ref, (q, k, v), d_ctx.float(), retain_graph=True)
        return torch.stack([gq, gk, gv], 0).permute(1, 3, 0, 2, 4).reshape(B * S, 3 * H)
    return g, qkv, probs.detach(), ctx_ref.detach(), grad


def _assert_dqkv(dqkv, ref, H):
    for i in range(3):
        assert rel(dqkv[:, i * H:(i + 1) * H], ref[:, i * H:(i + 1) * H]) < 1.5e-2, "qkv"[i]


def _assert_colsums(ops, qd, lse, B, S, heads, vd, v2, probs, pair=(0, 0)):
    """K4 plain, and split at S // 3 with only valid queries contributing (attention_log), against the dropped head mean."""
    pm = probs.mean(1)  # [B, q, k]
    colsum = torch.zeros(B, S, device=DEV)
    ops.attention_colsum(qd, lse, colsum, B, S, heads, vd, pair=pair, dropout=DROP)
    assert rel(colsum, pm.sum(1)) < 2e-3
    split = S // 3
    c1, c2 = torch.zeros(B, S, device=DEV), torch.zeros(B, S, device=DEV)
    ops.attention_colsum(qd, lse, c1, B, S, heads, vd, pair=pair, dropout=DROP, colsum2=c2, split=split, valid_q=v2 is not None)
    wq = (v2 if v2 is not None else torch.ones(B, S, dtype=torch.bool)).float()[:, :, None]
    assert rel(c1, (pm * wq)[:, :split].sum(1)) < 2e-3
    assert rel(c2, (pm * wq)[:, split:].sum(1)) < 2e-3


DQ_MODE_CASES = [(128, 1), (129, 2), (512, 4), (513, 0), (640, 0), (1100, 0), (3968, 0)]  # (S, dQ slices; 0 = atomic)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("S,parts", DQ_MODE_CASES)
def test_attention_dropout_values(ops, S, parts, masked):
    """ctx, dq/dk/dv, the fused q/k/v bias gradient and the column sums at the bars of the dropout-free tests; the LSE is the
    undropped one, bit for bit; in atomic dQ mode the workspace comes back zeroed."""
    from merlot_b200._lib import lib
    assert lib().merlot_attention_bwd_dq_parts(S) == parts
    B, heads = (1, 2) if S > 2048 else (2, 2)
    H = heads * 64
    v2 = _validity(B, S, masked, torch.Generator().manual_seed(5 * S + masked))
    vd = _u8(v2)
    g, qkv, probs, ctx_ref, ref_grad = _drop_case(B, S, heads, v2, seed=7 * S + masked)
    qd = qkv.to(DEV)
    ctx, lse = ops.attention_fwd(qd, B, S, heads, vd, dropout=DROP)
    assert rel(ctx, ctx_ref) < 1e-2
    _, lse0 = ops.attention_fwd(qd, B, S, heads, vd)
    assert torch.equal(lse, lse0)
    d_ctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16()
    start = torch.randn(3 * H, generator=g) * 0.1
    d_bias = start.to(DEV)
    ws = ops.attention_bwd_workspace(B, S, heads, DEV)
    dqkv = ops.attention_bwd(qd, ctx, d_ctx.to(DEV), lse, B, S, heads, vd, dq_accum=ws, d_bias_qkv=d_bias, dropout=DROP)
    ref = ref_grad(d_ctx)
    _assert_dqkv(dqkv, ref, H)
    if not parts:
        assert torch.equal(ws, torch.zeros_like(ws))
    d_bias = d_bias.cpu().double()
    assert rel(d_bias, start.double() + dqkv.cpu().double().sum(0)) < 1e-5
    got, ref = d_bias - start.double(), ref.double()
    for i, name in enumerate("qkv"):
        blk = slice(i * H, (i + 1) * H)
        if name == "k":  # zero in exact arithmetic (softmax shift invariance survives the dropout): error vs |dK| sums
            err = float((got[blk] - ref[:, blk].sum(0)).norm() / ref[:, blk].abs().sum(0).norm())
        else:
            err = rel(got[blk], ref[:, blk].sum(0))
        assert err < 1e-2, (name, err)
    _assert_colsums(ops, qd, lse, B, S, heads, vd, v2, probs)


@pytest.mark.parametrize("B,P_,chunk,nch,heads", [(2, 100, 32, 5, 4), (1, 56, 80, 8, 2)])
def test_attention_dropout_disable_pairwise_lang_attn(ops, B, P_, chunk, nch, heads):
    """model/modeling.py:160-168 with dropout: forward, backward (S = 696: atomic dQ), column sums (split, valid queries) and
    the export kernel against the oracle under the reference's explicit mask."""
    S = P_ + chunk * nch
    H = heads * 64
    g0 = torch.Generator().manual_seed(S + chunk)
    v2 = torch.ones(B, S, dtype=torch.bool)
    for b in range(B):
        for c in range(nch):
            n_pad = int(torch.randint(0, chunk // 2 + 1, (1,), generator=g0))
            if n_pad:
                v2[b, P_ + (c + 1) * chunk - n_pad:P_ + (c + 1) * chunk] = False
    vd = _u8(v2)
    pair = (P_, chunk)
    g, qkv, probs, ctx_ref, ref_grad = _drop_case(B, S, heads, v2, seed=S, pair=pair)
    qd = qkv.to(DEV)
    ctx, lse = ops.attention_fwd(qd, B, S, heads, vd, pair=pair, dropout=DROP)
    assert rel(ctx, ctx_ref) < 1e-2
    d_ctx = (torch.randn(B * S, H, generator=g) * 0.1).bfloat16()
    dqkv = ops.attention_bwd(qd, ctx, d_ctx.to(DEV), lse, B, S, heads, vd, pair=pair, dropout=DROP)
    _assert_dqkv(dqkv, ref_grad(d_ctx), H)
    _assert_colsums(ops, qd, lse, B, S, heads, vd, v2, probs, pair=pair)
    pm = ops.attention_probs(qd, lse, B, S, heads, vd, pair=pair, dropout=DROP)
    assert rel(pm, probs.mean(1)) < 2e-3


def test_attention_dropout_p0_is_the_default_call(ops):
    """dropout=(0, seed, site) runs the dropout-free kernels: every output bit for bit the same as without the argument.
    (heads = 1 and slices-mode dQ, so no output depends on the order of atomic adds.)"""
    B, S, heads = 2, 300, 1
    v2 = _validity(B, S, True, torch.Generator().manual_seed(3))
    vd = _u8(v2)
    g = torch.Generator().manual_seed(4)
    qd = torch.randn(B * S, 3 * 64, generator=g).bfloat16().to(DEV)
    d_ctx = (torch.randn(B * S, 64, generator=g) * 0.1).bfloat16().to(DEV)
    outs = []
    for kw in ({}, {"dropout": (0.0, SEED, SITE)}):
        ctx, lse = ops.attention_fwd(qd, B, S, heads, vd, **kw)
        dqkv = ops.attention_bwd(qd, ctx, d_ctx, lse, B, S, heads, vd, **kw)
        colsum = torch.zeros(B, S, device=DEV)
        ops.attention_colsum(qd, lse, colsum, B, S, heads, vd, **kw)
        outs.append((ctx, lse, dqkv, colsum, ops.attention_probs(qd, lse, B, S, heads, vd, **kw)))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("p", [1.0, -0.1])
def test_attention_dropout_rejects_p_outside_unit_interval(ops, p):
    """p must lie in [0, 1): MerlotError(EINVAL) from the host check of every entry point, before anything is launched."""
    from merlot_b200._lib import MERLOT_EINVAL, MerlotError, lib
    B, S, heads, H = 1, 200, 2, 128
    qkv = torch.randn(B * S, 3 * H, device=DEV).bfloat16()
    zeros = torch.zeros(B * S, H, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(B, heads, S, device=DEV)
    ctx_out = torch.full((B * S, H), 7.0, dtype=torch.bfloat16, device=DEV)
    lse_out = torch.full((B, heads, S), 7.0, device=DEV)
    dqkv = torch.full((B * S, 3 * H), 7.0, dtype=torch.bfloat16, device=DEV)
    dsum = torch.full((B, heads, S), 7.0, device=DEV)
    colsum = torch.full((B, S), 7.0, device=DEV)
    probs = torch.full((B, S, S), 7.0, device=DEV)
    drop = (p, SEED, SITE)
    torch.cuda.synchronize()
    lib().merlot_reset_launch_count()
    calls = [lambda: ops.attention_fwd(qkv, B, S, heads, ctx=ctx_out, lse=lse_out, dropout=drop),
             lambda: ops.attention_bwd(qkv, zeros, zeros, lse, B, S, heads, dqkv=dqkv, dsum=dsum, dropout=drop),
             lambda: ops.attention_colsum(qkv, lse, colsum, B, S, heads, dropout=drop),
             lambda: ops.attention_probs(qkv, lse, B, S, heads, out=probs, dropout=drop)]
    for call in calls:
        with pytest.raises(MerlotError) as e:
            call()
        assert e.value.code == MERLOT_EINVAL
    assert lib().merlot_launch_count() == 0
    torch.cuda.synchronize()
    for t in (ctx_out, lse_out, dqkv, dsum, colsum, probs):
        assert bool((t.float() == 7.0).all())


# ---------------------------------------------------------------------------------------------------------------
# the model: the training step, eval mode, layer groups, export
# ---------------------------------------------------------------------------------------------------------------
def _wrong_attention_masks(seed, p, p_vit, p_attn, how):
    """The oracle hook of a step run with dropout_seed=seed, except that the attention probabilities are dropped with the
    masks of another seed or of the next site."""
    good = AD.dropout_hook(seed, p, p_vit, p_attn)
    other = AD.dropout_hook(seed + 1, p, p_vit, p_attn)

    def hook(key, x):
        if key[-1] != "probs":
            return good(key, x)
        if how == "seed":
            return other(key, x)
        return good((key[0], key[1] + 1, "probs"), x)
    return hook


@pytest.fixture
def oracle_drops_probs(monkeypatch):
    """The oracle's transformer calls its dropout hook on the softmax probabilities as well (tests/attn_dropout_oracle.py)."""
    monkeypatch.setattr(O, "transformer", AD.transformer)


def _attention_dropout_step(tiny_cfg, batch=2, nc=4, Lc=16, **extra):
    """test_pretrain_step_parity_training_mode with attention_probs_dropout_prob 0.1 in all three stacks, against the oracle
    under the kernels' masks at _step_parity's bars (hidden states, attention sums, attention_log, losses, every gradient, the
    AdamW step).  Oracles whose attention masks come from another seed or site miss the attention-sum bar (2e-3)."""
    cfg = dict(tiny_cfg, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2, attention_probs_dropout_prob=0.1, **extra)
    seed = 2 ** 32 + 91
    m = _step_parity(cfg, is_training=True, dropout_seed=seed, oracle_dropout=AD.dropout_hook(seed, 0.1, 0.2, 0.1),
                     batch=batch, nc=nc, Lc=Lc)
    summs = m.lang_transformer_info["attention_summs"]
    image, ids, shuf, _ = synth(cfg, batch, nc, Lc, 64, 96, 0)
    params, _, _ = build(cfg)
    B, Lj = batch * nc // cfg["num_chunks_in_group"], Lc * cfg["num_chunks_in_group"]
    draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), cfg["vocab_size"], seed=5)
    for how in ("seed", "site"):
        bad = O.MerlotOracle(cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_draws=draws,
                             dropout=_wrong_attention_masks(seed, 0.1, 0.2, 0.1, how))
        assert rel(summs, bad.attention_summs) >= 2e-3, how
    return m


def test_pretrain_step_parity_attention_dropout(tiny_cfg, oracle_drops_probs):
    _attention_dropout_step(tiny_cfg)


def test_pretrain_step_parity_attention_dropout_long_sequence(tiny_cfg, oracle_drops_probs):
    """L = 640, Sj = 696: every attention backward reduces dQ atomically."""
    from merlot_b200._lib import lib
    m = _attention_dropout_step(tiny_cfg, batch=1, nc=8, Lc=80, num_chunks_in_group=8, max_position_embeddings=1024)
    assert m._dims["Sj"] == 696 and lib().merlot_attention_bwd_dq_parts(696) == 0 and lib().merlot_attention_bwd_dq_parts(640) == 0


def test_eval_mode_ignores_attention_dropout(tiny_cfg):
    """is_training=False forces attention_probs_dropout_prob to 0 (model/modeling.py:88-90): bit for bit the 0.0 model.
    In training mode a probability of 1 is rejected."""
    from merlot_b200._lib import MERLOT_EINVAL, MerlotError
    from merlot_b200.modeling import MerlotModel
    image, ids, shuf, _ = synth(tiny_cfg, 2, 4, 16, 64, 96, 0)
    _, store, _ = build(tiny_cfg)
    outs = []
    for p in (0.0, 0.1):
        m = MerlotModel(dict(tiny_cfg, attention_probs_dropout_prob=p), is_training=False, use_tpu=False, image=image.to(DEV),
                        input_ids=ids.to(DEV), mask_input=False, shuffled_idx_img=shuf.to(DEV), params=store, dropout_seed=SEED)
        outs.append({n: m.encoder_hidden_states[n].clone() for n in ("viz", "lang")})
    for n in ("viz", "lang"):
        assert torch.equal(outs[0][n], outs[1][n]), n
    with pytest.raises(MerlotError) as e:
        MerlotModel(dict(tiny_cfg, attention_probs_dropout_prob=1.0), is_training=True, use_tpu=False, image=image.to(DEV),
                    input_ids=ids.to(DEV), mask_input=False, shuffled_idx_img=shuf.to(DEV), params=store, dropout_seed=SEED)
    assert e.value.code == MERLOT_EINVAL


def test_partial_stack_backward_equals_full_attention_dropout(tiny_cfg):
    """Layer-group backward calls draw each layer's attention mask from the same site as the full backward."""
    _partial_backward_equals_full(dict(tiny_cfg, attention_probs_dropout_prob=0.1), training=True)


def test_exported_attention_probabilities_training_mode(tiny_cfg, oracle_drops_probs):
    """With attention dropout on, the exported self_attn_probs are the head means of the DROPPED probabilities
    (utils/transformer.py:138), as in the oracle under the kernels' masks."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2, attention_probs_dropout_prob=0.1)
    seed = 2 ** 32 + 93
    image, ids, shuf, _ = synth(cfg, 2, 4, 16, 64, 96, 0)
    params, store, _ = build(cfg)
    draws = O.make_mask_draws(4, 32, 6, cfg["vocab_size"], seed=5)
    m = MerlotModel(cfg, is_training=True, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True,
                    shuffled_idx_img=shuf.to(DEV), params=store, mask_draws=draws, export_attention_probs=True, dropout_seed=seed)
    gm = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(4, 32), "masked_idx": m.lang_mask_info["masked_idx"].cpu()}
    om = O.MerlotOracle(cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_override=gm,
                        dropout=AD.dropout_hook(seed, 0.1, 0.2, 0.1))
    pj, pl = m.encoder_info["self_attn_probs"], m.lang_transformer_info["self_attn_probs"]
    assert rel(pl, om.lang_transformer_info["self_attn_probs"]) < 5e-3
    assert rel(pj, om.encoder_info["self_attn_probs"]) < 1e-2
    assert float((pj.sum(-1) - 1).abs().max()) > 1e-2  # rows of dropped probabilities do not sum to one
