"""Several images per text through the joint encoder on the GPU (pytest -m gpu): num_imgs and img_mask of MerlotModel
(model/modeling.py:106-122), against the restatement in tests/multi_image_oracle.py.

  * the joint-validity kernel (merlot_joint_valid_img) bit for bit against NumPy;
  * K2/K3/K4 on masked vision spans, with masked images across the 64-key and 128-key tile edges, element by element on the
    constructions and bounds of tests/attention_exact_oracle.py;
  * the model at tiny width, (num_imgs, num_texts) = (2, 1) and (3, 4) with images masked, in eval and in training mode
    (hidden and attention-probability dropout under the kernels' own masks): hidden states, attention_log and every
    parameter gradient of an injected d_hidden_state, to DESIGN section 3's bars (activations 1e-2, gradients 4e-2
    relative Frobenius);
  * the VCR towers (merlot_b200/vcr.py) unchanged on a num_imgs = 2, num_texts = 4 model: multi-frame multiple choice;
  * equivalences: num_imgs = 1 with an all-true mask is bitwise the unmasked model; a masked image's pixels change no valid
    token's output;
  * one size close to real use: 2 questions x 6 frames of 192 x 352, 4 candidate texts of 64 tokens, ViT-B + 12 joint
    layers (Sj = 466), forward against the oracle; the errors go to a JSON report ($MERLOT_MULTI_IMAGE_REPORT, else a fresh
    directory under the temporary directory)."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import merlot_oracle as O
from tests import attention_exact_oracle as X
from tests import attn_dropout_oracle as AD
from tests import multi_image_oracle as MI
from tests.test_gpu_attention_exact import locators, run

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from merlot_b200 import ops as o
    return o


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


# ------------------------------------------------------------------------------------------------------------
# the joint-validity kernel
# ------------------------------------------------------------------------------------------------------------
def valid_np(ids, mask, B, nt, ni, span):
    """model/modeling.py:106-122,148,152: the mask tiled to the nt texts of each group, then over each image's span tokens."""
    viz = np.ones((B, ni * span), dtype=bool) if mask is None else np.repeat(np.repeat(mask != 0, nt, axis=0), span, axis=1)
    return np.concatenate([viz, ids != 0], 1).astype(np.uint8).reshape(-1)


# (B, nt, ni, span, L)
VALID_CASES = [(1, 1, 1, 5, 8), (4, 1, 2, 67, 16), (8, 4, 3, 7, 7), (8, 4, 6, 67, 64), (6, 3, 1, 10, 33), (5, 1, 4, 1, 1),
               (3, 1, 1, 268, 128)]


@pytest.mark.parametrize("B,nt,ni,span,L", VALID_CASES)
def test_joint_valid_img_kernel(ops, B, nt, ni, span, L):
    """Bit-exact against NumPy, every byte of valid written; mask values 2 and 255 count as valid; the first image group
    has every image masked and the last row only padding text.  A null mask is every image valid."""
    g = np.random.default_rng(B * 1000 + ni * 10 + span)
    ids = g.integers(0, 4, size=(B, L)).astype(np.int32) * g.integers(0, 2, size=(B, L)).astype(np.int32)
    ids[-1] = 0
    mask = g.choice(np.array([0, 1, 2, 255], dtype=np.uint8), size=(B // nt, ni))
    mask[0] = 0
    ids_d = torch.from_numpy(ids).to(DEV)
    for m in (mask, None):
        out = torch.full((B * (ni * span + L),), 0xAB, dtype=torch.uint8, device=DEV)
        ops.joint_valid_img(ids_d, None if m is None else torch.from_numpy(m).to(DEV), out, B, nt, ni, span, L)
        want = valid_np(ids, m, B, nt, ni, span)
        assert np.array_equal(out.cpu().numpy(), want), (m is None, np.flatnonzero(out.cpu().numpy() != want)[:8])
    if ni == 1 and nt == 1:  # no mask: exactly merlot_joint_valid
        old = torch.full_like(out, 0xAB)
        ops.joint_valid(ids_d, old, B, span, L)
        assert torch.equal(old, out)


def test_joint_valid_img_rejects_bad_shapes(ops):
    from merlot_b200._lib import MerlotShapeError
    ids = torch.zeros(6, 4, dtype=torch.int32, device=DEV)
    out = torch.empty(6 * 14, dtype=torch.uint8, device=DEV)
    for B, nt, ni, span in ((6, 4, 2, 5), (6, 1, 0, 5), (6, 1, 2, 0), (0, 1, 2, 5)):
        with pytest.raises(MerlotShapeError):
            ops.joint_valid_img(ids, None, out, B, nt, ni, span, 4)


# ------------------------------------------------------------------------------------------------------------
# K2 / K3 / K4 on masked vision spans
# ------------------------------------------------------------------------------------------------------------
# (B, heads, ni, vcl, L, {row: masked images}, language lengths): S = ni * vcl + L
ATTN_CASES = {
    # S = 257: image 0 (tokens 0-66) across the 64-key tile edge, image 1 (67-133) across 128; row 2 has every image masked
    "3img_S257": (3, 12, 3, 67, 56, {0: [0], 1: [1], 2: [0, 1, 2]}, (56, 40, 56)),
    # the size close to real use: 6 x 67 + 64 = 466 (four K3 key tiles, dQ in slices); image 2 (134-200) across 192
    "6img_S466": (2, 2, 6, 67, 64, {0: [2], 1: [0, 5]}, (64, 33)),
    # S = 600 > 512: dQ reduced atomically; images 1, 2 and 7 masked, a masked span from 67 to 200 and one to the end of viz
    "8img_S600": (1, 2, 8, 67, 64, {0: [1, 2, 7]}, (50,)),
}


def span_validity(B, ni, vcl, L, masked, lens):
    v = torch.ones(B, ni * vcl + L, dtype=torch.bool)
    for b, imgs in masked.items():
        for i in imgs:
            v[b, i * vcl:(i + 1) * vcl] = False
    for b, n in enumerate(lens):
        v[b, ni * vcl + n:] = False
    return v


@pytest.mark.parametrize("name", list(ATTN_CASES))
def test_attention_masked_spans_routed_exact(ops, name):
    """The routed construction (every output bitwise but the fp32 sums whose order the kernels leave open), as
    test_gpu_attention_exact.test_routed_exact checks it, on vision spans masked image by image."""
    B, heads, ni, vcl, L, masked, lens = ATTN_CASES[name]
    S, split = ni * vcl + L, ni * vcl
    v = span_validity(B, ni, vcl, L, masked, lens)
    pair = (0, 0)
    c = X.routed(B, S, heads, v, pair, seed=S)
    tg = c["targets"]
    ref = X.reference(c["qkv"], c["d_ctx"], B, S, heads, v, pair, split=split, device=DEV,
                      weights=lambda b, h: X.routed_weights(tg, v, b, h, S))
    got, start = run(ops, c["qkv"], c["d_ctx"], B, S, heads, v, pair, B % 2 == 0, split)
    Lc = locators(B, S, heads)
    tag = f"{name} B={B} heads={heads}"
    vb = v[:, None, :].expand(B, heads, S)
    X.exact_check(got["ctx"], ref["ctx_emul"], f"ctx {tag}", Lc["ctx"])
    X.exact_check(got["lse"][vb], ref["lse"][vb].float(), f"lse (valid rows) {tag}", lambda i: f"valid entry {i}")
    X.ulp_check(got["lse"][~vb], ref["lse"][~vb], 4, f"lse (masked rows: ln S) {tag}", lambda i: f"masked entry {i}")
    X.exact_check(got["D"], ref["D"].float(), f"D {tag}", Lc["D"])
    want_dqkv = ref["dqkv"].float().bfloat16()
    X.exact_check(got["dqkv"], want_dqkv, f"dqkv {tag}", Lc["dqkv"])
    X.exact_check(got["bias"], (start.double() + want_dqkv.double().sum(0)).float(), f"bias gradient {tag}", Lc["bias"])
    for nm, key in (("c1", (True, 0)), ("c2", (True, 1))):  # valid queries only, split at the end of the vision piece
        X.ulp_check(got[nm], ref["cs"][key], 0 if heads <= 2 else heads, f"colsum {nm} {tag}", Lc["cs"])
    # masked keys: no valid query puts weight on them; the masked query rows' uniform 1/S is all they receive
    assert torch.equal(got["c1"][~v] + got["c2"][~v], torch.zeros(int((~v).sum())))
    want = ((~v).sum(1, keepdim=True).double() / S).expand(B, S)[~v]
    X.bound_check(got["cs"][~v], want, want * (heads * 2.0 ** -23 + 2 * (S + 64) * X.U + 2.0 ** -17),
                  f"colsum of masked keys {tag}", lambda i: f"masked key {i}", out_bf16=False)
    acc = (ref["export"] * heads * 2).round() / 2
    want_ex = acc.float() * torch.tensor(1.0 / heads, dtype=torch.float32)
    rows = v[:, :, None].expand(B, S, S)
    X.exact_check(got["export"][rows], want_ex[rows], f"export (valid rows) {tag}", lambda i: f"valid element {i}")
    X.bound_check(got["export"][~rows], ref["export"][~rows], ref["export"][~rows] * (2.0 ** -17 + 2.0 ** -21 + heads * 2.0 ** -23),
                  f"export (masked rows) {tag}", lambda i: f"masked element {i}", out_bf16=False)


@pytest.mark.parametrize("name", list(ATTN_CASES))
@pytest.mark.parametrize("peaked", [False, True])
def test_attention_masked_spans_random(ops, name, peaked):
    """Random data: every output of K2/K3/K4 within the element bounds of tests/attention_exact_oracle.py."""
    B, heads, ni, vcl, L, masked, lens = ATTN_CASES[name]
    S, split = ni * vcl + L, ni * vcl
    v = span_validity(B, ni, vcl, L, masked, lens)
    qkv, d_ctx = X.random_case(B, S, heads, seed=S + int(peaked), peaked=peaked)
    ref = X.reference(qkv, d_ctx, B, S, heads, v, (0, 0), split=split, bounds=True, device=DEV)
    got, _ = run(ops, qkv, d_ctx, B, S, heads, v, (0, 0), peaked, split, bias_start=False)
    Lc = locators(B, S, heads)
    tag = f"{name} peaked={peaked}"
    H = heads * 64
    X.bound_check(got["ctx"], ref["ctx"], ref["bar_ctx"], f"ctx {tag}", Lc["ctx"])
    X.bound_check(got["lse"], ref["lse"], ref["bar_lse"], f"lse {tag}", Lc["lse"], out_bf16=False)
    X.bound_check(got["D"], ref["D"], ref["bar_D"], f"D {tag}", Lc["D"], out_bf16=False)
    X.bound_check(got["bias"], ref["bias"], ref["bar_bias"], f"bias gradient {tag}", Lc["bias"], out_bf16=False)
    X.bound_check(got["export"], ref["export"], ref["bar_export"], f"export {tag}", Lc["export"], out_bf16=False)
    for i, nm in enumerate(("dq", "dk", "dv")):
        blk = slice(i * H, (i + 1) * H)
        X.bound_check(got["dqkv"][:, blk], ref["dqkv"][:, blk], ref["bar_dqkv"][:, blk], f"{nm} {tag}",
                      lambda idx, i=i: Lc["dqkv"]((idx[0], idx[1] + i * H)))
    cs, bcs = ref["cs"], ref["bar_cs"]
    X.bound_check(got["cs"], cs[(False, 0)] + cs[(False, 1)], bcs[(False, 0)] + bcs[(False, 1)], f"colsum {tag}", Lc["cs"], out_bf16=False)
    X.bound_check(got["c1"], cs[(True, 0)], bcs[(True, 0)], f"colsum (viz queries) {tag}", Lc["cs"], out_bf16=False)
    X.bound_check(got["c2"], cs[(True, 1)], bcs[(True, 1)], f"colsum2 (lang queries) {tag}", Lc["cs"], out_bf16=False)


# ------------------------------------------------------------------------------------------------------------
# the model at tiny width
# ------------------------------------------------------------------------------------------------------------
def build(cfg, seed=1):
    from merlot_b200.params import ParamStore
    params = O.init_params(cfg, seed=seed, perturb=0.05)
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    store = ParamStore(cfg, device=DEV)
    store.load_tf_dict(params)
    return params, store


def synth(cfg, groups, ni, nt, L=16, hw=(64, 96), seed=0):
    """groups image groups of ni frames, each with nt texts of L tokens (ragged padding)."""
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(groups * ni, *hw, 3, generator=g).bfloat16().float()
    ids = torch.randint(100, cfg["vocab_size"], (groups * nt, L), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(L // 2, L + 1, (groups * nt,), generator=g)
    return image, (ids * (torch.arange(L)[None] < lens[:, None])).int()


MASKS = {2: [[1, 0], [1, 1], [0, 1]], 3: [[1, 1, 0], [0, 1, 1], [1, 0, 1]]}


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("ni,nt", [(2, 1), (3, 4)])
def test_model_against_oracle(tiny_cfg, monkeypatch, ni, nt, train):
    """Forward (hidden states of both pieces, attention_log) and every parameter gradient of an injected d_hidden_state
    [B, P * ni + L, H] against the oracle.  Training mode: hidden dropout 0.1 (ViT 0.2) and attention-probability dropout 0.1,
    the oracle applying the kernels' masks of the same seed.  The image-index table gets gradient in rows 0 .. ni-1 only."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, num_imgs=ni, num_texts=nt, num_chunks_in_group=1, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2,
               attention_probs_dropout_prob=0.1 if train else 0.0)
    groups = 3 if ni == 2 else 2
    image, ids = synth(cfg, groups, ni, nt, seed=ni * 10 + nt)
    mask = torch.tensor(MASKS[ni][:groups], dtype=torch.bool)
    params, store = build(cfg)
    seed = 2 ** 32 + 90 + ni
    m = MerlotModel(cfg, is_training=train, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                    params=store, save_for_backward=True, dropout_seed=seed)
    hook = None
    if train:
        monkeypatch.setattr(O, "transformer", AD.transformer)
        hook = AD.dropout_hook(seed, 0.1, 0.2, p_attn=0.1)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    om = MI.MultiImageOracle(cfg, leaf, image, ids, img_mask=mask, dropout=hook)
    B, H, vcl = groups * nt, cfg["hidden_size"], m.viz_chunk_length
    Sj = ni * vcl + 16
    assert (m.B, m.num_imgs, m._dims["Pz"], m._dims["Sj"], m._dims["N"]) == (B, ni, ni * vcl, Sj, groups * ni)
    assert m.encoder_pieces == [{"name": "viz", "start": 0, "end": ni * vcl}, {"name": "lang", "start": ni * vcl, "end": Sj}]
    for name in ("viz", "lang"):
        assert m.encoder_hidden_states[name].shape == om.encoder_hidden_states[name].shape
        assert rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name]) < 1e-2, name
    for k, v in om.attention_log.items():
        assert abs(float(m.attention_log[k]) - float(v)) < 2e-3, k
    g = torch.Generator().manual_seed(7)
    w = (torch.randn(B, Sj, H, generator=g) * 0.05).bfloat16()
    store.g.zero_()
    m.backward(d_hidden_state=w.to(DEV))
    (om.encoder_info["hidden_state"] * w.float()).sum().backward()
    grads = store.to_tf_dict("g")
    worst = {k: rel(grads[k], v.grad) for k, v in leaf.items() if v.grad is not None and float(v.grad.norm()) > 1e-7}
    for k in ("vision_backbone/img_idx_pe", "vision_backbone/final_pe/pos_embs", "vision_backbone/final_pe/cls_emb",
              "vision_backbone/LayerNorm_final_ln/gamma", "vision_backbone/vision_transformer/conv2d/kernel",
              "position_embeddings/position_embeddings", "encoder/layer00/query_layer/kernel"):
        assert k in worst, k
    assert max(worst.values()) < 4e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    g_pe = grads["vision_backbone/img_idx_pe"]
    assert float(g_pe[ni:].abs().max()) == 0.0 and bool((g_pe[:ni].abs().sum(1) > 0).all())
    store.g.zero_()


class _Hidden:
    """What the oracle's VCR head reads of a model: encoder_hidden_states['lang'] as an autograd leaf."""

    def __init__(self, lang):
        self.encoder_hidden_states = {"lang": lang}


def test_vcr_towers_on_multi_frame_model(tiny_cfg):
    """Multi-frame multiple choice: vcr.cls_head, cls_loss and cls_head_backward unchanged on a num_imgs = 2, num_texts = 4
    model (2 questions: 4 image groups of 2 frames, 16 texts), one frame masked.  Logits and loss against the oracle of
    downstream/vcr/modeling.py (tests/vcr_oracle.py) on top of the multi-image restatement; the towers' gradients and their
    d_hidden_state (non-zero only at the first language row, P * num_imgs) against autograd on the GPU's hidden state, as
    tests/test_gpu_vcr_train.py checks the head; then the encoder backward from that d_hidden_state against the oracle."""
    from merlot_b200 import vcr
    from merlot_b200.modeling import MerlotModel
    from tests import vcr_oracle as V
    from tests.test_gpu_vcr_train import build as vcr_build
    cfg = dict(tiny_cfg, num_texts=4, num_imgs=2, num_chunks_in_group=1, hidden_dropout_prob=0.1)
    params, store = vcr_build(cfg)
    image, ids = synth(cfg, 4, 2, 4, seed=5)
    mask = torch.tensor([[1, 1], [1, 0], [1, 1], [1, 1]], dtype=torch.bool)
    target = torch.tensor([1, 3, 0, 2], dtype=torch.int32)
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                    params=store, save_for_backward=True)
    B, Sj, H, lang0 = m.B, m._dims["Sj"], cfg["hidden_size"], m._dims["Pz"]
    assert (B, lang0, m.encoder_pieces[1]["start"]) == (16, 2 * m.viz_chunk_length, lang0)
    logits = vcr.cls_head(m, store)
    loss, _ = vcr.cls_loss(logits, target.to(DEV))
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    om = MI.MultiImageOracle(cfg, leaf, image, ids, img_mask=mask)
    ref = V.vcr_cls_head_train(om, leaf)
    ref_loss, _ = V.vcr_loss(ref, target)
    assert tuple(logits.shape) == (4, 4) and rel(logits, ref) < 1e-2
    assert abs(float(loss) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    # the towers on the GPU's own hidden state
    lang = m.encoder_info["hidden_state"].float().cpu()[:, lang0:].clone().requires_grad_(True)
    towers = {k: v.detach().clone().requires_grad_(True) for k, v in params.items() if k.split("/")[0] in V.TOWERS}
    head_loss, _ = V.vcr_loss(V.vcr_cls_head_train(_Hidden(lang), towers), target)
    store.g.zero_()
    d_hidden = vcr.cls_head_backward(m, store, target.to(DEV))
    head_loss.backward()
    grads = store.to_tf_dict("g")
    for k, v in towers.items():
        if not k.endswith("classifier_mlp1/bias"):  # softmax is shift invariant: that bias's gradient is zero
            assert rel(grads[k], v.grad) < 4e-2, k
    d3 = d_hidden.float().cpu().reshape(B, Sj, H)
    assert rel(d3[:, lang0], lang.grad[:, 0]) < 4e-2
    assert float(d3[:, :lang0].abs().max()) == 0.0 and float(d3[:, lang0 + 1:].abs().max()) == 0.0
    # the encoder from the towers' d_hidden_state
    m.backward(d_hidden_state=d_hidden)
    (om.encoder_info["hidden_state"] * d3).sum().backward()
    grads = store.to_tf_dict("g")
    worst = {k: rel(grads[k], v.grad) for k, v in leaf.items() if k.split("/")[0] not in V.TOWERS and v.grad is not None
             and float(v.grad.norm()) > 1e-7}
    assert len(worst) > 40 and "vision_backbone/img_idx_pe" in worst
    assert max(worst.values()) < 4e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    store.g.zero_()


# ------------------------------------------------------------------------------------------------------------
# equivalences
# ------------------------------------------------------------------------------------------------------------
def test_all_true_mask_is_the_unmasked_model(tiny_cfg):
    """num_imgs = 1: an all-true img_mask (bool or integer) builds the same validity, so every output is bitwise that of
    img_mask=None, which runs merlot_joint_valid as before."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, num_chunks_in_group=1)
    image, ids = synth(cfg, 3, 1, 1, seed=2)
    _, store = build(cfg)
    outs = []
    for mask in (None, torch.ones(3, dtype=torch.bool), torch.full((3, 1), 7, dtype=torch.int64)):
        m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV),
                        img_mask=None if mask is None else mask.to(DEV), params=store)
        outs.append((m.encoder_info["hidden_state"].clone(), {k: float(v) for k, v in m.attention_log.items()}))
    for h, log in outs[1:]:
        assert torch.equal(h, outs[0][0])
        assert all(abs(log[k] - outs[0][1][k]) <= 1e-6 for k in log)  # K4's fp32 column sums add in an open order
    # ... and a mask that drops an image changes the model
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV),
                    img_mask=torch.tensor([True, False, True], device=DEV), params=store)
    h = m.encoder_info["hidden_state"]
    assert torch.equal(h[0], outs[0][0][0]) and not torch.equal(h[1], outs[0][0][1])


@pytest.mark.parametrize("ni,nt", [(2, 1), (3, 4)])
def test_masked_pixels_change_no_valid_token(tiny_cfg, ni, nt):
    """Eval mode, patch-embed stem: new pixels in the masked frames leave every valid token's output bitwise unchanged (each
    frame runs the ViT on its own and no valid query sees a masked key).  The masked tokens' own rows, and padding query rows
    (which attend uniformly to every key), do change."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, num_imgs=ni, num_texts=nt, num_chunks_in_group=1)
    assert not cfg["resnet_layers"]
    groups = 2
    image, ids = synth(cfg, groups, ni, nt, seed=9)
    mask = torch.tensor(MASKS[ni][:groups], dtype=torch.bool)
    _, store = build(cfg)
    outs = []
    for perturb in (False, True):
        img = image.clone()
        if perturb:
            g = torch.Generator().manual_seed(3)
            img[~mask.reshape(-1)] = torch.rand(img[~mask.reshape(-1)].shape, generator=g).bfloat16().float()
        m = MerlotModel(cfg, is_training=False, use_tpu=False, image=img.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                        params=store)
        outs.append(m.encoder_info["hidden_state"].clone())
    vcl = m.viz_chunk_length
    valid = torch.cat([mask.repeat_interleave(nt, 0).repeat_interleave(vcl, 1), ids != 0], 1).to(DEV)
    assert torch.equal(outs[0][valid], outs[1][valid])
    assert not torch.equal(outs[0][~valid], outs[1][~valid])


def test_constructor_rejects(tiny_cfg):
    """MerlotModel raises the checks of check_num_imgs (tests/test_multi_image_host.py has all of them) before any launch,
    and still refuses use_bfloat16: False and share_params: False."""
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg, num_imgs=2, num_chunks_in_group=1)
    image, ids = synth(cfg, 2, 2, 1)
    _, store = build(cfg)
    kw = dict(is_training=False, use_tpu=False, params=store)
    with pytest.raises(ValueError, match="image batch 3"):
        MerlotModel(cfg, image=image[:3].to(DEV), input_ids=ids.to(DEV), **kw)
    with pytest.raises(ValueError, match="num_chunks == 1"):
        MerlotModel(cfg, image=image.to(DEV), input_ids=ids.reshape(1, 2, 16).to(DEV), **kw)
    with pytest.raises(NotImplementedError, match="shuffled_idx_img"):
        MerlotModel(cfg, image=image.to(DEV), input_ids=ids.to(DEV), shuffled_idx_img=torch.zeros(4, dtype=torch.int32, device=DEV), **kw)
    with pytest.raises(NotImplementedError, match="mask_input"):
        MerlotModel(cfg, image=image.to(DEV), input_ids=ids.to(DEV), mask_input=True, **kw)
    with pytest.raises(NotImplementedError, match="use_bfloat16"):
        MerlotModel(dict(cfg, use_bfloat16=False), image=image.to(DEV), input_ids=ids.to(DEV), **kw)
    with pytest.raises(NotImplementedError, match="share_params"):
        MerlotModel(dict(cfg, share_params=False), image=image.to(DEV), input_ids=ids.to(DEV), **kw)


# ------------------------------------------------------------------------------------------------------------
# one size close to real use
# ------------------------------------------------------------------------------------------------------------
def test_six_frames_full_width_forward():
    """2 questions x 6 frames of 192 x 352 (6 x 11 pooled patches: 67 viz tokens per frame), frame 4 of question 1 masked,
    4 candidate texts of 64 tokens each: B = 8, P * num_imgs = 402, Sj = 466; merlot.yaml widths (ViT-B, 12 joint layers).
    Forward against the oracle on the same bf16-rounded weights; bars as tests/test_gpu_fullsize.py (1.5e-2 after 12 + 12
    bf16 layers; attention_log 2e-3)."""
    import sys
    from merlot_b200.modeling import MerlotModel
    from merlot_b200.params import ParamStore
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import bench
    cfg = dict(bench.load_config().model, hidden_dropout_prob=0.0, num_imgs=6, num_texts=4, num_chunks_in_group=1)
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    params = O.init_params(cfg, seed=1, perturb=0.05)
    params = {k: (v.bfloat16().float() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in params.items()}
    store = ParamStore(cfg, device=DEV)
    store.load_tf_dict(params)
    g = torch.Generator().manual_seed(21)
    image = torch.rand(12, 192, 352, 3, generator=g).bfloat16().float()
    ids = torch.randint(100, 50357, (8, 64), generator=g)
    ids[:, 0] = O.START
    lens = torch.randint(32, 65, (8,), generator=g)
    ids = (ids * (torch.arange(64)[None] < lens[:, None])).int()
    mask = torch.ones(2, 6, dtype=torch.bool)
    mask[1, 4] = False
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(DEV), input_ids=ids.to(DEV), img_mask=mask.to(DEV),
                    params=store)
    om = MI.MultiImageOracle(cfg, params, image, ids, img_mask=mask)
    assert (m.viz_chunk_length, m._dims["Pz"], m._dims["Sj"], m.B) == (67, 402, 466, 8)
    rep = {"dims": dict(B=8, N=12, vcl=67, Pz=402, Sj=466, L=64)}
    for name in ("viz", "lang"):
        rep[f"hidden_{name}_rel"] = rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name])
    v = om.is_valid
    rep["hidden_valid_tokens_rel"] = rel(m.encoder_info["hidden_state"].cpu()[v], om.encoder_info["hidden_state"][v])
    rep["attention_log_abs"] = {k: abs(float(m.attention_log[k]) - float(val)) for k, val in om.attention_log.items()}
    path = os.environ.get("MERLOT_MULTI_IMAGE_REPORT") or os.path.join(tempfile.mkdtemp(prefix="merlot_multi_image_"), "parity.json")
    with open(path, "w") as f:
        json.dump(rep, f, indent=1, sort_keys=True)
    print(f"multi-image parity report: {path}")
    for name in ("viz", "lang"):
        assert rep[f"hidden_{name}_rel"] < 1.5e-2, (name, rep)
    assert max(rep["attention_log_abs"].values()) < 2e-3, rep
