"""Known-answer tests derived by hand from the reference SOURCE (SURVEY.md 8(c) i-x): the reference ships no tests,
so these pin the oracle (and the host logic) to closed-form facts.  CPU only."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import merlot_oracle as O
from oracle import oracle_np as N

HERE = os.path.dirname(os.path.abspath(__file__))


def _model(tiny_cfg, n=4, B=1):
    class M:
        pass
    m = object.__new__(O.MerlotOracle)
    m.config = dict(tiny_cfg, num_chunks_in_group=n)
    m.num_chunks_in_group, m.batch_size, m.num_chunks = n, B, n
    return m


def test_kat_i_temporal_labels(tiny_cfg):  # model/modeling.py:598-620
    m = _model(tiny_cfg)
    lab = m.allpairs_temporal_labels(torch.zeros(1, 4, dtype=torch.int32)).reshape(4, 4)
    assert lab.tolist() == [[1, 2, 2, 2], [3, 1, 2, 2], [3, 3, 1, 2], [3, 3, 3, 1]]
    lab = m.allpairs_temporal_labels(torch.tensor([[0, 0, 1, 1]])).reshape(4, 4)
    assert lab.tolist() == [[1, 2, 0, 0], [3, 1, 0, 0], [0, 0, 1, 2], [0, 0, 3, 1]]


def test_kat_iii_topk_val():  # model/modeling.py:418-419 with p=0.5, f=0.2
    assert abs(0.01 * 0.5 * 0.8 / (0.2 * 0.5) - 0.04) < 1e-12


def test_kat_iv_lr_schedule():  # utils/optimization.py:94-115
    T, W = 460000, 10000
    assert float(O.lr_scale(5000, T, W)) == pytest.approx(0.5, abs=1e-7)
    assert float(O.lr_scale(10000, T, W)) == pytest.approx(460000 / 450001 * (1 - 10000 / 460000), rel=1e-6)
    assert float(O.lr_scale(460000, T, W)) == 0.0
    assert float(O.lr_scale(0, T, W)) == 0.0
    from merlot_b200.optimization import learning_rate_scale
    for s in (0, 1, 5000, 9999, 10000, 123456, 460000, 999999):
        assert learning_rate_scale(s, T, W) == O.lr_scale(s, T, W)


def test_kat_v_packed_v_roundtrip():  # utils/optimization.py:267-288
    g = torch.Generator().manual_seed(0)
    v = torch.rand(20000, generator=g) * 10 ** torch.randint(-12, 2, (20000,), generator=g).float()
    dec = O.decode_v(O.encode_v(v))
    e = v.bfloat16().float()
    bound = torch.minimum((e - v).abs(), (e * 1.00390625 - v).abs())
    assert torch.all((dec - v).abs() <= bound * (1 + 1e-6) + 1e-45)
    assert torch.equal(O.decode_v(torch.tensor([2.0]).bfloat16()), torch.tensor([2.0]))
    assert torch.equal(O.decode_v(torch.tensor([-2.0]).bfloat16()), torch.tensor([2.0 * 1.00390625]))
    # numpy restatement agrees bit for bit
    assert np.array_equal(N.encode_v(v.numpy()), O.encode_v(v).float().numpy())


def test_kat_vi_uniform_softmax_for_padded_query():  # utils/transformer.py:109-112
    scores = torch.randn(1, 1, 3, 5)
    m = torch.zeros(1, 1, 3, 5)
    m[:, :, 0] = 1
    p = torch.softmax(scores * m - 1e10 * (1 - m), -1)
    assert torch.allclose(p[0, 0, 1], torch.full((5,), 0.2))


def test_kat_vii_contrastive_labels_single_replica(tiny_cfg):  # model/modeling.py:519 with my_group_idx = 0
    assert torch.arange(8).tolist() == list(range(8))


def test_kat_viii_shapes(tiny_cfg):  # utils/vision_transformer.py:225-233,263-264
    for (h, w), (sv, vcl) in {(192, 352): (266, 67), (192, 320): (242, 61), (384, 384): (578, 145)}.items():
        h1, w1 = h // 16, w // 16
        assert h1 * w1 + 2 == sv and (h1 // 2) * (w1 // 2) + 1 == vcl


def test_kat_ix_tokenizer_fixture():  # utils/encode/encoder.py, via tests/golden/reference_facts.json
    d = json.load(open(os.path.join(HERE, "golden", "reference_facts.json")))
    assert d["tokenizer"]["encode"][" answer question:"] == [3380, 1908, 125]
    assert d["tokenizer"]["specials"] == {"PADDING": 0, "MASK": 1, "START": 2}
    assert (O.PADDING, O.MASK, O.START) == (0, 1, 2)
    from merlot_b200 import modeling
    assert (modeling.PADDING, modeling.MASK, modeling.START) == (0, 1, 2)


def test_kat_x_weight_decay_regex():  # utils/optimization.py:125-147 + merlot.yaml param_overrides
    cfg = {"weight_decay_rate": 0.1, "learning_rate": 1e-3,
           "param_overrides": [[["LayerNorm", "layer_norm", "GroupNorm", "bias"], {"weight_decay_rate": 0}]]}
    from merlot_b200.params import hyper_for
    for name, wd in [("encoder/layer00/query_layer/bias", 0), ("lm_head/output_bias", 0),
                     ("encoder/layer03/LayerNorm_attn_ln0/gamma", 0), ("encoder/layer00/query_layer/kernel", 0.1),
                     ("word_embeddings/word_embeddings", 0.1), ("vision_backbone/vision_transformer/pos_embs/pos_embs", 0.1),
                     ("vision_backbone/vision_transformer/pos_embs/cls_emb", 0.1), ("vision_backbone/img_idx_pe", 0.1)]:
        assert O.weight_decay_for(name, cfg) == wd
        assert hyper_for(name, cfg)[1] == wd
    with pytest.raises(ValueError):
        O.weight_decay_for("x", {"param_overrides": [[["x"], {"momentum": 1}]]})
    with pytest.raises(ValueError):
        hyper_for("x", {"learning_rate": 1, "param_overrides": [[["x"], {"momentum": 1}]]})


def test_temporal_weights_all_easy_in_pretraining():  # SURVEY quirk 4: dataloader offset 16 < 64 => every pair weighs 0.01
    easy = torch.tensor([0, 1, 16, 19]) < 64
    w = (~(easy[:, None] & easy[None])).float() * 0.99 + 0.01
    assert torch.all(w == 0.01)


def test_mask_inputs_properties(tiny_cfg):  # model/modeling.py:381-489
    B, L = 3, 32
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(100, 1000, (B, L), generator=g)
    ids[:, ::16] = O.START
    ids[:, -4:] = 0
    summ = torch.rand(B, L, generator=g)
    draws = O.make_mask_draws(B, L, 6, 1000, seed=1)
    out = O.mask_inputs(ids, summ, tiny_cfg, draws)
    idx = out["masked_idx"]
    assert idx.shape == (B, 6) and torch.all(idx[:, 1:] > idx[:, :-1])  # sorted, distinct
    assert torch.all(torch.gather(ids, 1, idx.long()) >= 100)  # special tokens are never chosen
    changed = out["masked_ids"] != ids
    member = torch.zeros(B, L, dtype=torch.bool).scatter_(1, idx.long(), True)
    assert torch.all(member | ~changed)  # only chosen positions may change
    assert abs(out["topk_val"] - 0.04) < 1e-12


def test_two_restatements_agree():  # torch fp64 path vs independent numpy fp64 path
    g = torch.Generator().manual_seed(3)
    B, S, H, heads = 2, 7, 16, 2
    x = torch.randn(B, S, H, generator=g, dtype=torch.float64)
    p = {}
    for nm in ("query_layer", "key_layer", "value_layer", "context_projection_layer"):
        p[f"s/{nm}/kernel"] = torch.randn(H, H, generator=g, dtype=torch.float64) * 0.3
        p[f"s/{nm}/bias"] = torch.randn(H, generator=g, dtype=torch.float64) * 0.1
    valid = torch.tensor([[1, 1, 1, 1, 1, 0, 0], [1, 1, 1, 0, 1, 1, 1]], dtype=torch.float64)
    mask = valid[:, None] * valid[:, :, None]
    out, probs = O.attention_layer(x.reshape(B * S, H), mask, B, S, heads, p, "s")
    n = {k: v.numpy() for k, v in p.items()}
    out_n, probs_n = N.attention(x.numpy(), n["s/query_layer/kernel"], n["s/query_layer/bias"], n["s/key_layer/kernel"],
                                 n["s/key_layer/bias"], n["s/value_layer/kernel"], n["s/value_layer/bias"],
                                 n["s/context_projection_layer/kernel"], n["s/context_projection_layer/bias"], mask.numpy(), heads)
    assert np.allclose(out.reshape(B, S, H).numpy(), out_n, rtol=1e-9, atol=1e-11)
    assert np.allclose(probs.numpy(), probs_n, rtol=1e-9, atol=1e-12)
    assert np.allclose(probs_n[0, :, 5].sum(-1), 1.0) and np.allclose(probs_n[0, 0, 5], 1.0 / S)  # padded query: uniform
    gam, bet = torch.randn(H, generator=g, dtype=torch.float64), torch.randn(H, generator=g, dtype=torch.float64)
    ln = O.layer_norm(x, {"l/gamma": gam, "l/beta": bet}, "l")
    assert np.allclose(ln.numpy(), N.layer_norm(x.numpy(), gam.numpy(), bet.numpy()), rtol=1e-9, atol=1e-11)
    assert np.allclose(O.gelu(x).numpy(), N.gelu(x.numpy()), rtol=1e-12, atol=1e-14)
    logits = torch.randn(5, 11, generator=g, dtype=torch.float64)
    lab = torch.randint(0, 11, (5,), generator=g)
    assert np.allclose(O.raw_cross_entropy_with_logits(logits, lab).numpy(), N.cross_entropy(logits.numpy(), lab.numpy()))
    v = torch.randn(1000, generator=g).float()
    assert np.array_equal(N.bf16_round(v.numpy()), v.bfloat16().float().numpy())


def test_oracle_model_runs_and_is_deterministic(tiny_cfg):
    g = torch.Generator().manual_seed(0)
    image = torch.rand(4, 64, 96, 3, generator=g)
    ids = torch.randint(100, 1000, (2, 2, 16), generator=g, dtype=torch.int32)
    ids[:, :, 0] = O.START
    ids[:, :, 12:] = 0
    params = O.init_params(tiny_cfg, 1)
    shuf = torch.tensor([0, 1, 17, 16], dtype=torch.int32)
    vid = torch.zeros(2, 2, dtype=torch.int32)
    draws = O.make_mask_draws(2, 32, 6, 1000, seed=2)
    vals = []
    for _ in range(2):
        m = O.MerlotOracle(tiny_cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_draws=draws)
        tot, info = O.pretrain_losses(m, shuf, vid)
        vals.append(float(tot))
    assert vals[0] == vals[1] and math.isfinite(vals[0])
    assert m.encoder_hidden_states["viz"].shape == (2, 2 * 7, 128) and m.encoder_hidden_states["lang"].shape == (2, 32, 128)
    assert abs(sum(float(v) for v in m.attention_log.values()) - 1.0) < 1e-5
    # 2-D input_ids path (config 1): num_chunks = 1 (model/modeling.py:72-77)
    m1 = O.MerlotOracle(tiny_cfg, params, image[:2], ids[:, 0], mask_input=False)
    assert m1.num_chunks == 1 and m1.encoder_hidden_states["lang"].shape == (2, 16, 128)


def test_adam_oracle_matches_closed_form():  # utils/optimization.py:339-416, first step from zero moments
    p = {"w/kernel": torch.tensor([1.0, -2.0, 0.5]), "w/bias": torch.tensor([0.1])}
    g = {"w/kernel": torch.tensor([0.1, -0.2, 0.0]), "w/bias": torch.tensor([1.0])}
    cfg = dict(learning_rate=1e-2, num_train_steps=100, num_warmup_steps=0, weight_decay_rate=0.1, beta_2=0.98, epsilon=1e-6,
               use_bfloat16_adam=False, param_overrides=[[["bias"], {"weight_decay_rate": 0}]])
    opt = O.AdamOracle(p, cfg)
    p0 = {k: v.clone() for k, v in p.items()}
    opt.apply_gradients(p, g)
    lr_t = 1e-2 * 1.0 * math.sqrt(1 - 0.98) / (1 - 0.9)
    for k in p:
        m = 0.1 * g[k]
        v = 0.02 * (g[k] ** 2 + 1e-30)
        u = m / (v.sqrt() + 1e-6) + (0.1 * p0[k] if "kernel" in k else 0)
        assert torch.allclose(p[k], p0[k] - lr_t * u, rtol=1e-5, atol=1e-8)


# ---------------------------------------------------------------------------------------------------------------
# Hybrid ResNet-lite stem (SURVEY.md 8(f) next-row 1, Appendix D): restated in the oracle ahead of the CUDA path
# ---------------------------------------------------------------------------------------------------------------
def test_hybrid_stem_stage_shapes_and_parameter_count():  # utils/vision_transformer.py:118-170,206-223
    vt = "vision_backbone/vision_transformer"
    shapes = O.resnet_param_shapes(vt, [3, 4, 9], 64, 768)
    count = lambda pred: sum(int(np.prod(v)) for k, v in shapes.items() if pred(k))
    expect, cin = (27 * 32 + 9 * 32 * 32 + 9 * 32 * 64) + 2 * (32 + 32 + 64), 64   # three stem convs + their GroupNorms
    for f, blocks in ((64, 3), (128, 4), (256, 9)):                                # closed form, independent of the name walk
        expect += cin * 4 * f + 2 * 4 * f                                           # projection shortcut + GN (first block only)
        for b in range(blocks):
            expect += (cin if b == 0 else 4 * f) * f + 9 * f * f + f * 4 * f + 2 * (f + f + 4 * f)
        cin = 4 * f
    assert count(lambda k: "resnet50lite" in k) == expect == 11_914_080             # SURVEY Appendix D: 11.91 M
    assert count(lambda k: "conv_postresnet_proj" in k) == 1024 * 768 + 768  # + 0.79 M
    # creation-order names inside one variable scope (Appendix A)
    g1 = [k for k in shapes if "/block_group1/" in k and k.endswith("kernel")]
    assert [k.split("/")[-2] for k in g1[:5]] == ["conv2d", "conv2d_1", "conv2d_2", "conv2d_3", "conv2d_4"]
    assert shapes[f"{vt}/resnet50lite/block_group1/conv2d/kernel"] == (1, 1, 64, 256)     # projection shortcut first
    assert shapes[f"{vt}/resnet50lite/block_group1/conv2d_2/kernel"] == (3, 3, 64, 64)
    assert shapes[f"{vt}/resnet50lite/block_group3/conv2d/kernel"] == (1, 1, 512, 1024)
    assert f"{vt}/resnet50lite/stem/GroupNorm_stem2/gamma" in shapes
    cfg = dict(patch_size=16, hidden_size=768, resnet_layers=[3, 4, 9], num_hidden_layers=1, num_attention_heads=12,
               intermediate_size=3072, vocab_size=1000, max_position_embeddings=64, spatial_pool_size=2)
    p = O.init_params(cfg, seed=0)
    x = torch.rand(1, 192, 352, 3, generator=torch.Generator().manual_seed(0)) - 0.5
    st = O._ScopeNames(f"{vt}/resnet50lite/stem")
    x0 = torch.relu(O.group_norm(O.conv2d_fixed_padding(x, p[st.conv()], strides=2), p, st.gn("stem0")))
    assert tuple(x0.shape) == (1, 96, 176, 32)                                            # Appendix D, stem0
    rc = O.lite_resnet50(x, p, f"{vt}/resnet50lite", [3, 4, 9])
    assert tuple(rc.shape) == (1, 12, 22, 1024)                                           # Appendix D, block_group3
    info = O.vision_transformer_backbone(x + 0.5, cfg, p)
    assert tuple(info["seq"].shape) == (1, 66, 768) and tuple(info["cls"].shape) == (1, 2, 768)


def test_group_norm_and_weight_standardisation_kats():  # utils/model_utils.py:196-205, utils/vision_transformer.py:56-60
    c = 64
    p = {"g/gamma": torch.full((c,), 2.0), "g/beta": torch.full((c,), 0.25)}
    const = torch.ones(2, 3, 5, c) * torch.arange(c).float().div(2, rounding_mode="floor")  # constant inside every group of 2
    assert torch.allclose(O.group_norm(const, p, "g"), torch.full_like(const, 0.25))       # zero variance -> beta
    pm = torch.ones(1, 4, 4, c)
    pm[:, ::2] = -1.0                                                                      # every group: mean 0, E[x^2] = 1
    assert torch.allclose(O.group_norm(pm, p, "g"), pm * 2.0 / math.sqrt(1.0 + 1e-4) + 0.25, atol=1e-6)
    with pytest.raises(ValueError):
        O.group_norm(torch.zeros(1, 2, 2, 48), {"g/gamma": torch.ones(48), "g/beta": torch.zeros(48)}, "g")
    k = torch.randn(3, 3, 8, 16, generator=torch.Generator().manual_seed(1)) * 3 + 1
    delta = torch.zeros(1, 5, 5, 8)
    delta[0, 2, 2, 0] = 1.0  # an impulse reads the standardised kernel back (flipped): y[2-i+1, 2-j+1, :] = k_std[i, j, 0, :]
    y = O.conv2d_fixed_padding(delta, k)
    kstd = torch.stack([y[0, 3 - i, 3 - j] for i in range(3) for j in range(3)])           # [9, cout] for cin = 0
    full = (k - k.mean((0, 1, 2), keepdim=True)) / torch.sqrt(k.var((0, 1, 2), unbiased=False, keepdim=True) + 1e-5)
    assert torch.allclose(kstd, full[:, :, 0, :].reshape(9, 16), atol=1e-5)
    assert torch.allclose(full.mean((0, 1, 2)), torch.zeros(16), atol=1e-6)


def test_hybrid_stem_two_restatements_agree():  # torch fp64 (merlot_oracle) vs independent numpy fp64 (oracle_np)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 9, 7, 64, generator=g, dtype=torch.float64)
    gam, bet = torch.randn(64, generator=g, dtype=torch.float64), torch.randn(64, generator=g, dtype=torch.float64)
    a = O.group_norm(x, {"s/gamma": gam, "s/beta": bet}, "s")
    assert np.allclose(a.numpy(), N.group_norm(x.numpy(), gam.numpy(), bet.numpy()), rtol=1e-9, atol=1e-9)
    for k, s_, cin, cout in ((3, 2, 3, 8), (3, 1, 64, 16), (1, 1, 64, 32)):
        xi = torch.randn(2, 9, 7, cin, generator=g, dtype=torch.float64)
        w = torch.randn(k, k, cin, cout, generator=g, dtype=torch.float64)
        assert np.allclose(O.conv2d_fixed_padding(xi, w, strides=s_).numpy(), N.conv2d_ws(xi.numpy(), w.numpy(), s_), rtol=1e-9, atol=1e-9)
    assert np.allclose(O.avg_pool_same(x, 2).numpy(), N.avg_pool_same(x.numpy(), 2), rtol=1e-12)  # odd sizes: ragged last cell
    # a whole (tiny) stem end to end, numpy side composed here from the numpy primitives
    vt = "v"
    shapes = O.resnet_param_shapes(vt, [1, 1], 64, 32)
    p = {n_: (torch.randn(sh, generator=g, dtype=torch.float64) * (0.3 if n_.endswith("kernel") else 1.0)) for n_, sh in shapes.items()}
    img = torch.rand(1, 32, 48, 3, generator=g, dtype=torch.float64) - 0.5
    ref = O.lite_resnet50(img, p, f"{vt}/resnet50lite", [1, 1]).numpy()
    q = {k_: v.numpy() for k_, v in p.items()}

    def gn(xn, name):
        return N.group_norm(xn, q[f"{name}/gamma"], q[f"{name}/beta"])

    st, relu = f"{vt}/resnet50lite/stem", lambda t: np.maximum(t, 0.0)
    y = relu(gn(N.conv2d_ws(img.numpy(), q[f"{st}/conv2d/kernel"], 2), f"{st}/GroupNorm_stem0"))
    y = relu(gn(N.conv2d_ws(y, q[f"{st}/conv2d_1/kernel"]), f"{st}/GroupNorm_stem1"))
    y = relu(gn(N.conv2d_ws(y, q[f"{st}/conv2d_2/kernel"]), f"{st}/GroupNorm_stem2"))
    y = N.avg_pool_same(y, 2)
    for gi, stride in ((1, 1), (2, 2)):
        bg = f"{vt}/resnet50lite/block_group{gi}"
        sc = gn(N.conv2d_ws(N.avg_pool_same(y, stride) if stride > 1 else y, q[f"{bg}/conv2d/kernel"]), f"{bg}/GroupNorm")
        z = relu(gn(N.conv2d_ws(y, q[f"{bg}/conv2d_1/kernel"]), f"{bg}/GroupNorm_1"))
        z = relu(gn(N.conv2d_ws(z, q[f"{bg}/conv2d_2/kernel"]), f"{bg}/GroupNorm_2"))
        if stride > 1:
            z = N.avg_pool_same(z, stride)
        z = gn(N.conv2d_ws(z, q[f"{bg}/conv2d_3/kernel"]), f"{bg}/GroupNorm_3")
        y = relu(z + sc)
    assert ref.shape == y.shape == (1, 4, 6, 512)
    assert np.allclose(ref, y, rtol=1e-7, atol=1e-8)


# ---------------------------------------------------------------------------------------------------------------
# Training-mode dropout: the CUDA path's counter-based mask restated from its definition (oracle/dropout_mask.py), and the
# hook through which the oracle applies it at the reference's dropout call sites
# ---------------------------------------------------------------------------------------------------------------
def test_philox4x32_known_answers():
    """The round function and key schedule against the Philox4x32-10 known-answer vectors published with Random123
    (kat_vectors); the dropout mask runs the same rounds, 7 of them."""
    from oracle import dropout_mask as DM
    kats = [((0, 0, 0, 0), (0, 0), [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
            ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
            ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
             [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1])]
    for ctr, key, want in kats:
        assert [int(w) for w in DM.philox4x32(ctr, key, 10)] == want
    assert DM.DROPOUT_ROUNDS == 7


def test_dropout_threshold_and_scale():  # float32 host arithmetic: 0.1f * 65536 = 6553.6001, + 0.5, truncated
    from oracle import dropout_mask as DM
    assert (DM.thresh16(0.1), DM.thresh16(0.2), DM.thresh16(0.5)) == (6554, 13107, 32768)
    assert DM.dropout_scale(0.5) == np.float32(2.0) and DM.dropout_scale(0.1) == np.float32(1.1111112)


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_counter_dropout_keep_rate(p):
    from oracle import dropout_mask as DM
    keep = DM.counter_dropout_keep(2 ** 40 + 3, 223, 2048, 512, p)
    q = 1.0 - DM.thresh16(p) / 65536.0
    assert abs(keep.mean() - q) < 5.0 * math.sqrt(q * (1.0 - q) / keep.size)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_counter_dropout_keep_pairwise_uncorrelated(p):
    """Adjacent 16-bit lanes of one Philox word, adjacent counters (idx8), adjacent sites, and seeds s / s + 2^32 (the key's
    high word): every pair's correlation within 5 / sqrt(n)."""
    from oracle import dropout_mask as DM
    s, site, rows, N = 7, 1, 1024, 512
    k = DM.counter_dropout_keep(s, site, rows, N, p).reshape(-1, 8).astype(np.float64)

    def check(a, b):
        a, b = a.ravel(), b.ravel()
        assert abs(np.corrcoef(a, b)[0, 1]) < 5.0 / math.sqrt(a.size)

    check(k[:, 0::2], k[:, 1::2])  # low / high half of each word
    check(k[:-1], k[1:])  # idx8 and idx8 + 1
    check(k, DM.counter_dropout_keep(s, site + 1, rows, N, p).reshape(-1, 8))
    check(k, DM.counter_dropout_keep(s + 2 ** 32, site, rows, N, p).reshape(-1, 8))


def test_counter_dropout_keep_depends_on_linear_index_only():
    from oracle import dropout_mask as DM
    a = DM.counter_dropout_keep(2 ** 40 + 3, 301, 96, 768, 0.2)
    assert np.array_equal(a.ravel(), DM.counter_dropout_keep(2 ** 40 + 3, 301, 96 * 768 // 8, 8, 0.2).ravel())
    assert np.array_equal(a.ravel(), DM.counter_dropout_keep(2 ** 40 + 3, 301, 96 * 6, 128, 0.2).ravel())
    with pytest.raises(ValueError):
        DM.counter_dropout_keep(0, 0, 2, 12, 0.1)


def test_dropout_kernel_sites():  # merlot_b200/modeling.py _SITE_*, merlot_stack_forward: base + 2l (out-proj), + 2l + 1 (FFN2)
    from oracle import dropout_mask as DM
    assert [DM.kernel_site(k) for k in (("vit", 0, "attn"), ("vit", 0, "ffn"), ("vit", 3, "ffn"), ("langonly", 1, "attn"),
                                        ("joint", 11, "ffn"), ("embed", "langonly"), ("embed", "joint"))] == \
        [0, 1, 7, 102, 223, 300, 301]


def _oracle_case(tiny_cfg):
    g = torch.Generator().manual_seed(0)
    image = torch.rand(4, 64, 96, 3, generator=g)
    ids = torch.randint(100, 1000, (2, 2, 16), generator=g, dtype=torch.int32)
    ids[:, :, 0] = O.START
    ids[:, :, 12:] = 0
    params = O.init_params(tiny_cfg, 1, perturb=0.05)
    shuf = torch.tensor([0, 1, 17, 16], dtype=torch.int32)
    vid = torch.zeros(2, 2, dtype=torch.int32)
    draws = O.make_mask_draws(2, 32, 6, 1000, seed=2)
    return image, ids, params, shuf, vid, draws


def _oracle_outputs(m, shuf, vid):
    tot, info = O.pretrain_losses(m, shuf, vid)
    out = {"total": tot, "lang_trg_h": m.lang_trg_h, "img_trg_h": m.img_trg_h, "attention_summs": m.attention_summs,
           "masked_ids": m.lang_mask_info["masked_ids"], "masked_idx": m.lang_mask_info["masked_idx"],
           "vit": m.vision_transformer_info["hidden_state"], "lo": m.lang_transformer_info["hidden_state"],
           "joint": m.encoder_info["hidden_state"], "joint_probs": m.encoder_info["self_attn_probs"]}
    out.update({f"log/{k}": v for k, v in m.attention_log.items()})
    out.update({f"{h}/{k}": v for h, d in info.items() for k, v in d.items()})
    return out


def test_dropout_hook_off_leaves_the_oracle_unchanged(tiny_cfg):
    """No hook, dropout=None, an identity hook and a p = 0 training hook: every output bit for bit the same."""
    from oracle import dropout_mask as DM
    image, ids, params, shuf, vid, draws = _oracle_case(tiny_cfg)
    kw = dict(mask_input=True, shuffled_idx_img=shuf, mask_draws=draws)
    ref = _oracle_outputs(O.MerlotOracle(tiny_cfg, params, image, ids, **kw), shuf, vid)
    for hook in (None, lambda key, x: x, DM.dropout_hook(5, 0.0, 0.0)):
        got = _oracle_outputs(O.MerlotOracle(tiny_cfg, params, image, ids, dropout=hook, **kw), shuf, vid)
        assert got.keys() == ref.keys()
        for k in ref:
            assert torch.equal(torch.as_tensor(got[k]), torch.as_tensor(ref[k])), k


def test_dropout_hook_call_sites(tiny_cfg):
    """The hook runs exactly where the reference applies hidden dropout: 2 per layer in each of the three stacks (after the
    context projection, after the FFN output) and once after each embedding LayerNorm, on [rows, H] in logical row order."""
    image, ids, params, shuf, vid, draws = _oracle_case(tiny_cfg)
    calls = []

    def spy(key, x):
        calls.append((key, tuple(x.shape)))
        return x

    m = O.MerlotOracle(tiny_cfg, params, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_draws=draws, dropout=spy)
    H = tiny_cfg["hidden_size"]
    n_vit, n_lo, n_j = (tiny_cfg["num_vision_transformer_hidden_layers"], tiny_cfg["num_lang_transformer_hidden_layers"],
                        tiny_cfg["num_hidden_layers"])
    rows_vit = image.shape[0] * ((64 // 16) * (96 // 16) + 2)
    rows_lo = ids.shape[0] * ids.shape[1] * ids.shape[2]
    rows_j = m.B * (m.P + m.L)

    def stack(name, n, rows):
        return [((name, l, kind), (rows, H)) for l in range(n) for kind in ("attn", "ffn")]

    want = (stack("vit", n_vit, rows_vit) + [(("embed", "langonly"), (rows_lo, H))] + stack("langonly", n_lo, rows_lo)
            + [(("embed", "joint"), (m.B * m.L, H))] + stack("joint", n_j, rows_j))
    assert calls == want
    assert len(calls) == 2 * (n_vit + n_lo + n_j) + 2


def test_dropout_hook_mask_scale_and_gradient(tiny_cfg):
    """The training hook multiplies by keep * 1/(1-p) of the restated mask (vit_hidden_dropout_prob in the ViT), autograd
    carries the same factor back, and a whole oracle step with it is finite and differs from the eval step."""
    from oracle import dropout_mask as DM
    seed = 2 ** 32 + 9
    hook = DM.dropout_hook(seed, 0.2, 0.5)
    for key, p in ((("joint", 1, "ffn"), 0.2), (("vit", 0, "attn"), 0.5), (("embed", "langonly"), 0.2)):
        x = torch.randn(64, 128, generator=torch.Generator().manual_seed(1), requires_grad=True)
        y = hook(key, x)
        keep = torch.from_numpy(DM.counter_dropout_keep(seed, DM.kernel_site(key), 64, 128, p))
        factor = keep.float() * float(DM.dropout_scale(p))
        assert torch.equal(y, x * factor)
        y.sum().backward()
        assert torch.equal(x.grad, factor)
    image, ids, params, shuf, vid, draws = _oracle_case(tiny_cfg)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    kw = dict(mask_input=True, shuffled_idx_img=shuf, mask_draws=draws)
    m = O.MerlotOracle(tiny_cfg, leaf, image, ids, dropout=hook, **kw)
    tot, _ = O.pretrain_losses(m, shuf, vid)
    ev, _ = O.pretrain_losses(O.MerlotOracle(tiny_cfg, params, image, ids, **kw), shuf, vid)
    assert math.isfinite(float(tot.detach())) and float(tot.detach()) != float(ev)
    tot.backward()
    g = leaf["encoder/layer00/output/bias"].grad
    assert g is not None and torch.isfinite(g).all() and float(g.norm()) > 0
