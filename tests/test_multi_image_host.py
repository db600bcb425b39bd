"""Several images per text (num_imgs, img_mask; model/modeling.py:106-122) without a GPU: the oracle restatement
(tests/multi_image_oracle.py) against MerlotOracle where they overlap and against hand-derived answers, the image-count
arithmetic, and every ValueError / NotImplementedError of merlot_b200.modeling.check_num_imgs."""
import pytest
import torch

from oracle import merlot_oracle as O
from tests import multi_image_oracle as MI
from merlot_b200.modeling import check_num_imgs


def small_cfg(**kw):
    """Tiny widths; 64 x 64 frames: 4 x 4 patches, pooled to 2 x 2, so vcl = 5 viz tokens per image."""
    cfg = dict(use_bfloat16=True, hidden_size=128, vocab_size=1000, patch_size=16, spatial_pool_size=2, num_attention_heads=2,
               num_hidden_layers=2, num_vision_transformer_hidden_layers=1, num_lang_transformer_hidden_layers=1,
               intermediate_size=256, initializer_range=0.02, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
               max_position_embeddings=64, num_chunks_in_group=1, resnet_layers=[])
    cfg.update(kw)
    return cfg


def inputs(cfg, n_images, n_texts, L=8, seed=0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(n_images, 64, 64, 3, generator=g, dtype=dtype)
    ids = torch.randint(100, cfg["vocab_size"], (n_texts, L), generator=g)
    ids[:, 0] = O.START
    ids[:, L - 2:] = 0
    return image, ids.int()


def params(cfg, dtype=torch.float64):
    return {k: v.to(dtype) for k, v in O.init_params(cfg, seed=1, perturb=0.05).items()}


# ---- the restatement where it overlaps the existing oracle ----
@pytest.mark.parametrize("nt", [1, 4])
def test_one_image_matches_merlot_oracle(nt):
    """num_imgs = 1 with img_mask None or all true: exactly MerlotOracle's forward (mask_input=False)."""
    cfg = small_cfg(num_texts=nt)
    p = params(cfg)
    image, ids = inputs(cfg, 2, 2 * nt)
    ref = O.MerlotOracle(cfg, p, image, ids)
    for mask in (None, torch.ones(2, dtype=torch.bool), torch.ones(2, 1, dtype=torch.int64)):
        got = MI.MultiImageOracle(cfg, p, image, ids, img_mask=mask)
        for name in ("viz", "lang"):
            assert torch.equal(got.encoder_hidden_states[name], ref.encoder_hidden_states[name]), (name, mask)
        for k, v in ref.attention_log.items():
            assert torch.equal(got.attention_log[k], v), k


# ---- hand-derived known answers ----
def test_kat_masked_image_attention():
    """A row of two images with image 1 masked (plus a row with both valid).  The reference's mask (:152-158) scores every
    pair that touches a masked token -1e10 (utils/transformer.py:109-110), so, in every layer and head:
      * each query row of image 1 has all S scores equal: its softmax is exactly uniform, 1/S on every key;
      * every other row's weight on image 1's keys is exp(-1e10 - max) = 0 exactly, and its weights over the rest sum to 1.
    The row without a masked image sees no zero column."""
    cfg = small_cfg(num_imgs=2)
    p = params(cfg)
    image, ids = inputs(cfg, 4, 2, L=8)
    ids[:, 6:] = 3  # no padding text: the only masked tokens are image 1's of row 0
    m = MI.MultiImageOracle(cfg, p, image, ids, img_mask=torch.tensor([[1, 0], [1, 1]]))
    vcl = m.viz_chunk_length
    S = 2 * vcl + 8
    assert vcl == 5 and m.encoder_pieces[0]["end"] == 2 * vcl and m.encoder_info["hidden_state"].shape[1] == S
    probs = m.encoder_info["self_attn_probs"]  # [B, layers, S, S], head mean
    img1 = slice(vcl, 2 * vcl)
    rest = torch.cat([torch.arange(vcl), torch.arange(2 * vcl, S)])
    assert torch.equal(probs[0, :, img1], torch.full((2, vcl, S), 1.0 / S, dtype=torch.float64))
    assert torch.equal(probs[0][:, rest][:, :, img1], torch.zeros(2, len(rest), vcl, dtype=torch.float64))
    assert float((probs[0][:, rest][:, :, rest].sum(-1) - 1).abs().max()) < 1e-12
    assert float(probs[1].min()) > 0.0
    # attention_log sees the same validity (:192-193): the masked rows and columns are out of every block
    assert torch.equal(m.is_valid[0], torch.tensor([True] * vcl + [False] * vcl + [True] * 8))


def test_kat_image_position_embeddings():
    """vision_pos_emb without shuffling (:312-315,336): token t of image i gets img_idx_pe[i] + final_pe[t], images 0..n-1."""
    cfg = small_cfg()
    p = params(cfg)
    pe = MI.image_pos_emb(p, 3, 5, 2, 2)[0]
    for i in range(3):
        for t in range(5):
            want = p["vision_backbone/img_idx_pe"][i] + (p["vision_backbone/final_pe/cls_emb"][0, 0] if t == 0 else
                                                          p["vision_backbone/final_pe/pos_embs"][0, (t - 1) // 2, (t - 1) % 2])
            assert torch.equal(pe[i * 5 + t], want), (i, t)


@pytest.mark.parametrize("ni,nt", [(2, 1), (3, 1), (3, 4)])
def test_image_count_arithmetic(ni, nt):
    """(batch_size // nt) * ni images; image group g = images g*ni .. g*ni+ni-1 for texts g*nt .. g*nt+nt-1, its ni * vcl viz
    tokens first in each of them; joint token t < ni * vcl of row b is valid iff img_mask[b // nt, t // vcl]."""
    cfg = small_cfg(num_imgs=ni, num_texts=nt)
    groups = 2
    batch = groups * nt
    assert check_num_imgs(cfg, batch, 1, batch, groups * ni) == ni
    for n in (groups * ni - 1, groups * ni + 1, groups * nt):
        if n != groups * ni:
            with pytest.raises(ValueError, match=f"image batch {n} != "):
                check_num_imgs(cfg, batch, 1, batch, n)
    p = params(cfg)
    image, ids = inputs(cfg, groups * ni, batch)
    mask = torch.ones(groups, ni, dtype=torch.int32)
    mask[0, ni - 1] = 0
    m = MI.MultiImageOracle(cfg, p, image, ids, img_mask=mask)
    vcl = m.viz_chunk_length
    assert m.encoder_pieces[0]["end"] == ni * vcl == m.P * ni and m.encoder_pieces[1]["end"] == ni * vcl + 8
    t = torch.arange(ni * vcl)
    for b in range(batch):
        assert torch.equal(m.is_valid[b, :ni * vcl], mask[b // nt, t // vcl] != 0), b
    # the texts of one group see the same images: their viz hidden states differ only through the text they attend to
    if nt > 1:
        fresh = MI.MultiImageOracle(cfg, p, image, ids[[0] * batch], img_mask=mask)  # every row gets text 0
        assert torch.equal(fresh.encoder_hidden_states["viz"][0], fresh.encoder_hidden_states["viz"][nt - 1])
        assert not torch.equal(fresh.encoder_hidden_states["viz"][0], fresh.encoder_hidden_states["viz"][nt])


# ---- the checks of MerlotModel's constructor ----
def test_one_image_path_is_not_checked():
    """num_imgs = 1 and no img_mask: nothing new is checked (the existing path and its own checks)."""
    assert check_num_imgs(small_cfg(), 4, 2, 2, 999, mask_input=True, shuffled_idx_img=torch.zeros(4),
                          frame_copies=2) == 1
    assert check_num_imgs(small_cfg(disable_pairwise_lang_attn=True), 4, 1, 4, 4) == 1


def test_value_errors():
    cfg = small_cfg(num_imgs=2)
    with pytest.raises(ValueError, match="num_chunks == 1"):  # rule 1: the reshapes at :112, :121
        check_num_imgs(cfg, 2, 2, 2, 8)
    with pytest.raises(ValueError, match="image batch 5 != \\(batch_size 2 // num_texts 1\\) x num_imgs 2"):
        check_num_imgs(cfg, 2, 1, 2, 5)
    with pytest.raises(ValueError, match="not a multiple of num_texts"):
        check_num_imgs(small_cfg(num_imgs=2, num_texts=4), 6, 1, 6, 2)
    with pytest.raises(ValueError, match="img_mask has 3 entries"):  # :109
        check_num_imgs(cfg, 2, 1, 2, 4, img_mask=torch.ones(3, dtype=torch.bool))
    with pytest.raises(ValueError, match=r"\[1, 2\]"):
        check_num_imgs(small_cfg(num_imgs=2, num_texts=4), 4, 1, 4, 2, img_mask=torch.ones(4, dtype=torch.bool))
    with pytest.raises(ValueError, match="bool or integer"):
        check_num_imgs(cfg, 2, 1, 2, 4, img_mask=torch.ones(2, 2))
    with pytest.raises(ValueError, match="img_mask has 4 entries"):  # ni = 1: one entry per row of B // num_texts
        check_num_imgs(small_cfg(), 2, 1, 2, 2, img_mask=torch.ones(4, dtype=torch.uint8))
    # rule 3: more images than image position embeddings
    with pytest.raises(ValueError, match="num_imgs 5 exceeds max_vision_pos_embeddings 4"):
        check_num_imgs(small_cfg(num_imgs=5, max_vision_pos_embeddings=4), 1, 1, 1, 5)
    assert check_num_imgs(small_cfg(num_imgs=4, max_vision_pos_embeddings=4), 1, 1, 1, 4) == 4
    assert check_num_imgs(small_cfg(num_imgs=1024), 1, 1, 1, 1024) == 1024  # the default table has 1024 rows
    with pytest.raises(ValueError, match="1025 exceeds max_vision_pos_embeddings 1024"):
        check_num_imgs(small_cfg(num_imgs=1025), 1, 1, 1, 1025)
    with pytest.raises(ValueError, match="num_imgs must be >= 1"):
        check_num_imgs(small_cfg(num_imgs=0), 1, 1, 1, 0)


@pytest.mark.parametrize("ni,mask", [(2, None), (2, "mask"), (1, "mask")])
def test_not_implemented(ni, mask):
    """Rule 5: combinations the reference cannot run, or that no program of it uses."""
    cfg = small_cfg(num_imgs=ni)
    m = torch.ones(2, ni, dtype=torch.bool) if mask else None
    if ni > 1:
        with pytest.raises(NotImplementedError, match="shuffled_idx_img.*:319"):
            check_num_imgs(cfg, 2, 1, 2, 2 * ni, m, shuffled_idx_img=torch.zeros(2, dtype=torch.int32))
    with pytest.raises(NotImplementedError, match="mask_input"):
        check_num_imgs(cfg, 2, 1, 2, 2 * ni, m, mask_input=True)
    with pytest.raises(NotImplementedError, match="disable_pairwise_lang_attn"):
        check_num_imgs(small_cfg(num_imgs=ni, disable_pairwise_lang_attn=True), 2, 1, 2, 2 * ni, m)
    with pytest.raises(NotImplementedError, match="frame_copies"):
        check_num_imgs(cfg, 2, 1, 2, ni, m, frame_copies=2)
    assert check_num_imgs(cfg, 2, 1, 2, 2 * ni, m) == ni
