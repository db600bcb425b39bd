"""The per-loss gradient checks of tests/test_gpu_loss_paths.py, shown to discriminate without a GPU: on the float64 oracle at
the GPU test's inputs, the per-loss gradients are linear, the MLM loss's share of the vision tower is below the summed-step
bar (the gap the per-loss checks close), the rows each table receives follow from the inputs, and an oracle with one path
cut or misrouted misses the per-loss bars by a wide margin while passing the summed one."""
import pytest
import torch

from oracle import merlot_oracle as O
from tests import loss_paths_oracle as LP
from tests.test_gpu_model import synth

MARGIN = 5.0  # a wrong path must miss its bar by at least this factor


@pytest.fixture(scope="module")
def case(tiny_cfg):
    """test_gpu_loss_paths.py's eval case: 2 videos x 4 segments, 16-token captions, 64x96 frames, mask draws seed 5; the
    masks are the ones the oracle chooses from those draws."""
    cfg = dict(tiny_cfg)
    image, ids, shuf, vid = synth(cfg, 2, 4, 16, 64, 96, 0)
    params = LP.tiny_params(cfg)
    draws = O.make_mask_draws(4, 32, 6, cfg["vocab_size"], seed=5)
    om = O.MerlotOracle(cfg, {k: v.float() for k, v in params.items()}, image, ids, mask_input=True, shuffled_idx_img=shuf,
                        mask_draws=draws)
    masks = {k: om.lang_mask_info[k] for k in ("masked_ids", "masked_idx")}
    args = (cfg, params, image, ids, shuf, vid, masks)
    return {"args": args, "ref": LP.oracle_grads(*args), "cfg": cfg, "ids": ids, "shuf": shuf, "masks": masks}


def _is_vision(name):
    return name.startswith("vision_backbone/")


def test_per_loss_gradients_add_up_to_the_step(case):
    """d(sum)/dp == sum of d(loss)/dp, in float64 (the key biases are rounding noise on both sides and are left out)."""
    ref = case["ref"]
    errs = {k: LP.rel(sum(ref[s][k] for s in LP.LOSSES), v) for k, v in ref["all"].items()
            if not LP.is_shift_invariant(k) and float(v.abs().max()) > 0}
    assert len(errs) > 100 and max(errs.values()) < 1e-12, max(errs.items(), key=lambda kv: kv[1])


def test_mlm_share_of_the_vision_tower_is_below_the_summed_bar(case):
    """At these inputs the MLM loss gives some vision tensors less of their gradient than the summed-step bar of
    tests/test_gpu_model.py (4e-2), so that bar cannot see the MLM path into the vision tower: the reason for the per-loss
    comparison."""
    ref = case["ref"]
    share = {k: float(ref["mlm"][k].norm() / v.norm()) for k, v in ref["all"].items()
             if _is_vision(k) and not LP.is_shift_invariant(k) and float(v.abs().max()) > 0}
    small = {k: s for k, s in share.items() if s < LP.SUMMED_STEP_BAR}
    assert all(s > 0 for s in share.values())  # the MLM loss does reach every vision tensor
    assert len(small) >= 10 and min(small.values()) < 1e-2, sorted(share.items(), key=lambda kv: kv[1])[:5]


def _grid(nh, nw):
    return {i * 64 + j for i in range(nh) for j in range(nw)}


def test_oracle_rows_follow_the_inputs(case):
    """The rows of each gathered table that receive a gradient, derived from the inputs alone, are the oracle's: word rows of
    the original ids under the contrastive loss (the language-only stack), of the masked ids under the temporal loss (the
    joint stack: [MASK] and random replacements included), every row under MLM (the tied output layer); position rows where
    some sequence has a valid token; the 4x6 ViT grid and the 2x3 final grid inside their 64x64 tables; img_idx_pe rows of
    shuffled_idx_img.  Padding rows get exactly nothing."""
    ref, ids, shuf, masks, cfg = case["ref"], case["ids"], case["shuf"], case["masks"], case["cfg"]
    mids = masks["masked_ids"].reshape(4, 32)
    lo = ids.reshape(2, 64)
    joint_pos = set(torch.nonzero((mids != 0).any(0)).reshape(-1).tolist())
    lo_pos = set(torch.nonzero((lo != 0).any(0)).reshape(-1).tolist())
    want = {
        "ctr": {"word_embeddings/word_embeddings": set(ids[ids != 0].tolist()),
                "position_embeddings/position_embeddings": set(), "langonly_embeddings/position_embeddings": lo_pos,
                "vision_backbone/final_pe/pos_embs": set(), "vision_backbone/final_pe/cls_emb": set(),
                "vision_backbone/img_idx_pe": set()},
        "tmp": {"word_embeddings/word_embeddings": set(mids[mids != 0].tolist()),
                "position_embeddings/position_embeddings": joint_pos, "langonly_embeddings/position_embeddings": set()},
        "mlm": {"word_embeddings/word_embeddings": set(range(cfg["vocab_size"])),
                "position_embeddings/position_embeddings": joint_pos, "langonly_embeddings/position_embeddings": set()},
    }
    for sub in ("tmp", "mlm"):
        want[sub].update({"vision_backbone/final_pe/pos_embs": _grid(2, 3), "vision_backbone/final_pe/cls_emb": {0},
                          "vision_backbone/img_idx_pe": set(shuf.tolist())})
    for sub in want:
        want[sub].update({"vision_backbone/vision_transformer/pos_embs/pos_embs": _grid(4, 6),
                          "vision_backbone/vision_transformer/pos_embs/cls_emb": {0, 1}})
        assert set(want[sub]) == set(LP.ROW_TABLES)
        for name, rows in want[sub].items():
            assert LP.nonzero_rows(name, ref[sub][name]) == rows, (sub, name)
    # the cases the table distinguishes are really there: masked ids differ from the originals, shuffled groups are offset
    assert set(mids[mids != 0].tolist()) != set(ids[ids != 0].tolist()) and 1 in set(mids.reshape(-1).tolist())
    assert max(joint_pos) < 32 and max(lo_pos) < 64 and {16, 64} & set(shuf.tolist())


@pytest.mark.parametrize("variant,loss", [("mlm_no_viz", "mlm"), ("tmp_swap", "tmp"), ("ctr_no_lang", "ctr")])
def test_wrong_path_misses_its_per_loss_bar(case, variant, loss):
    """An oracle with one path of `loss` cut or misrouted, compared as the GPU's gradient is: some tensor misses the per-loss
    bar by MARGIN or more, and a cut path also breaks the zero pattern."""
    ref = case["ref"]
    got = LP.oracle_grads(*case["args"], variant=variant)
    errs = LP.tensor_errors(got[loss], ref[loss])
    worst = max(errs.items(), key=lambda kv: kv[1])
    assert worst[1] >= MARGIN * LP.BARS["eval"][loss], worst
    if variant != "tmp_swap":  # a cut path leaves gradients the oracle gives a value entirely zero
        assert LP.zero_pattern_violations(got[loss], ref[loss])
    for other in set(LP.LOSSES) - {loss}:  # the cut touches its own loss only
        assert max(LP.tensor_errors(got[other], ref[other]).values()) < 1e-12
    if variant == "mlm_no_viz":
        # ... and the old summed-gradient bar does not see it: vision tensors it leaves within 4e-2
        summed = {k: e for k, e in LP.tensor_errors(got["all"], ref["all"]).items() if _is_vision(k)}
        hidden = [k for k, e in summed.items() if e < LP.SUMMED_STEP_BAR and errs[k] >= MARGIN * LP.BARS["eval"][loss]]
        assert len(hidden) >= 10, sorted(summed.items(), key=lambda kv: kv[1])[:5]


def test_misrouted_position_row_misses_the_row_check(case):
    """One row of a table's gradient moved to its neighbour: the row sets differ and the moved rows miss the per-row bar by
    MARGIN or more.  In the 1000-row word table the same move stays under the summed-step bar as a whole tensor."""
    ref = case["ref"]["tmp"]
    name = "position_embeddings/position_embeddings"
    rows = sorted(LP.nonzero_rows(name, ref[name]))
    r = rows[len(rows) // 2]
    assert r + 1 in rows
    rep = LP.row_report(name, LP.move_row(ref, name, r)[name], ref[name])
    assert rep["missing"] == [r] and not rep["extra"]
    assert rep["worst"][0] in (r, r + 1) and rep["worst"][1] >= MARGIN * LP.ROW_BARS["eval"]["tmp"], rep["worst"]
    word = "word_embeddings/word_embeddings"
    mlm = case["ref"]["mlm"]
    moved = LP.move_row(mlm, word, 500)
    assert LP.rel(moved[word], mlm[word]) < LP.SUMMED_STEP_BAR  # invisible to a whole-tensor bar ...
    wrep = LP.row_report(word, moved[word], mlm[word])
    assert wrep["missing"] == [500] and wrep["worst"][1] >= MARGIN * LP.ROW_BARS["eval"]["mlm"]  # ... not to the rows
