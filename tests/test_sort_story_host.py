"""CPU tests of zero-shot story unshuffling's host side (downstream/sort_story): the story-record parser against a NumPy
restatement, errors naming the story, the evaluation resize plan, record order and the dropped remainder, the story-major
layout of a batch, score_file, and MerlotModel's frame_copies argument checks."""
import numpy as np
import pytest
import torch

from merlot_b200 import sort_story as S
from merlot_b200.dataloader import interleave_records
from merlot_b200.tfrecord import parse_example, read_records
from tests import story_records as R


def _parsed(s, **kw):
    return S.parse_story(parse_example(R.story_example(s, **kw)))


def test_parser_matches_numpy_restatement():
    rng = np.random.default_rng(3)
    for k in range(6):  # sentences of 0..59 ids: padded, and truncated past 32 tokens
        s = R.story(rng, 100 + k, max_sentence=60, drop_sentence=k if k < 5 else None)
        got = _parsed(s)
        assert (got["story_id"], got["permutation_identity_encode"]) == (100 + k, s["permutation_identity_encode"])
        assert got["sentences"].dtype == np.int32 and got["sentences"].shape == (5, 32)
        np.testing.assert_array_equal(got["sentences"], R.sentences_np(s["sentences"]))
        assert got["frames"] == s["frames"]
    long = R.story(rng, 7)
    long["sentences"][2] = list(range(100, 140))
    np.testing.assert_array_equal(_parsed(long)["sentences"][2], np.array([2] + list(range(100, 131)), np.int32))


def test_parser_defaults():
    s = R.story(np.random.default_rng(0), 5)
    s["sentences"] = [None] * 5
    s["frames"][3] = None
    got = _parsed(s, with_ids=False)
    assert got["story_id"] == -1 and got["permutation_identity_encode"] == -1  # FixedLenFeature default_value=-1
    np.testing.assert_array_equal(got["sentences"][:, 0], 2)
    assert not got["sentences"][:, 1:].any()
    assert got["frames"][3] == b""


def test_missing_or_broken_image_raises_with_story_id():
    s = R.story(np.random.default_rng(1), 41)
    s["frames"][2] = None
    p = _parsed(s)
    assert S.decode_frame(p, 0).shape[2] == 3
    with pytest.raises(ValueError, match="story 41: image 2 is missing"):
        S.decode_frame(p, 2)
    s["frames"][2] = b"\xff\xd8 not a jpeg"
    with pytest.raises(ValueError, match="story 41: image 2 cannot be decoded"):
        S.decode_frame(_parsed(s), 2)


def test_grayscale_frame_decodes_to_rgb():
    p = _parsed(R.story(np.random.default_rng(2), 3, gray_frame=1))
    f = S.decode_frame(p, 1)
    assert f.dtype == np.uint8 and f.shape[2] == 3 and (f[..., 0] == f[..., 1]).all() and (f[..., 1] == f[..., 2]).all()


@pytest.mark.parametrize("desired", [(384, 384), (32, 48), (192, 352)])
def test_plan_frames_eval_matches_float32_restatement(desired):
    rng = np.random.default_rng(11)
    hw = np.concatenate([np.array(R.SIZES), rng.integers(1, 2000, (300, 2))])
    got = S.plan_frames_eval(hw[:, 0], hw[:, 1], desired)
    for k, (h, w) in enumerate(hw):
        assert (got["scaled_h"][k], got["scaled_w"][k], got["offset_y"][k], got["offset_x"][k]) == R.eval_plan(h, w, desired), (h, w)


def test_plan_frames_eval_kats():
    def one(h, w, d):
        p = S.plan_frames_eval([h], [w], d)
        return tuple(int(p[k][0]) for k in ("scaled_h", "scaled_w", "offset_y", "offset_x"))
    assert one(384, 384, (384, 384)) == (384, 384, 0, 0)  # exact size: the identity plan
    assert one(200, 400, (384, 384)) == (192, 384, 0, 0)  # 2:1 fills the width, pads 192 rows at the bottom
    assert one(20, 900, (384, 384)) == (8, 384, 0, 0)     # no 64-pixel floor, unlike the training branch
    assert one(3, 5000, (384, 384)) == (0, 384, 0, 0)     # truncates to 0: eval_frame_plan rejects it


def test_eval_frame_plan_rejects_empty_frame():
    hw = np.array([[48, 48]] * 5 + [[48, 48], [3, 5000], [48, 48], [48, 48], [48, 48]])
    with pytest.raises(ValueError, match="story 9: image 1 of 3x5000"):
        S.eval_frame_plan(hw, [8, 9], (384, 384))
    plan = S.eval_frame_plan(hw[:5], [8], (384, 384))
    assert (plan["method"] == 0).all() and (plan["augment"] == 0).all() and (plan["factor"] == 1).all()


@pytest.mark.parametrize("counts,b", [([5, 3, 4], 4), ([7], 3), ([2, 2], 2), ([1, 6, 2, 3], 5)])
def test_record_order_and_remainder(tmp_path, counts, b):
    R.write_stories(tmp_path, counts, max_sentence=4, sizes=[(8, 8)])
    files = sorted(str(p) for p in tmp_path.glob("val-*.tfrecord"))
    cycle = min(2, len(files))
    order = []  # the interleave restated: two open files, one record each in turn, an ended file replaced by the next
    queues = [list(read_records(f)) for f in files]
    open_, nxt = list(range(cycle)), cycle
    while open_:
        f = open_.pop(0)
        if queues[f]:
            order.append(queues[f].pop(0))
            open_.append(f)
        elif nxt < len(files):
            open_.append(nxt)
            nxt += 1
    for _ in range(2):  # deterministic: the same order twice
        tail = []
        got = list(S.batch_records(interleave_records(iter(files), cycle, files), b, tail))
        assert [r for batch in got for r in batch] == order[:len(got) * b]
        assert all(len(batch) == b for batch in got)
        assert len(tail) == sum(counts) % b and tail == order[len(got) * b:]


def test_val_files_sorted(tmp_path):
    R.write_stories(tmp_path, [1, 1, 1], max_sentence=2, sizes=[(8, 8)])
    from merlot_b200.config import NeatConfig
    cfg = NeatConfig.from_dict({"data": {"val_file": str(tmp_path / "val-*.tfrecord")}, "model": {}, "optimizer": {},
                                "device": {"output_dir": str(tmp_path)}})
    assert S.val_files(cfg) == sorted(str(p) for p in tmp_path.glob("val-*.tfrecord"))


def test_story_major_layout_and_shuffle_indices():
    sents = torch.arange(3 * 5 * 32, dtype=torch.int32).reshape(3, 5, 32)
    ids, shuf = S.tiled_inputs(sents, 2, seed=9)
    assert ids.shape == (6, 5, 32) and shuf.shape == (30,) and shuf.dtype == torch.int32
    for s in range(3):
        for d in range(2):
            assert torch.equal(ids[s * 2 + d], sents[s])  # row s*dup + d is copy d of story s
    np.testing.assert_array_equal(shuf.numpy(), S.fixed_shuffle_index(6, 5, 9).reshape(-1))
    rows = shuf.numpy().reshape(6, 5) - 64
    assert all(sorted(r) == list(range(5)) for r in rows)
    assert any((rows[2 * s] != rows[2 * s + 1]).any() for s in range(3))  # the copies of a story see different orders


def test_score_file_npz_equals_evaluate(tmp_path):
    rng = np.random.default_rng(4)
    preds = []
    for sid in [12, 3, 100, 7, 25]:
        p = rng.uniform(0.05, 1.0, (5, 5, 3)).astype(np.float32)
        p /= p.sum(-1, keepdims=True)
        preds.append({"story_id": sid, "permutation_identity_encode": np.int64(sid % 7), "sentences": np.zeros((5, 32), np.int32),
                      "lang_viz_probs": p, "viz_viz_probs": p[::-1].copy()})
    path = str(tmp_path / "logits_val.npz")
    assert S.write_logits_npz(path, preds) == 5
    got = S.score_file(path)
    order = sorted(range(5), key=lambda i: preds[i]["story_id"])  # sorted integer story ids, like the reference
    ref = S.evaluate([preds[i]["lang_viz_probs"] for i in order])
    assert got == ref


def test_h5_output_needs_h5py(tmp_path):
    try:
        import h5py  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match="h5py"):
            S.main([str(tmp_path / "none.yaml"), "--out", str(tmp_path / "x.h5")])  # raised before the config is read
        return
    pytest.skip("h5py is installed: the HDF5 writer itself is exercised by the GPU driver test")


def test_bad_output_extension_raises(tmp_path):
    with pytest.raises(ValueError, match=".h5 or .npz"):
        S.main([str(tmp_path / "none.yaml"), "--out", str(tmp_path / "x.txt")])


@pytest.mark.parametrize("kw", [dict(is_training=True), dict(mask_input=True), dict(save_for_backward=True),
                                dict(num_texts=4), dict(frame_copies=0)])
def test_frame_copies_argument_checks(tiny_cfg, kw):
    from merlot_b200.modeling import MerlotModel
    cfg = dict(tiny_cfg)
    if "num_texts" in kw:
        cfg["num_texts"] = kw.pop("num_texts")
    args = dict(is_training=False, mask_input=False, frame_copies=2)
    args.update(kw)
    img, ids = torch.zeros(4, 32, 32, 3), torch.zeros(4, 2, 8, dtype=torch.int32)
    with pytest.raises(ValueError if args["frame_copies"] < 1 else NotImplementedError, match="frame_copies"):
        MerlotModel(cfg, use_tpu=False, image=img, input_ids=ids, params=None, **args)
