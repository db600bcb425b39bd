"""CPU tests of the VCR input and validator host side: the record parser against a NumPy restatement of both reference
parsers (empty ctx or choice, texts truncated past 184 / 134, another `draw`), the label rule, missing images, the prompts
against the golden fixture, the training resize plan, shuffle and shard determinism, the checkpoint follower under an
injected clock, and the results / predictions files."""
import json
import os

import numpy as np
import pytest

from merlot_b200 import vcr_input as VI
from merlot_b200 import vcr_validate as VV
from merlot_b200.dataloader import shard_files, shuffled_records
from merlot_b200.tfrecord import parse_example, read_records
from tests import input_oracle as IO
from tests import story_records as SR
from tests import vcr_records as R


def _joint(q, draw="segm"):
    return VI.parse_question(parse_example(R.vcr_example(q)), VI.MODES, draw, {m: 184 for m in VI.MODES})


def _eval(q, mode, draw="segm"):
    return VI.parse_question(parse_example(R.vcr_example(q)), (mode,), draw, VI.EVAL_MAX_NUM_TOKENS)


def _cases():
    """Questions covering an empty ctx, an empty choice, absent lists, and texts past 134 and past 184 tokens."""
    rng = np.random.default_rng(7)
    qs = [R.question(rng, k) for k in range(4)]
    qs[0]["answer/ctx"] = []
    qs[0]["rationale/choice_2"] = []
    qs[1]["answer/ctx"] = None
    qs[1]["rationale/choice_0"] = None
    qs[2]["answer/ctx"] = list(range(1000, 1140))   # 4 + 140 + choice + 1 > 134 and, for the longest choices, > 184
    qs[2]["rationale/ctx"] = list(range(2000, 2200))  # > 184 on its own
    qs[3]["answer/choice_3"] = list(range(3000, 3125))  # 4 + ctx + 125 + 1: the END falls past 134
    return qs


def test_prompts_match_golden_fixture():
    assert {m: list(p) for m, p in VI.VCR_PROMPT.items()} == R.prompts()
    assert R.golden()["specials"] == {"START": VI.START, "END": VI.END} == {"START": R.START, "END": R.END}
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_facts.json")) as f:
        facts = json.load(f)["tokenizer"]
    assert facts["encode"][" answer question:"] == R.golden()["encode"][" answer question:"]  # the two fixtures agree
    assert facts["specials"]["START"] == VI.START and facts["specials"]["PADDING"] == VI.PADDING


def test_joint_parse_matches_restatement():
    for q in _cases():
        got = _joint(q)
        lm, labels = R.joint_np(q)
        assert got["lm_input"].dtype == np.int32 and got["lm_input"].shape == (2, 4, 184)
        np.testing.assert_array_equal(got["lm_input"], lm)
        np.testing.assert_array_equal(got["labels"], labels)
        assert (got["img_id"], got["annot_id"]) == (q["img_id"], q["annot_id"])
        assert got["jpegs"] == [q["answer/segm/image"], q["rationale/segm/image"]]
    long = _joint(_cases()[2])["lm_input"][1]
    assert (long != 0).all() and (long != VI.END).all()  # cut at 184: no padding, and the END is lost


@pytest.mark.parametrize("mode", ["answer", "rationale"])
def test_eval_parse_matches_restatement(mode):
    L = {"answer": 134, "rationale": 184}[mode]
    for q in _cases():
        got = _eval(q, mode)
        lm, label = R.eval_np(q, mode)
        assert got["lm_input"].shape == (1, 4, L)
        np.testing.assert_array_equal(got["lm_input"][0], lm)
        assert list(got["labels"]) == [label] and got["jpegs"] == [q[f"{mode}/segm/image"]]
    cut = _eval(_cases()[3], "answer")["lm_input"][0, 3]
    assert (cut != 0).all() and cut[-1] != VI.END  # the 134-token answer input drops the END of a long choice


def test_other_draw_reads_its_own_images():
    q = R.question(np.random.default_rng(1), 0, draws=("segm", "bbox"))
    got = _joint(q, draw="bbox")
    assert got["jpegs"] == [q["answer/bbox/image"], q["rationale/bbox/image"]]
    assert _eval(q, "rationale", draw="bbox")["jpegs"] == [q["rationale/bbox/image"]]
    assert _joint(q, draw="nodraw")["jpegs"] == [b"", b""]


def test_tags_are_not_read():
    q = R.question(np.random.default_rng(2), 0)
    bare = dict(q)
    for k in list(bare):
        if "_tags" in k:
            bare[k] = None
    a, b = _joint(q), _joint(bare)
    np.testing.assert_array_equal(a["lm_input"], b["lm_input"])


@pytest.mark.parametrize("value", [None, -1, 4])
def test_label_outside_range_raises_naming_annot_id(value):
    q = R.question(np.random.default_rng(3), 12)
    q["label/rationale_label"] = value
    p = _joint(q)
    assert p["labels"][1] == (-1 if value is None else value)
    with pytest.raises(ValueError, match=r"annot_id='val-12': label/rationale_label is %d" % (-1 if value is None else value)):
        VI.check_labels([_joint(R.question(np.random.default_rng(4), 11)), p], VI.MODES)
    VI.check_labels([_eval(q, "answer")], ("answer",))  # the answer label alone is fine


def test_missing_or_broken_image_raises_naming_annot_id():
    q = R.question(np.random.default_rng(5), 21)
    q["rationale/segm/image"] = None
    p = _joint(q)
    assert VI.decode_image(p, 0, "answer").shape[2] == 3
    with pytest.raises(ValueError, match="annot_id='val-21': the rationale image is missing"):
        VI.decode_image(p, 1, "rationale")
    q["rationale/segm/image"] = b"\xff\xd8 not a jpeg"
    with pytest.raises(ValueError, match="annot_id='val-21': the rationale image cannot be decoded"):
        VI.decode_image(_joint(q), 1, "rationale")


@pytest.mark.parametrize("out", [(384, 704), (48, 64)])
def test_train_plan_matches_float32_restatement(out):
    hw = np.concatenate([np.array(R.SIZES), np.random.default_rng(0).integers(1, 1500, (200, 2))])
    got = VI.train_plan(np.random.default_rng([5, 1]), hw, out)
    rng = np.random.default_rng([5, 1])  # the same draws, in the same order
    f32 = np.float32
    scale = f32(0.9) + rng.random(len(hw), dtype=f32) * (f32(1.1) - f32(0.9))
    u_y, u_x = rng.random(len(hw), dtype=f32), rng.random(len(hw), dtype=f32)
    assert (scale >= 0.9).all() and (scale < 1.1).all()
    for k, (h, w) in enumerate(hw):
        want = IO.resize_plan(h, w, out, scale[k], u_y[k], u_x[k])
        assert tuple(int(got[n][k]) for n in ("scaled_h", "scaled_w", "offset_y", "offset_x")) == want, (h, w)
    assert min(got["scaled_h"].min(), got["scaled_w"].min()) >= 63  # the 64-pixel floor (a float32 product, truncated)


def test_eval_plan_is_the_story_plan():
    hw = np.array(R.SIZES)
    got = VI.plan_frames_eval(hw[:, 0], hw[:, 1], (48, 64))
    for k, (h, w) in enumerate(hw):
        assert tuple(int(got[n][k]) for n in ("scaled_h", "scaled_w", "offset_y", "offset_x")) == SR.eval_plan(h, w, (48, 64))


def test_shuffle_and_shard_determinism(tmp_path):
    R.write_questions(tmp_path, [3, 4, 2, 5], max_ctx=2, max_choice=2, sizes=[(8, 8)])
    files = sorted(str(p) for p in tmp_path.glob("vcr-*.tfrecord"))
    every = {r for f in files for r in read_records(f)}

    def take(seed, rank, world, n=40):
        shard = shard_files(files, rank, world)
        recs = shuffled_records(shard, np.random.default_rng([seed, rank]), min(2, len(shard)), 4)
        return [next(recs) for _ in range(n)]
    assert take(0, 0, 1) == take(0, 0, 1)
    assert take(0, 0, 1) != take(1, 0, 1)
    assert set(take(0, 0, 1, 200)) == every  # repeated forever: every record comes back
    r0, r1 = take(3, 0, 2), take(3, 1, 2)
    assert r0 == take(3, 0, 2) and r1 == take(3, 1, 2)
    in0 = {r for f in files[0::2] for r in read_records(f)}
    assert set(r0) <= in0 and not set(r1) & in0  # rank r reads files r, r + world, ...


class _Clock:
    """A fake clock whose sleep advances time and lets the test add checkpoints at given times."""

    def __init__(self, events):
        self.t, self.events, self.sleeps = 0.0, sorted(events, key=lambda e: e[0]), 0

    def __call__(self):
        return self.t

    def sleep(self, s):
        self.sleeps += 1
        self.t += s
        while self.events and self.events[0][0] <= self.t:
            self.events.pop(0)[1]()


def _save(out, step):
    from merlot_b200.tf_checkpoint import update_checkpoint_state
    out.mkdir(exist_ok=True)
    (out / f"model.ckpt-{step}.index").write_bytes(b"")
    update_checkpoint_state(str(out), str(out / f"model.ckpt-{step}"))


def test_follow_checkpoints_visits_new_checkpoints_in_order_and_stops(tmp_path):
    out = tmp_path / "out"
    _save(out, 2)
    _save(out, 4)
    clk = _Clock([(1030, lambda: _save(out, 6)), (1030, lambda: _save(out, 8)), (1090, lambda: _save(out, 10)),
                  (1095, lambda: _save(out, 12))])
    seen = []
    for p in VV.follow_checkpoints(str(out), 10, timeout=100, poll_interval=10, clock=clk, sleep=clk.sleep):
        seen.append(VV.checkpoint_step(p))
        if seen[-1] == 4:
            clk.t += 1000  # an evaluation longer than the timeout does not count against it
    assert seen == [2, 4, 6, 8, 10]  # oldest first, each once, and nothing after num_train_steps
    assert clk.t == 1090


def test_follow_checkpoints_times_out(tmp_path):
    out = tmp_path / "out"
    clk = _Clock([(20, lambda: _save(out, 3))])
    seen = [VV.checkpoint_step(p) for p in VV.follow_checkpoints(str(out), 100, timeout=50, poll_interval=7, clock=clk,
                                                                    sleep=clk.sleep)]
    assert seen == [3] and 21 + 50 <= clk.t < 21 + 50 + 7  # no checkpoint within 50 s of the last one
    clk = _Clock([])
    assert list(VV.follow_checkpoints(str(tmp_path / "none"), 1, timeout=5, poll_interval=2, clock=clk, sleep=clk.sleep)) == []
    assert clk.t == 6


def test_deleted_checkpoint_is_skipped(tmp_path):
    out = tmp_path / "out"
    for s in (1, 2, 3):
        _save(out, s)
    (out / "model.ckpt-2.index").unlink()
    clk = _Clock([])
    seen = [VV.checkpoint_step(p) for p in VV.follow_checkpoints(str(out), 3, 5, 1, clk, clk.sleep)]
    assert seen == [1, 3]


def test_results_jsonl_and_predictions_npz(tmp_path):
    res = {"global_step": 6, "avg": 0.375, "loss": 1.25, "questions": 8, "predictions": None}
    path = VV.append_result(str(tmp_path), res)
    VV.append_result(str(tmp_path), dict(res, global_step=8, avg=0.5))
    assert path == str(tmp_path / "eval" / "results.jsonl")
    lines = [json.loads(x) for x in open(path).read().splitlines()]
    assert lines == [{"global_step": 6, "avg": 0.375, "loss": 1.25, "questions": 8},
                     {"global_step": 8, "avg": 0.5, "loss": 1.25, "questions": 8}]
    logits = np.random.default_rng(0).normal(0, 3, (5, 4)).astype(np.float32)
    lp = VV.log_softmax(logits)
    for i in range(5):
        x = logits[i].astype(np.float64)
        np.testing.assert_allclose(lp[i], x - np.log(np.exp(x).sum()), rtol=0, atol=1e-6)
    preds = {"annot_id": np.array(["val-1", "val-22"]), "img_id": np.array(["a.jpg", "b.jpg"]), "log_prob": lp[:2],
             "prediction": lp[:2].argmax(-1), "label": np.array([1, -1])}
    VV.write_predictions(str(tmp_path / "p.npz"), preds)
    with np.load(tmp_path / "p.npz") as z:  # no pickled objects
        assert sorted(z.files) == ["annot_id", "img_id", "label", "log_prob", "prediction"]
        for k in preds:
            np.testing.assert_array_equal(z[k], preds[k])


@pytest.mark.parametrize("args,match", [(["--predictions", "p.npz"], "--checkpoint"),
                                        (["--checkpoint", "x", "--predictions", "p.txt"], ".npz"),
                                        (["--unlabelled"], "--predictions"),
                                        (["--chunk", "-1"], "--chunk")])
def test_validator_argument_checks(tmp_path, args, match):
    with pytest.raises(ValueError, match=match):
        VV.main([str(tmp_path / "none.yaml")] + args)  # raised before the config is read


def test_placeholder_train_file_matches_nothing():
    from merlot_b200.config import NeatConfig
    from merlot_b200.dataloader import train_files
    cfg = NeatConfig.from_dict({"data": {"train_file": "TRAIN_FILE_PATH", "val_file": ""}, "model": {}, "optimizer": {},
                                "device": {"output_dir": "/tmp/x"}})
    assert train_files(cfg.data) == []
    with pytest.raises(ValueError, match="matches no file"):
        VI.input_fn_builder(cfg, is_training=True)
    with pytest.raises(ValueError, match="matches no file"):
        VI.input_fn_builder(cfg, is_training=False)
