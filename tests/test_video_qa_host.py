"""CPU tests of open-ended video QA (downstream.task: video_qa) on the host: the record parser against a NumPy restatement
(texts, padding, truncation, answers -1 / absent / out of range in labelled and unlabelled runs, record errors), the config
errors, the parameter arena of ParamStore(task="video_qa") (entries, ref_cols, zero output bias, zero padding columns,
to_tf_dict shapes, a pretraining checkpoint), the training input's skipping and counting of out-of-vocabulary questions,
the step dispatch, and the validator's results-line arithmetic and predictions."""
import json

import numpy as np
import pytest
import torch

from merlot_b200 import video_qa as VQ
from merlot_b200 import video_qa_input as QI
from merlot_b200 import video_qa_validate as QV
from merlot_b200.tfrecord import parse_example
from tests.test_gpu_video_qa import example, question, text_np
from tests.test_video_mc_host import _tiny

F, L, VOCAB, A = 3, 40, 1000, 13


def _parse(q, num_frames=F, max_len=L):
    return QI.parse_question(parse_example(example(q)), num_frames, max_len, VOCAB)


def _q(k=0, seed=0, **kw):
    return question(np.random.default_rng(seed), k, F, A, **kw)


def test_texts_padding_and_truncation_match_restatement():
    rng = np.random.default_rng(1)
    qs = [question(rng, k, F, A) for k in range(5)]
    qs[0]["question"] = []
    qs[1]["question"] = None  # absent: an empty question
    qs[2]["question"] = list(range(100, 150))  # 1 + 50 + 1 > 40: truncated, the END lost
    for q in qs:
        got = _parse(q)
        assert got["lm_input"].dtype == np.int32 and got["lm_input"].shape == (L,)
        np.testing.assert_array_equal(got["lm_input"], text_np(q, L))
        assert got["id"] == q["id"] and got["answer"] == q["answer"] and got["jpegs"] == q["frames"]
    long = _parse(qs[2])["lm_input"]
    assert long[-1] != 0 and QI.END not in long.tolist() and long[0] == QI.START
    assert _parse(qs[0])["lm_input"][:3].tolist() == [QI.START, QI.END, QI.PADDING]


def test_answer_rules_labelled_and_unlabelled():
    q = _q(4)
    good, oov, absent = _parse(q), _parse(dict(q, answer=-1)), _parse(dict(q, answer=None))
    QI.check_answers([good, oov], A)  # -1 is a valid label: an answer outside the vocabulary
    assert QI.labels([good, oov, absent]).tolist() == [q["answer"], -1, -1]
    assert QI.labels([good]).dtype == np.int32
    with pytest.raises(ValueError, match=r"id='q-4': answer is missing"):
        QI.check_answers([good, absent], A)
    for bad in (-2, -7, A, 500):
        p = _parse(dict(q, id="q-bad", answer=bad))
        with pytest.raises(ValueError, match=r"id='q-bad': answer is %d, outside \[-1, 13\)" % bad):
            QI.check_answers([good, p], A)
    with pytest.raises(ValueError, match=r"id='q-4': answer has 2 values"):
        _parse_two_answers(q)


def _parse_two_answers(q):
    from tests import tfrecord_writer as W
    feats = {"id": ("bytes", [q["id"].encode()]), "frames/encoded": ("bytes", list(q["frames"])),
             "question": ("int64", q["question"]), "answer": ("int64", [1, 2])}
    return QI.parse_question(parse_example(W.example(feats)), F, L, VOCAB)


class _Fields(QI._QA):
    """The batch-field methods of the video_qa pipelines without a device pipeline."""

    def __init__(self, labelled):
        self.labelled, self.num_answers = labelled, A


def test_batch_fields_labelled_and_unlabelled():
    qs = [_parse(_q(k)) for k in range(3)] + [_parse(dict(_q(3), answer=-1))]
    f = _Fields(True)._text_fields(qs)
    assert f["lm_input"].shape == (4, L) and f["lm_input"].dtype == np.int32
    assert f["lm_targets"].tolist() == [q["answer"] for q in qs] and f["lm_targets"][3] == -1
    unl = [_parse(dict(_q(k), answer=None)) for k in range(2)]
    with pytest.raises(ValueError, match="answer is missing"):
        _Fields(True)._text_fields(unl)
    assert _Fields(False)._text_fields(unl)["lm_targets"].tolist() == [-1, -1]
    with pytest.raises(ValueError, match=r"answer is 13, outside"):
        _Fields(True)._text_fields([_parse(dict(_q(5), answer=A))])
    _Fields(False)._text_fields([_parse(dict(_q(5), answer=A))])  # unlabelled runs do not read answers


@pytest.mark.parametrize("case,match", [
    ("no_frames", r"video_qa record id='q-7': 0 frames, expected 1 to 3"),
    ("too_many_frames", r"id='q-7': 4 frames, expected 1 to 3"),
    ("token_too_large", r"id='q-7': question holds token id 1000 outside the vocabulary \[0, 1000\)"),
    ("negative_token", r"id='q-7': question holds token id -5 outside the vocabulary"),
])
def test_record_errors_name_the_id(case, match):
    q = _q(7)
    if case == "no_frames":
        q["frames"] = None
    elif case == "too_many_frames":
        q["frames"] = q["frames"][:1] * (F + 1)
    elif case == "token_too_large":
        q["question"] = [5, VOCAB]
    else:
        q["question"] = [10, -5]
    with pytest.raises(ValueError, match=match):
        _parse(q)


def test_training_input_skips_and_counts_oov_questions():
    qs = [dict(_q(k), answer=(-1 if k in (1, 2, 6) else k % A)) for k in range(10)]
    records = iter([example(q) for q in qs])
    parse = lambda r: QI.parse_question(parse_example(r), F, L, VOCAB)  # noqa: E731
    recs, got, skipped = QI.take_answerable(records, 3, parse, A)
    assert [q["id"] for q in got] == ["q-0", "q-3", "q-4"] and skipped == 2 and len(recs) == 3
    recs, got, skipped = QI.take_answerable(records, 3, parse, A)
    assert [q["id"] for q in got] == ["q-5", "q-7", "q-8"] and skipped == 1
    bad = iter([example(dict(_q(0), answer=A))])
    with pytest.raises(ValueError, match=r"id='q-0': answer is 13"):
        QI.take_answerable(bad, 1, parse, A)


@pytest.mark.parametrize("model,downstream,match", [
    (dict(num_imgs=0), {"num_answers": 10}, "num_imgs .* got 0"),
    (dict(num_imgs=2, num_texts=4), {"num_answers": 10}, "num_texts must be 1.* got 4"),
    (dict(num_imgs=2), {}, "num_answers .* missing, got None"),
    (dict(num_imgs=2), {"num_answers": 1}, "num_answers must be >= 2, got 1"),
])
def test_config_errors(model, downstream, match):
    cfg = _tiny(**model)
    with pytest.raises(ValueError, match=match):
        VQ.check_config(cfg, downstream)
    from merlot_b200.config import NeatConfig
    with pytest.raises(ValueError, match=match):
        VQ.video_qa_model_fn_builder(NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {},
                                                          "device": {"output_dir": "/tmp/merlot_video_qa"},
                                                          "downstream": dict(downstream, task="video_qa")}), device="cpu")


def test_config_accepts_one_text():
    assert VQ.check_config(_tiny(num_imgs=6, num_texts=1), {"num_answers": 1500}) == (6, 1500)
    assert VQ.check_config(_tiny(num_imgs=1), {"num_answers": 2}) == (1, 2)


@pytest.mark.parametrize("num_answers,stored", [(13, 16), (16, 16), (1500, 1504), (2, 8)])
def test_video_qa_store_entries_padding_and_round_trip(num_answers, stored):
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F)
    vcr = ParamStore(cfg, device="cpu", task="vcr", with_optimizer_state=False)
    st = ParamStore(cfg, device="cpu", task="video_qa", num_answers=num_answers, with_optimizer_state=False)
    tower = sorted(n for n in st.entries if n.startswith("qa_cls/"))
    assert tower == ["qa_cls/classifier_mlp0/bias", "qa_cls/classifier_mlp0/kernel", "qa_cls/classifier_mlp1/bias",
                     "qa_cls/classifier_mlp1/kernel"]
    model = {n: e.shape for n, e in vcr.entries.items() if not n.startswith(("answer_cls/", "rationale_cls/"))}
    assert {n: e.shape for n, e in st.entries.items() if not n.startswith("qa_cls/")} == model
    e0, k1, b1 = (st.entries[f"qa_cls/{n}"] for n in ("classifier_mlp0/kernel", "classifier_mlp1/kernel", "classifier_mlp1/bias"))
    assert e0.shape == (128, 64) and e0.ref_cols == 0
    assert k1.shape == (64, stored) and b1.shape == (stored,) and k1.ref_cols == b1.ref_cols == num_answers
    shapes = {k: tuple(v.shape) for k, v in st.to_tf_dict().items()}
    assert shapes["qa_cls/classifier_mlp1/kernel"] == (64, num_answers) and shapes["qa_cls/classifier_mlp1/bias"] == (num_answers,)
    assert shapes["qa_cls/classifier_mlp0/kernel"] == (128, 64) and shapes["qa_cls/classifier_mlp0/bias"] == (64,)
    vcr_names = {k for k in vcr.to_tf_dict() if not k.startswith(("answer_cls/", "rationale_cls/"))}
    assert set(shapes) == vcr_names | {f"qa_cls/{n}" for n in ("classifier_mlp0/kernel", "classifier_mlp0/bias",
                                                                "classifier_mlp1/kernel", "classifier_mlp1/bias")}
    st.init_reference(seed=0)
    assert float(st.P("qa_cls/classifier_mlp1/bias").abs().max()) == 0.0  # no answer is favoured
    kern = st.P("qa_cls/classifier_mlp1/kernel")
    assert kern[:, num_answers:].count_nonzero() == 0
    assert float(kern[:, :num_answers].abs().max()) > 0
    g = torch.Generator().manual_seed(1)
    d = {k: torch.randn(v.shape, generator=g) for k, v in st.to_tf_dict().items()}
    st.load_tf_dict(d)
    back = st.to_tf_dict()
    for k in d:
        assert torch.equal(back[k], d[k]), k
    if stored > num_answers:
        assert float(st.P("qa_cls/classifier_mlp1/kernel")[:, num_answers:].abs().max()) == 0.0
        assert float(st.P("qa_cls/classifier_mlp1/bias")[num_answers:].abs().max()) == 0.0
    assert st.num_params() == vcr.num_params() - 2 * (128 * 64 + 64 + 64 + 1) + (128 * 64 + 64 + 64 * num_answers + num_answers)


def test_other_towers_keep_their_output_bias():
    from merlot_b200.params import VCR_BIAS_PI, ParamStore
    cfg = _tiny(num_imgs=F, num_texts=4)
    for task in ("vcr", "video_mc"):
        st = ParamStore(cfg, device="cpu", task=task, with_optimizer_state=False)
        st.init_reference(seed=0)
        for n in st.entries:
            if n.endswith("_cls/classifier_mlp1/bias"):
                assert float(st.P(n)[0]) == pytest.approx(-np.log((1 - VCR_BIAS_PI) / VCR_BIAS_PI))


def test_store_needs_num_answers_exactly_for_video_qa():
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F)
    with pytest.raises(ValueError, match="num_answers"):
        ParamStore(cfg, device="cpu", task="video_qa", with_optimizer_state=False)
    with pytest.raises(ValueError, match="num_answers"):
        ParamStore(cfg, device="cpu", task="vcr", num_answers=10, with_optimizer_state=False)
    with pytest.raises(ValueError, match="num_answers must be >= 2, got 1"):
        ParamStore(cfg, device="cpu", task="video_qa", num_answers=1, with_optimizer_state=False)


def test_pretraining_checkpoint_leaves_the_tower_missing():
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F)
    pre = ParamStore(cfg, device="cpu", task="pretrain", with_optimizer_state=False).to_tf_dict()
    st = ParamStore(cfg, device="cpu", task="video_qa", num_answers=A, with_optimizer_state=False)
    st.init_reference(seed=0)
    before = st.P("qa_cls/classifier_mlp1/kernel").clone()
    missing = st.load_tf_dict(pre, strict=False)
    assert sorted(missing) == ["qa_cls/classifier_mlp0/bias", "qa_cls/classifier_mlp0/kernel", "qa_cls/classifier_mlp1/bias",
                               "qa_cls/classifier_mlp1/kernel"]
    assert torch.equal(st.P("qa_cls/classifier_mlp1/kernel"), before)


def test_store_of_another_task_or_size_is_refused():
    from merlot_b200.config import NeatConfig
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F)
    config = NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {"learning_rate": 1e-4},
                                   "device": {"output_dir": "/tmp/merlot_video_qa"},
                                   "downstream": {"task": "video_qa", "num_answers": A}})
    for task in ("video_mc", "pretrain"):
        with pytest.raises(ValueError, match=f"ParamStore\\(task='video_qa'\\), got task='{task}'"):
            VQ.video_qa_model_fn_builder(config, store=ParamStore(cfg, device="cpu", task=task), device="cpu")
    with pytest.raises(ValueError, match="holds 20 answers, downstream.num_answers is 13"):
        VQ.video_qa_model_fn_builder(config, store=ParamStore(cfg, device="cpu", task="video_qa", num_answers=20),
                                     device="cpu")


def test_synthetic_batch_and_dispatch():
    from merlot_b200 import train
    from merlot_b200.config import NeatConfig
    from merlot_b200.params import ParamStore
    cfg = NeatConfig.from_dict({"data": {}, "model": _tiny(num_imgs=F, image_size=[32, 48]), "optimizer": {},
                                "device": {"output_dir": "/tmp/merlot_video_qa"},
                                "downstream": {"task": "video_qa", "max_text_len": 24, "num_answers": A}})
    f = train.synthetic_video_qa_batch(cfg, 4, seed=1, device="cpu")
    assert f["images"].shape == (4 * F, 32, 48, 3) and f["images"].dtype == torch.bfloat16
    assert f["lm_input"].shape == (4, 24) and f["lm_targets"].shape == (4,) and f["img_mask"].shape == (4, F)
    assert ((f["lm_targets"] >= 0) & (f["lm_targets"] < A)).all() and (f["lm_input"][:, 0] == 2).all()
    assert train._step_for(cfg) == (VQ.video_qa_model_fn_builder, train.synthetic_video_qa_batch)
    st = ParamStore(cfg.model, device="cpu", task="video_qa", num_answers=A, with_optimizer_state=False)
    assert train.variables_without_gradient(cfg.model, st) == []


def test_predict_and_pretrain_validate_refuse_video_qa(tmp_path):
    import yaml
    from merlot_b200 import predict, pretrain_validate
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump({"data": {}, "model": {}, "optimizer": {}, "device": {"output_dir": str(tmp_path)},
                                    "downstream": {"task": "video_qa"}}))
    with pytest.raises(ValueError, match="'video_qa'"):
        predict.main([str(path), "--out", str(tmp_path / "o")])
    with pytest.raises(ValueError, match="video_qa fine-tuning with merlot_b200.video_qa_validate"):
        pretrain_validate.main([str(path)])


def test_validator_needs_the_video_qa_task(tmp_path):
    import yaml
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump({"data": {}, "model": {}, "optimizer": {}, "device": {"output_dir": str(tmp_path)},
                                    "downstream": {"task": "video_mc"}}))
    with pytest.raises(ValueError, match="video_qa validation needs 'video_qa'"):
        QV.main([str(path)])


@pytest.mark.parametrize("args,match", [(["--predictions", "p.npz"], "--checkpoint"), (["--unlabelled"], "--predictions"),
                                        (["--chunk", "-1"], "--chunk")])
def test_validator_argument_checks(tmp_path, args, match):
    with pytest.raises(ValueError, match=match):
        QV.main([str(tmp_path / "none.yaml")] + args)


def _chunks(per_row_ce, target, correct, chunk):
    """The per-chunk (loss_sum, in_vocab, correct) a validator collects, as fp32 values, for chunks of `chunk` rows."""
    out = {"loss_sum": [], "in_vocab": [], "correct": []}
    w = (target >= 0).astype(np.float32)
    for a in range(0, len(target), chunk):
        s = slice(a, a + chunk)
        out["loss_sum"].append(np.float32((per_row_ce[s] * w[s]).sum(dtype=np.float32)))
        out["in_vocab"].append(np.float32(w[s].sum()))
        out["correct"].append(np.float32((correct[s] * w[s]).sum()))
    return out


def test_results_arithmetic_over_all_questions_and_in_vocabulary_loss():
    """accuracy = correct / every question (OOV questions count wrong), loss = CE summed over the in-vocabulary questions /
    their number, oov = the rest; every chunking of the same rows gives the same line."""
    rng = np.random.default_rng(3)
    n = 12
    ce = rng.random(n).astype(np.float32) * 3
    target = rng.integers(0, A, n)
    target[[1, 4, 5, 11]] = -1
    correct = (rng.random(n) < 0.5).astype(np.float32)
    iv = target >= 0
    want = {"accuracy": float((correct * iv).sum()) / n, "loss": float(ce[iv].astype(np.float64).mean()), "oov": 4}
    for chunk in (1, 2, 3, 4, 6, 12):
        c = _chunks(ce, target, correct, chunk)
        got = QV.results(c["loss_sum"], c["in_vocab"], c["correct"], n)
        assert got["oov"] == want["oov"] and got["accuracy"] == want["accuracy"]
        assert got["loss"] == pytest.approx(want["loss"], rel=1e-6)
    assert QV.results([0.0], [0.0], [0.0], 3) == {"accuracy": 0.0, "loss": None, "oov": 3}


def test_results_line_names_accuracy_and_oov(tmp_path):
    from merlot_b200 import vcr_validate as VV
    res = {"global_step": 3, "accuracy": 0.5, "loss": 1.5, "questions": 8, "oov": 2, "x": 1}
    path = VV.append_result(str(tmp_path), res, "accuracy", QV.Validator.EXTRA_KEYS)
    assert [json.loads(x) for x in open(path).read().splitlines()] == [
        {"global_step": 3, "accuracy": 0.5, "loss": 1.5, "questions": 8, "oov": 2}]


def test_top_k_predictions():
    g = np.random.default_rng(0)
    logits = g.standard_normal((5, 9)).astype(np.float32)
    logits[0, [2, 7]] = 9.0  # a tie: the lower index first
    idx, lp = QV.top_k(logits)
    assert idx.shape == lp.shape == (5, 5) and idx.dtype == np.int64 and lp.dtype == np.float32
    assert idx[0, :2].tolist() == [2, 7]
    from merlot_b200.vcr_validate import log_softmax
    full = log_softmax(logits)
    np.testing.assert_array_equal(idx[:, 0], full.argmax(-1))
    np.testing.assert_array_equal(lp, np.take_along_axis(full, idx, 1))
    assert (np.diff(lp, axis=1) <= 0).all()
    idx3, lp3 = QV.top_k(logits[:, :3])
    assert idx3.shape == (5, 3)  # k = min(5, A)
