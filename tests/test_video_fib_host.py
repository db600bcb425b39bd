"""CPU tests of fill-in-the-blank video QA (downstream.task: video_fib) on the host: the record parser against a NumPy
restatement (texts, blank positions, exactly one MASK, a MASK lost to truncation, frame / token / answer errors naming
the id), the answer_tokens file and config errors, the parameter arena of ParamStore(task="video_fib") (entries,
checkpoint shapes, the other tasks' layouts unchanged), the answer layer's derivation against a float64 NumPy mean, the
step dispatch and synthetic batch, the refusals of the other programs, and the validator's command line and results
line."""
import hashlib
import json

import numpy as np
import pytest
import torch

from merlot_b200 import video_fib as VF
from merlot_b200 import video_fib_input as FI
from merlot_b200 import video_fib_validate as FV
from merlot_b200.tfrecord import parse_example
from tests import video_fib_records as FR
from tests.test_video_mc_host import _tiny

F, L, VOCAB, A = 3, 40, 1000, 13


def _parse(q, num_frames=F, max_len=L):
    return FI.parse_question(parse_example(FR.example(q)), num_frames, max_len, VOCAB)


def _q(k=0, seed=0, **kw):
    return FR.question(np.random.default_rng(seed), k, F, A, **kw)


def test_texts_and_blank_positions_match_restatement():
    rng = np.random.default_rng(1)
    qs = [FR.question(rng, k, F, A) for k in range(8)]
    qs[0]["question"] = [FR.MASK]  # the blank alone
    qs[1]["question"] = [FR.MASK] + list(range(100, 137))  # 1 + 38 + 1 = 40 tokens: nothing cut
    qs[2]["question"] = list(range(100, 137)) + [FR.MASK, 500, 501]  # the MASK at position 38 survives, the END does not
    for q in qs:
        got = _parse(q)
        assert got["lm_input"].dtype == np.int32 and got["lm_input"].shape == (L,)
        np.testing.assert_array_equal(got["lm_input"], FR.text_np(q, L))
        assert got["blank_pos"] == FR.blank_np(q) and got["lm_input"][got["blank_pos"]] == FR.MASK
        assert got["id"] == q["id"] and got["answer"] == q["answer"] and got["jpegs"] == q["frames"]
    assert _parse(qs[0])["lm_input"][:4].tolist() == [2, FR.MASK, 3, 0]  # START, the blank, END, PADDING
    assert _parse(qs[2])["blank_pos"] == 38


@pytest.mark.parametrize("case,match", [
    ("no_mask", r"video_fib record id='q-7': question holds 0 MASK tokens \(id 1\), expected exactly one"),
    ("two_masks", r"video_fib record id='q-7': question holds 2 MASK tokens"),
    ("no_question", r"video_fib record id='q-7': question holds 0 MASK tokens"),
    ("truncated", r"video_fib record id='q-7': the MASK \(the blank\) is cut off by downstream.max_text_len 40"),
    ("no_frames", r"video_fib record id='q-7': 0 frames, expected 1 to 3"),
    ("too_many_frames", r"video_fib record id='q-7': 4 frames, expected 1 to 3"),
    ("token_too_large", r"video_fib record id='q-7': question holds token id 1000 outside the vocabulary \[0, 1000\)"),
    ("negative_token", r"video_fib record id='q-7': question holds token id -5 outside the vocabulary"),
])
def test_record_errors_name_the_id(case, match):
    q = _q(7)
    if case == "no_mask":
        q["question"] = [10, 11, 12]
    elif case == "two_masks":
        q["question"] = [10, FR.MASK, 12, FR.MASK]
    elif case == "no_question":
        q["question"] = None
    elif case == "truncated":
        q["question"] = list(range(100, 139)) + [FR.MASK]  # START + 39 words fill the 40 slots: the MASK is cut
    elif case == "no_frames":
        q["frames"] = None
    elif case == "too_many_frames":
        q["frames"] = q["frames"][:1] * (F + 1)
    elif case == "token_too_large":
        q["question"] = [FR.MASK, VOCAB]
    else:
        q["question"] = [FR.MASK, -5]
    with pytest.raises(ValueError, match=match):
        _parse(q)


def test_answer_rules_and_batch_fields():
    qs = [_parse(_q(k)) for k in range(3)] + [_parse(dict(_q(3), answer=-1))]

    class Fields(FI._FiB):
        def __init__(self, labelled):
            self.labelled, self.num_answers = labelled, A

    f = Fields(True)._text_fields(qs)
    assert f["lm_input"].shape == (4, L) and f["lm_input"].dtype == np.int32
    assert f["blank_pos"].dtype == np.int32 and f["blank_pos"].tolist() == [q["blank_pos"] for q in qs]
    assert (f["lm_input"][np.arange(4), f["blank_pos"]] == FR.MASK).all()
    assert f["lm_targets"].tolist() == [q["answer"] for q in qs] and f["lm_targets"][3] == -1
    unl = [_parse(dict(_q(k), answer=None)) for k in range(2)]
    with pytest.raises(ValueError, match=r"video_fib record id='q-0': answer is missing"):
        Fields(True)._text_fields(unl)
    assert Fields(False)._text_fields(unl)["lm_targets"].tolist() == [-1, -1]
    with pytest.raises(ValueError, match=r"video_fib record id='q-5': answer is 13, outside \[-1, 13\)"):
        Fields(True)._text_fields([_parse(dict(_q(5), answer=A))])
    with pytest.raises(ValueError, match=r"video_fib record id='q-5': answer is -2"):
        Fields(True)._text_fields([_parse(dict(_q(5), answer=-2))])


def _ds(tmp_path, ans, **kw):
    return dict({"answer_tokens": FR.write_answers(tmp_path / "answers.json", ans)}, **kw)


def test_answer_tokens_file(tmp_path):
    ans = [[7], [999], [100, 200, 300], [42, 42]]
    assert VF.check_config(_tiny(num_imgs=6), _ds(tmp_path, ans)) == (6, ans)
    assert VF.check_config(_tiny(num_imgs=2, num_texts=1), _ds(tmp_path, ans, num_answers=4)) == (2, ans)
    for bad, match in [([[7]], r"must hold a list of >= 2 answers, got 1"),
                       ({"a": [7]}, r"must hold a list of >= 2 answers, got dict"),
                       ([[7], []], r"answer 1 of .* must be a non-empty list of token ids, got \[\]"),
                       ([[7], 8], r"answer 1 of .* must be a non-empty list of token ids, got 8"),
                       ([[7], [6]], r"answer 1 of .* holds token id 6 outside \[7, 1000\)"),
                       ([[1], [8]], r"answer 0 of .* holds token id 1 outside"),
                       ([[7], [8, 1000]], r"answer 1 of .* holds token id 1000 outside \[7, 1000\)"),
                       ([[7], [8.0]], r"holds token id 8.0 outside"),
                       ([[7], [True]], r"holds token id True outside")]:
        with pytest.raises(ValueError, match=match):
            VF.check_config(_tiny(num_imgs=2), _ds(tmp_path, bad))


@pytest.mark.parametrize("model,downstream,match", [
    (dict(num_imgs=0), {}, "num_imgs .* got 0"),
    (dict(num_imgs=2, num_texts=4), {}, "num_texts must be 1.* got 4"),
    (dict(num_imgs=2), {"answer_tokens": None}, "answer_tokens .* is missing"),
    (dict(num_imgs=2), {"num_answers": 5}, "num_answers is 5, downstream.answer_tokens holds 4 answers"),
])
def test_config_errors(tmp_path, model, downstream, match):
    cfg = _tiny(**model)
    ds = _ds(tmp_path, [[7], [8], [9, 10], [11]])
    ds.update(downstream)
    with pytest.raises(ValueError, match=match):
        VF.check_config(cfg, ds)
    from merlot_b200.config import NeatConfig
    with pytest.raises(ValueError, match=match):
        VF.video_fib_model_fn_builder(NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {},
                                                            "device": {"output_dir": str(tmp_path)},
                                                            "downstream": dict(ds, task="video_fib")}), device="cpu")


def _digest(store):
    lay = [(e.name, list(e.shape), list(e.tf_names), e.offset, e.padded, e.ref_cols, list(e.hyper)) for e in store.entries.values()]
    return hashlib.sha256(json.dumps([lay, store.total]).encode()).hexdigest()


# the arena layouts (names, shapes, offsets, padding, hyper-parameters) before the video_fib task was added; video_qa at A = 13
_PARENT_DIGESTS = {
    ("tiny", "pretrain"): "5ca2e67342741c3fab98219b357666456ae603d3606d74624892d3467f253576",
    ("tiny", "vcr"): "00709e427000d71adb14f473ac47dadb1e94c8497defad3e0efee1a718b2a822",
    ("tiny", "video_mc"): "0b704ec04546321c14af1eb04d1063f07f096d86fd76f9f3ba30e81a7cfb0f44",
    ("tiny", "video_qa"): "e7ac1b0759680c67e1cd8bbebd053e3fc6509330c16b431bfd6fc06deedc9f5d",
    ("hybrid", "pretrain"): "fa0f7e63c7d51aee9614ce2723bd54b7fc96dd4fe4cba11e5c62965b305697ca",
    ("hybrid", "vcr"): "9c5bc6ba86a2bddcf10e019fda3a9e64e2d02e9ca3f195d014a6f45479d50e46",
    ("hybrid", "video_mc"): "19292f9897ece107c312be73554210f56866921231733e65f3d753249ca05955",
    ("hybrid", "video_qa"): "31190c9db5fc305f6eee408236dc9d680ba14a922bd7b4ba12b6a54bfaed3918",
    ("separate", "pretrain"): "fc9335373e56983ad1105e75825c9af9f8cdf3d35f91d065fdd58199d72073b9",
    ("separate", "vcr"): "00709e427000d71adb14f473ac47dadb1e94c8497defad3e0efee1a718b2a822",
    ("separate", "video_mc"): "0b704ec04546321c14af1eb04d1063f07f096d86fd76f9f3ba30e81a7cfb0f44",
    ("separate", "video_qa"): "e7ac1b0759680c67e1cd8bbebd053e3fc6509330c16b431bfd6fc06deedc9f5d",
    ("noproj", "pretrain"): "3076c74f4fb3738232d968e7232a0ea20fd9eb1002e2974b92c2826b3477a222",
    ("noproj", "vcr"): "00709e427000d71adb14f473ac47dadb1e94c8497defad3e0efee1a718b2a822",
    ("noproj", "video_mc"): "0b704ec04546321c14af1eb04d1063f07f096d86fd76f9f3ba30e81a7cfb0f44",
    ("noproj", "video_qa"): "e7ac1b0759680c67e1cd8bbebd053e3fc6509330c16b431bfd6fc06deedc9f5d",
}
_VARIANTS = {"tiny": {}, "hybrid": {"resnet_layers": [1, 2, 1]}, "separate": {"share_params": False},
             "noproj": {"do_projection": False, "do_bias": False}}


@pytest.mark.parametrize("variant,task", sorted(_PARENT_DIGESTS))
def test_other_arenas_are_unchanged(variant, task):
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F, **_VARIANTS[variant])
    kw = {"num_answers": 13} if task == "video_qa" else {}
    assert _digest(ParamStore(cfg, device="cpu", task=task, with_optimizer_state=False, **kw)) == _PARENT_DIGESTS[(variant, task)]


@pytest.mark.parametrize("do_projection", [True, False])
@pytest.mark.parametrize("num_answers,stored", [(13, 16), (16, 16), (1500, 1504), (2, 8)])
def test_video_fib_store_entries_and_checkpoint_shapes(num_answers, stored, do_projection):
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F, do_projection=do_projection)
    vcr = ParamStore(cfg, device="cpu", task="vcr", with_optimizer_state=False)
    st = ParamStore(cfg, device="cpu", task="video_fib", num_answers=num_answers, with_optimizer_state=False)
    head = sorted(n for n in st.entries if n.startswith(("lm_head/", "fib_cls/")))
    proj = ["lm_head/LayerNorm/beta", "lm_head/LayerNorm/gamma", "lm_head/projection/bias", "lm_head/projection/kernel"]
    assert head == ["fib_cls/answers/bias", "fib_cls/answers/kernel"] + (proj if do_projection else [])
    model = {n: e.shape for n, e in vcr.entries.items() if not n.startswith(("answer_cls/", "rationale_cls/"))}
    assert {n: e.shape for n, e in st.entries.items() if n not in head} == model
    k, b = st.entries["fib_cls/answers/kernel"], st.entries["fib_cls/answers/bias"]
    assert k.shape == (128, stored) and b.shape == (stored,) and k.ref_cols == b.ref_cols == num_answers
    if do_projection:
        assert st.entries["lm_head/projection/kernel"].shape == (128, 128) and st.entries["lm_head/LayerNorm/gamma"].shape == (128,)
    assert "lm_head/output_bias" not in st.entries  # nothing trains a [V] bias; the derivation reads it from the checkpoint
    shapes = {k: tuple(v.shape) for k, v in st.to_tf_dict().items()}
    assert shapes["fib_cls/answers/kernel"] == (128, num_answers) and shapes["fib_cls/answers/bias"] == (num_answers,)
    g = torch.Generator().manual_seed(1)
    d = {k: torch.randn(v.shape, generator=g) for k, v in st.to_tf_dict().items()}
    st.load_tf_dict(d)
    back = st.to_tf_dict()
    for name in d:
        assert torch.equal(back[name], d[name]), name
    assert st.P("fib_cls/answers/kernel")[:, num_answers:].count_nonzero() == 0
    head_params = 128 * num_answers + num_answers + (128 * 128 + 3 * 128 if do_projection else 0)
    assert st.num_params() == vcr.num_params() - 2 * (128 * 64 + 64 + 64 + 1) + head_params
    # the head's kernels decay, its biases and LayerNorm do not (the reference's param_overrides)
    ocfg = {"learning_rate": 1e-4, "weight_decay_rate": 0.01, "param_overrides": [[["LayerNorm", "bias"], {"weight_decay_rate": 0}]]}
    st2 = ParamStore(cfg, device="cpu", task="video_fib", num_answers=num_answers, optimizer_cfg=ocfg, with_optimizer_state=False)
    assert st2.entries["fib_cls/answers/kernel"].hyper[1] == 0.01 and st2.entries["fib_cls/answers/bias"].hyper[1] == 0


def test_store_needs_num_answers_for_video_fib():
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F)
    with pytest.raises(ValueError, match="num_answers is the size of the video_fib answer vocabulary"):
        ParamStore(cfg, device="cpu", task="video_fib", with_optimizer_state=False)
    with pytest.raises(ValueError, match="video_fib: num_answers must be >= 2, got 1"):
        ParamStore(cfg, device="cpu", task="video_fib", num_answers=1, with_optimizer_state=False)


def _derive_np(emb, ans, bias):
    """fp32 [H, A] kernel and [A] bias: float64 means of the rows / bias entries of every answer's tokens, rounded."""
    emb64 = emb.double().numpy()
    kern = np.stack([emb64[a].mean(0) for a in ans], 1).astype(np.float32)
    b = np.zeros(len(ans), np.float32) if bias is None else np.array([bias.double().numpy()[a].mean() for a in ans], np.float32)
    return kern, b


@pytest.mark.parametrize("with_bias", [True, False])
@pytest.mark.parametrize("max_tokens", [1, 4])
def test_derivation_against_float64_mean(with_bias, max_tokens):
    from merlot_b200.params import ParamStore, derive_fib_answers
    rng = np.random.default_rng(max_tokens)
    ans = FR.answers(rng, A, max_tokens=max_tokens)
    if max_tokens > 1:
        ans[0] = [50, 50, 51]  # a repeated token counts twice
    st = ParamStore(_tiny(num_imgs=F), device="cpu", task="video_fib", num_answers=A, with_optimizer_state=False)
    st.init_reference(seed=3)
    emb = st.P("word_embeddings/word_embeddings").clone()
    bias = torch.randn(VOCAB, generator=torch.Generator().manual_seed(4)) if with_bias else None
    st.P("fib_cls/answers/kernel").fill_(7.0)  # every column written, the padding zeroed
    derive_fib_answers(st, ans, bias)
    kern, b = _derive_np(emb, ans, bias)
    np.testing.assert_array_equal(st.P("fib_cls/answers/kernel")[:, :A].numpy(), kern)
    np.testing.assert_array_equal(st.P("fib_cls/answers/bias")[:A].numpy(), b)
    assert float(st.P("fib_cls/answers/kernel")[:, A:].abs().max()) == 0.0
    assert float(st.P("fib_cls/answers/bias")[A:].abs().max()) == 0.0
    assert torch.equal(st.W("fib_cls/answers/kernel"), st.P("fib_cls/answers/kernel").bfloat16())  # bf16 copy refreshed
    assert torch.equal(st.P("word_embeddings/word_embeddings"), emb)  # the input table is untouched
    if max_tokens == 1:  # a one-token answer's column is its embedding row exactly: its MLM logit
        for a, toks in enumerate(ans):
            assert torch.equal(st.P("fib_cls/answers/kernel")[:, a], emb[toks[0]])
            if bias is not None:
                assert float(st.P("fib_cls/answers/bias")[a]) == float(bias[toks[0]])


def test_derivation_refuses_another_store_or_size():
    from merlot_b200.params import ParamStore, derive_fib_answers
    cfg = _tiny(num_imgs=F)
    with pytest.raises(ValueError, match="ParamStore\\(task='video_fib'\\), got 'video_qa'"):
        derive_fib_answers(ParamStore(cfg, device="cpu", task="video_qa", num_answers=A, with_optimizer_state=False), [[7]] * A)
    with pytest.raises(ValueError, match="3 answers given, the store holds 13"):
        derive_fib_answers(ParamStore(cfg, device="cpu", task="video_fib", num_answers=A, with_optimizer_state=False), [[7]] * 3)


def test_pretraining_variables_restore_by_name_into_the_head():
    """A pretraining store's variables fill a video_fib store by name: lm_head/projection and LayerNorm are restored, only
    fib_cls/answers is missing (so it is derived)."""
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F)
    pre = ParamStore(cfg, device="cpu", task="pretrain", with_optimizer_state=False)
    pre.init_reference(seed=5)
    st = ParamStore(cfg, device="cpu", task="video_fib", num_answers=A, with_optimizer_state=False)
    st.init_reference(seed=0)
    missing = st.load_tf_dict(pre.to_tf_dict(), strict=False)
    assert sorted(missing) == ["fib_cls/answers/bias", "fib_cls/answers/kernel"]
    for n in ("lm_head/projection/kernel", "lm_head/LayerNorm/gamma", "word_embeddings/word_embeddings"):
        assert torch.equal(st.P(n), pre.P(n)), n


def test_store_of_another_task_or_size_is_refused(tmp_path):
    from merlot_b200.config import NeatConfig
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F)
    config = NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {"learning_rate": 1e-4},
                                   "device": {"output_dir": str(tmp_path)},
                                   "downstream": _ds(tmp_path, [[7 + a] for a in range(A)], task="video_fib")})
    with pytest.raises(ValueError, match="ParamStore\\(task='video_fib'\\), got task='video_qa'"):
        VF.video_fib_model_fn_builder(config, store=ParamStore(cfg, device="cpu", task="video_qa", num_answers=A), device="cpu")
    with pytest.raises(ValueError, match="holds 20 answers, downstream.answer_tokens holds 13"):
        VF.video_fib_model_fn_builder(config, store=ParamStore(cfg, device="cpu", task="video_fib", num_answers=20),
                                      device="cpu")


def test_blank_positions_on_the_device_side():
    ids = torch.tensor([[2, 5, 1, 3, 0], [2, 1, 9, 9, 3]], dtype=torch.int32)
    assert VF.blank_positions(ids).tolist() == [2, 1] and VF.blank_positions(ids).dtype == torch.int32
    for bad in ([[2, 5, 6, 3, 0], [2, 1, 9, 9, 3]], [[2, 1, 1, 3, 0], [2, 1, 9, 9, 3]]):
        with pytest.raises(ValueError, match="exactly one MASK"):
            VF.blank_positions(torch.tensor(bad))


def test_synthetic_batch_and_dispatch(tmp_path):
    from merlot_b200 import train
    from merlot_b200.config import NeatConfig
    from merlot_b200.params import ParamStore
    cfg = NeatConfig.from_dict({"data": {}, "model": _tiny(num_imgs=F, image_size=[32, 48]), "optimizer": {},
                                "device": {"output_dir": str(tmp_path)},
                                "downstream": _ds(tmp_path, [[7 + a] for a in range(A)], task="video_fib", max_text_len=24)})
    f = train.synthetic_video_fib_batch(cfg, 5, seed=1, device="cpu")
    assert f["images"].shape == (5 * F, 32, 48, 3) and f["lm_input"].shape == (5, 24) and f["img_mask"].shape == (5, F)
    assert ((f["lm_targets"] >= 0) & (f["lm_targets"] < A)).all() and (f["lm_input"][:, 0] == 2).all()
    assert ((f["lm_input"] == 1).sum(1) == 1).all() and f["blank_pos"].dtype == torch.int32
    assert torch.equal(VF.blank_positions(f["lm_input"]), f["blank_pos"])
    assert train._step_for(cfg) == (VF.video_fib_model_fn_builder, train.synthetic_video_fib_batch)
    st = ParamStore(cfg.model, device="cpu", task="video_fib", num_answers=A, with_optimizer_state=False)
    assert train.variables_without_gradient(cfg.model, st) == []


def test_predict_and_pretrain_validate_refuse_video_fib(tmp_path):
    import yaml
    from merlot_b200 import predict, pretrain_validate
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump({"data": {}, "model": {}, "optimizer": {}, "device": {"output_dir": str(tmp_path)},
                                    "downstream": {"task": "video_fib"}}))
    with pytest.raises(ValueError, match="'video_fib'"):
        predict.main([str(path), "--out", str(tmp_path / "o")])
    with pytest.raises(ValueError, match="video_fib fine-tuning with merlot_b200.video_fib_validate"):
        pretrain_validate.main([str(path)])


def test_validator_needs_the_video_fib_task(tmp_path):
    import yaml
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump({"data": {}, "model": {}, "optimizer": {}, "device": {"output_dir": str(tmp_path)},
                                    "downstream": {"task": "video_qa"}}))
    with pytest.raises(ValueError, match="video_fib validation needs 'video_fib'"):
        FV.main([str(path)])


@pytest.mark.parametrize("args,match", [(["--predictions", "p.npz"], "--checkpoint"), (["--unlabelled"], "--predictions"),
                                        (["--chunk", "-1"], "--chunk"), (["--zero-shot"], "--zero-shot .* --checkpoint")])
def test_validator_argument_checks(tmp_path, args, match):
    with pytest.raises(ValueError, match=match):
        FV.main([str(tmp_path / "none.yaml")] + args)


def test_other_validators_have_no_zero_shot_option(tmp_path):
    from merlot_b200 import vcr_validate, video_mc_validate, video_qa_validate
    for mod in (vcr_validate, video_mc_validate, video_qa_validate):
        with pytest.raises(SystemExit):
            mod.main([str(tmp_path / "none.yaml"), "--zero-shot"])


def test_results_line_arithmetic():
    """video_qa_validate's line: accuracy over every question with OOV wrong, loss over the in-vocabulary ones, oov the
    rest; any chunking of the same rows gives the same line."""
    assert FV.Validator.METRIC == "accuracy" and FV.Validator.EXTRA_KEYS == ("oov",) and FV.Validator.ID_KEYS == ("id",)
    rng = np.random.default_rng(3)
    n = 12
    ce = rng.random(n).astype(np.float32) * 3
    target = rng.integers(0, A, n)
    target[[0, 7]] = -1
    correct = (rng.random(n) < 0.5).astype(np.float32) * (target >= 0)
    iv = target >= 0
    for chunk in (1, 3, 4, 12):
        sl = [slice(a, a + chunk) for a in range(0, n, chunk)]
        got = FV.video_qa_validate.results([ce[s][iv[s]].sum(dtype=np.float32) for s in sl],
                                           [np.float32(iv[s].sum()) for s in sl], [correct[s].sum() for s in sl], n)
        assert got["oov"] == 2 and got["accuracy"] == float(correct.sum()) / n
        assert got["loss"] == pytest.approx(float(ce[iv].astype(np.float64).mean()), rel=1e-6)


def test_results_line_names(tmp_path):
    from merlot_b200 import vcr_validate as VV
    res = {"global_step": 0, "accuracy": 0.25, "loss": 2.5, "questions": 8, "oov": 1, "x": 1}
    path = VV.append_result(str(tmp_path), res, FV.Validator.METRIC, FV.Validator.EXTRA_KEYS)
    assert [json.loads(x) for x in open(path).read().splitlines()] == [
        {"global_step": 0, "accuracy": 0.25, "loss": 2.5, "questions": 8, "oov": 1}]
