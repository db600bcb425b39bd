"""CPU tests of multiple-choice video QA (downstream.task: video_mc) on the host: the record parser against a NumPy
restatement (texts, padding, truncation, img_mask for every frame count, labels and every record error), the training
shard and shuffle, the evaluation batch order and its independence of the number of ranks, the parameter arena of
ParamStore(task="video_mc") beside unchanged pretraining and VCR arenas, the config errors and the command-line checks."""
import hashlib
import json

import numpy as np
import pytest
import torch

from merlot_b200 import video_mc as VM
from merlot_b200 import video_mc_input as MI
from merlot_b200 import video_mc_validate as MV
from merlot_b200.dataloader import shard_files, shuffled_records
from merlot_b200.sort_story import eval_batches
from merlot_b200.tfrecord import parse_example, read_records
from tests import video_mc_oracle as MO
from tests import video_mc_records as R

F, C, L, VOCAB = 3, 5, 40, 1000


def _parse(q, num_frames=F, num_choices=C, max_len=L):
    return MI.parse_question(parse_example(R.example(q)), num_frames, num_choices, max_len, VOCAB)


def _q(k=0, seed=0, **kw):
    return R.question(np.random.default_rng(seed), k, F, C, **kw)


def test_texts_padding_and_truncation_match_restatement():
    rng = np.random.default_rng(1)
    qs = [R.question(rng, k, F, C) for k in range(6)]
    qs[0]["question"] = []
    qs[1]["question"] = None  # absent: an empty question
    qs[2]["choice_3"] = []
    qs[3]["question"] = list(range(100, 137))  # 1 + 37 + choice + 1 > 40: truncated, the END lost
    for q in qs:
        got = _parse(q)
        assert got["lm_input"].dtype == np.int32 and got["lm_input"].shape == (C, L)
        np.testing.assert_array_equal(got["lm_input"], R.texts_np(q, C, L))
        assert got["id"] == q["id"] and got["label"] == q["label"] and got["jpegs"] == q["frames"]
    long = _parse(qs[3])["lm_input"]
    assert (long[:, -1] != 0).all() and (long != MI.END).all() and (long[:, 0] == MI.START).all()
    short = _parse(qs[0])["lm_input"][2 if qs[0]["choice_2"] == [] else 0]
    assert MI.END in short.tolist() and short[-1] == MI.PADDING


@pytest.mark.parametrize("k", range(1, F + 1))
def test_img_mask_for_every_frame_count(k):
    q = _q(k, frames=k)
    p = _parse(q)
    assert len(p["jpegs"]) == k
    np.testing.assert_array_equal(MI.img_mask([p], F)[0], R.mask_np(q, F))
    np.testing.assert_array_equal(MI.img_mask([p, _parse(_q(9, frames=F))], F), [R.mask_np(q, F), [True] * F])


def test_label_rules():
    q = _q(4)
    assert _parse(dict(q, label=None))["label"] == -1
    MI.check_labels([_parse(q)], C)
    for bad in (None, -1, C, 17):
        p = _parse(dict(q, id="q-bad", label=bad))
        with pytest.raises(ValueError, match=r"id='q-bad': label is %d, outside \[0, 5\)" % (-1 if bad is None else bad)):
            MI.check_labels([_parse(q), p], C)


@pytest.mark.parametrize("case,match", [
    ("no_frames", r"id='q-7': 0 frames, expected 1 to 3"),
    ("absent_frames", r"id='q-7': 0 frames, expected 1 to 3"),
    ("too_many_frames", r"id='q-7': 4 frames, expected 1 to 3"),
    ("missing_choice", r"id='q-7': choice_4 is missing"),
    ("token_too_large", r"id='q-7': choice_1 holds token id 1000 outside the vocabulary \[0, 1000\)"),
    ("negative_token", r"id='q-7': question holds token id -5 outside the vocabulary"),
])
def test_record_errors_name_the_id(case, match):
    q = _q(7)
    if case == "no_frames":
        q["frames"] = []
    elif case == "absent_frames":
        q["frames"] = None
    elif case == "too_many_frames":
        q["frames"] = q["frames"][:1] * (F + 1)
    elif case == "missing_choice":
        q["choice_4"] = None
    elif case == "token_too_large":
        q["choice_1"] = [5, VOCAB]
    else:
        q["question"] = [10, -5]
    with pytest.raises(ValueError, match=match):
        _parse(q)


def test_undecodable_frame_names_the_id():
    q = _q(8, frames=2)
    q["frames"][1] = b"\xff\xd8 not a jpeg"
    p = _parse(q)
    assert MI.decode_frame(p, 0).shape[2] == 3
    with pytest.raises(ValueError, match="id='q-8': frame 1 cannot be decoded"):
        MI.decode_frame(p, 1)


def test_training_draws_one_per_question():
    d = MI.train_draws(np.random.default_rng([5, 1]), 7)
    rng = np.random.default_rng([5, 1])
    f32 = np.float32
    np.testing.assert_array_equal(d["scale"], f32(0.9) + rng.random(7, dtype=f32) * (f32(1.1) - f32(0.9)))
    np.testing.assert_array_equal(d["u_y"], rng.random(7, dtype=f32))
    np.testing.assert_array_equal(d["u_x"], rng.random(7, dtype=f32))
    assert (d["scale"] >= 0.9).all() and (d["scale"] < 1.1).all()


def test_training_shard_and_shuffle(tmp_path):
    R.write_questions(tmp_path, [3, 4, 2, 5], F, C, prefix="train", max_question=2, max_choice=2, sizes=[(8, 8)])
    files = sorted(str(p) for p in tmp_path.glob("train-*.tfrecord"))
    every = {r for f in files for r in read_records(f)}

    def take(seed, rank, world, n=40):
        shard = shard_files(files, rank, world)
        recs = shuffled_records(shard, np.random.default_rng([seed, rank]), min(2, len(shard)), 4)
        return [next(recs) for _ in range(n)]
    assert take(0, 0, 1) == take(0, 0, 1) and take(0, 0, 1) != take(1, 0, 1)
    assert set(take(0, 0, 1, 200)) == every
    r0, r1 = take(3, 0, 2), take(3, 1, 2)
    in0 = {r for f in files[0::2] for r in read_records(f)}
    assert set(r0) <= in0 and not set(r1) & in0  # rank r reads files r, r + world, ...


def test_eval_order_dropped_and_ranks(tmp_path):
    R.write_questions(tmp_path, [5, 3, 4], F, C, prefix="val", max_question=2, max_choice=2, sizes=[(8, 8)])
    files = sorted(str(p) for p in tmp_path.glob("val-*.tfrecord"))

    def ids(records):
        return [parse_example(r)["id"][0].decode() for r in records]
    tail = []
    one = [ids(b) for b in eval_batches(files, 2, 2, tail)]
    # sorted files, two interleaved readers, no shuffle: file 0 and file 1 alternate, then file 2 after file 1 ends
    assert [i for b in one for i in b][:6] == ["q-0", "q-5", "q-1", "q-6", "q-2", "q-7"]
    assert len(one) == 6 and len(tail) == 0
    tail3 = []
    assert len([b for b in eval_batches(files, 2, 5, tail3)]) == 2 and len(tail3) == 2  # 12 records: 2 dropped
    for world in (2, 3):
        got = {}
        for rank in range(world):
            t = []
            for k, b in zip(range(rank, 100, world), eval_batches(files, 2, 2, t, rank=rank, world=world)):
                got[k] = ids(b)
            assert len(t) == 0
        assert [got[k] for k in range(len(one))] == one  # global batch k on rank k % world, the same batches


def _tiny(**kw):
    return dict(dict(use_bfloat16=True, hidden_size=128, vocab_size=1000, patch_size=16, spatial_pool_size=2, num_attention_heads=2,
                num_hidden_layers=2, num_vision_transformer_hidden_layers=2, num_lang_transformer_hidden_layers=2,
                intermediate_size=256, initializer_range=0.02, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.0,
                max_position_embeddings=64, num_chunks_in_group=2, do_projection=True, do_bias=True, contrastive_size=128,
                contrast_coef=0.25, contrast_temp=0.05, image_shuffle_prob=0.4, masking_rate=0.2, resnet_layers=[]), **kw)


def _digest(store):
    lay = [(e.name, list(e.shape), list(e.tf_names), e.offset, e.padded, e.ref_cols, list(e.hyper)) for e in store.entries.values()]
    return hashlib.sha256(json.dumps([lay, store.total]).encode()).hexdigest()


# the arena layouts (names, shapes, offsets, padding, hyper-parameters) before the video_mc task was added
_PARENT_DIGESTS = {
    ("tiny", "pretrain"): "5ca2e67342741c3fab98219b357666456ae603d3606d74624892d3467f253576",
    ("tiny", "vcr"): "00709e427000d71adb14f473ac47dadb1e94c8497defad3e0efee1a718b2a822",
    ("hybrid", "pretrain"): "fa0f7e63c7d51aee9614ce2723bd54b7fc96dd4fe4cba11e5c62965b305697ca",
    ("hybrid", "vcr"): "9c5bc6ba86a2bddcf10e019fda3a9e64e2d02e9ca3f195d014a6f45479d50e46",
    ("separate", "pretrain"): "fc9335373e56983ad1105e75825c9af9f8cdf3d35f91d065fdd58199d72073b9",
    ("separate", "vcr"): "00709e427000d71adb14f473ac47dadb1e94c8497defad3e0efee1a718b2a822",
}


@pytest.mark.parametrize("variant,task", sorted(_PARENT_DIGESTS))
def test_pretrain_and_vcr_arenas_are_unchanged(variant, task):
    from merlot_b200.params import ParamStore
    cfg = {"tiny": _tiny(), "hybrid": _tiny(resnet_layers=[1, 2, 1]), "separate": _tiny(share_params=False)}[variant]
    assert _digest(ParamStore(cfg, device="cpu", task=task, with_optimizer_state=False)) == _PARENT_DIGESTS[(variant, task)]


def test_video_mc_store_names_shapes_and_round_trip():
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F, num_texts=C)
    vcr = ParamStore(cfg, device="cpu", task="vcr", with_optimizer_state=False)
    st = ParamStore(cfg, device="cpu", task="video_mc", with_optimizer_state=False)
    towers = sorted(n for n in st.entries if n.startswith("mc_cls/"))
    assert towers == ["mc_cls/classifier_mlp0/bias", "mc_cls/classifier_mlp0/kernel", "mc_cls/classifier_mlp1/bias",
                      "mc_cls/classifier_mlp1/kernel"]
    model = {n: e.shape for n, e in vcr.entries.items() if not n.startswith(("answer_cls/", "rationale_cls/"))}
    assert {n: e.shape for n, e in st.entries.items() if not n.startswith("mc_cls/")} == model
    for n in towers:  # the answer tower's shapes, classifier_mlp1 padded to 8 columns
        a = vcr.entries[n.replace("mc_cls/", "answer_cls/")]
        assert st.entries[n].shape == a.shape and st.entries[n].ref_cols == a.ref_cols
    shapes = {k: tuple(v.shape) for k, v in st.to_tf_dict().items()}
    assert shapes == {k: tuple(v) for k, v in MO.param_shapes(cfg).items()}
    assert shapes["mc_cls/classifier_mlp1/kernel"] == (64, 1) and shapes["mc_cls/classifier_mlp1/bias"] == (1,)
    params = MO.init_params(cfg, seed=3, perturb=0.05)
    st.load_tf_dict(params)
    back = st.to_tf_dict()
    assert set(back) == set(params)
    for k in params:
        assert torch.equal(back[k], params[k].float().reshape(back[k].shape)), k
    assert float(st.P("mc_cls/classifier_mlp1/kernel")[:, 1:].abs().max()) == 0.0
    st.init_reference(seed=0)
    assert float(st.P("mc_cls/classifier_mlp1/bias")[0]) == pytest.approx(-np.log(3.0))


def test_pretraining_checkpoint_leaves_the_tower_missing():
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F, num_texts=C)
    pre = ParamStore(cfg, device="cpu", task="pretrain", with_optimizer_state=False).to_tf_dict()
    st = ParamStore(cfg, device="cpu", task="video_mc", with_optimizer_state=False)
    st.init_reference(seed=0)
    before = st.P("mc_cls/classifier_mlp0/kernel").clone()
    missing = st.load_tf_dict(pre, strict=False)
    assert sorted(missing) == ["mc_cls/classifier_mlp0/bias", "mc_cls/classifier_mlp0/kernel", "mc_cls/classifier_mlp1/bias",
                               "mc_cls/classifier_mlp1/kernel"]
    assert torch.equal(st.P("mc_cls/classifier_mlp0/kernel"), before)


@pytest.mark.parametrize("num_imgs,num_texts,ok", [(1, 2, True), (6, 8, True), (3, 1, False), (3, 9, False), (0, 4, False)])
def test_config_errors(num_imgs, num_texts, ok):
    cfg = _tiny(num_imgs=num_imgs, num_texts=num_texts)
    if ok:
        assert VM.check_config(cfg) == (num_imgs, num_texts)
        return
    match = "num_imgs" if num_imgs < 1 else r"num_texts .* must be in \[2, 8\]"
    with pytest.raises(ValueError, match=match):
        VM.check_config(cfg)
    from merlot_b200.config import NeatConfig
    with pytest.raises(ValueError, match=match):
        VM.video_mc_model_fn_builder(NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {}, "device": {"output_dir": "/tmp/merlot_video_mc"},
                                                          "downstream": {"task": "video_mc"}}), device="cpu")


def test_store_of_another_task_is_refused():
    from merlot_b200.config import NeatConfig
    from merlot_b200.params import ParamStore
    cfg = _tiny(num_imgs=F, num_texts=C)
    config = NeatConfig.from_dict({"data": {}, "model": cfg, "optimizer": {"learning_rate": 1e-4}, "device": {"output_dir": "/tmp/merlot_video_mc"},
                                   "downstream": {"task": "video_mc"}})
    for task in ("vcr", "pretrain"):
        with pytest.raises(ValueError, match=f"ParamStore\\(task='video_mc'\\), got task='{task}'"):
            VM.video_mc_model_fn_builder(config, store=ParamStore(cfg, device="cpu", task=task), device="cpu")


def test_synthetic_batch_and_cli_dispatch():
    from merlot_b200 import train
    from merlot_b200.config import NeatConfig
    cfg = NeatConfig.from_dict({"data": {}, "model": _tiny(num_imgs=F, num_texts=C, image_size=[32, 48]), "optimizer": {},
                                "device": {"output_dir": "/tmp/merlot_video_mc"}, "downstream": {"task": "video_mc", "max_text_len": 24}})
    f = train.synthetic_video_mc_batch(cfg, 4, seed=1, device="cpu")
    assert f["images"].shape == (4 * F, 32, 48, 3) and f["images"].dtype == torch.bfloat16
    assert f["lm_input"].shape == (4 * C, 24) and f["lm_targets"].shape == (4,)
    assert f["img_mask"].tolist() == [[True, False, False], [True, True, False], [True, True, True], [True, False, False]]
    empty = ~f["img_mask"].reshape(-1)
    assert float(f["images"][empty].abs().max()) == 0.0 and float(f["images"][~empty].abs().max()) > 0
    assert ((f["lm_targets"] >= 0) & (f["lm_targets"] < C)).all() and (f["lm_input"][:, 0] == 2).all()
    assert train._step_for(cfg) == (VM.video_mc_model_fn_builder, train.synthetic_video_mc_batch)


@pytest.mark.parametrize("args,match", [(["--predictions", "p.npz"], "--checkpoint"),
                                        (["--checkpoint", "x", "--predictions", "p.txt"], ".npz"),
                                        (["--unlabelled"], "--predictions"),
                                        (["--chunk", "-1"], "--chunk")])
def test_validator_argument_checks(tmp_path, args, match):
    with pytest.raises(ValueError, match=match):
        MV.main([str(tmp_path / "none.yaml")] + args)  # raised before the config is read


def test_validator_needs_the_video_mc_task(tmp_path):
    import yaml
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump({"data": {}, "model": {}, "optimizer": {}, "device": {"output_dir": str(tmp_path)},
                                    "downstream": {"task": "vcr"}}))
    with pytest.raises(ValueError, match="video_mc validation needs 'video_mc'"):
        MV.main([str(path)])


def test_results_line_names_accuracy(tmp_path):
    from merlot_b200 import vcr_validate as VV
    path = VV.append_result(str(tmp_path), {"global_step": 3, "accuracy": 0.5, "loss": 1.5, "questions": 8, "x": 1}, "accuracy")
    assert [json.loads(x) for x in open(path).read().splitlines()] == [
        {"global_step": 3, "accuracy": 0.5, "loss": 1.5, "questions": 8}]
