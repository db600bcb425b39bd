"""CPU tests of the pretraining input's host half: TFRecord framing, tf.train.Example decoding, the text parser, the frame plan,
file sharding -- against tests/input_oracle.py -- and the oracle's own hand-derived known answers."""
import numpy as np
import pytest

from merlot_b200 import dataloader as D
from merlot_b200.config import NeatConfig
from merlot_b200.tfrecord import RecordFormatError, parse_example, read_records
from tests import input_oracle as O
from tests import tfrecord_writer as W


# ---- record framing ---------------------------------------------------------------------------------------------------
def test_record_framing_roundtrip(tmp_path):
    recs = [b"", b"a", bytes(range(256)) * 300]  # the last one takes crc32c's vectorised path
    p = tmp_path / "x.tfrecord"
    W.write_records(p, recs)
    assert list(read_records(str(p))) == recs


@pytest.mark.parametrize("where", ["length_crc", "data", "data_crc"])
def test_corrupted_checksum_raises(tmp_path, where):
    p = tmp_path / "x.tfrecord"
    W.write_records(p, [b"hello world", b"second"])
    raw = bytearray(p.read_bytes())
    raw[{"length_crc": 9, "data": 14, "data_crc": 24}[where]] ^= 0x01
    p.write_bytes(bytes(raw))
    with pytest.raises(RecordFormatError, match="checksum"):
        list(read_records(str(p)))


@pytest.mark.parametrize("cut", [5, 12 + 3, 12 + 11 + 2])
def test_truncated_file_raises(tmp_path, cut):
    p = tmp_path / "x.tfrecord"
    W.write_records(p, [b"hello world"])
    p.write_bytes(p.read_bytes()[:cut])
    with pytest.raises(RecordFormatError, match="truncated"):
        list(read_records(str(p)))


# ---- tf.train.Example -------------------------------------------------------------------------------------------------
def test_example_decoding_every_kind():
    ex = parse_example(W.example({
        "b": ("bytes", [b"jpeg", b"", b"\x00\xff"]),
        "i_packed": ("int64", [0, 1, 300, -1, -(1 << 63), (1 << 63) - 1], True),
        "i_unpacked": ("int64", [7, -2, 1 << 40], False),
        "f_packed": ("float", [0.5, -1.25, 3.0e38], True),
        "f_unpacked": ("float", [1.0, float(np.float32(0.1))], False),
        "empty_i": ("int64", []),
    }))
    assert ex["b"] == [b"jpeg", b"", b"\x00\xff"]
    assert ex["i_packed"].dtype == np.int64
    assert ex["i_packed"].tolist() == [0, 1, 300, -1, -(1 << 63), (1 << 63) - 1]
    assert ex["i_unpacked"].tolist() == [7, -2, 1 << 40]
    assert ex["f_packed"].dtype == np.float32
    np.testing.assert_array_equal(ex["f_packed"], np.array([0.5, -1.25, 3.0e38], np.float32))
    np.testing.assert_array_equal(ex["f_unpacked"], np.array([1.0, 0.1], np.float32))
    assert len(ex["empty_i"]) == 0


# ---- text part of _dataset_parser --------------------------------------------------------------------------------------
@pytest.mark.parametrize("do_clean", [True, False])
@pytest.mark.parametrize("max_caption", [5, 80])  # shorter and longer than chunk_text_len
def test_parse_text_matches_oracle(do_clean, max_caption):
    rng = np.random.default_rng(7 + max_caption)
    chunks = W.video_chunks(rng, 6, frame_hw=(8, 8), max_caption=max_caption)
    ex = parse_example(W.chunks_example(chunks))
    got = D.parse_text(ex, 6, 32, do_clean)
    ref = O.dataset_parser_text(chunks, 32, do_clean)
    assert set(got) == set(ref)
    for k in ref:
        assert got[k].dtype == ref[k].dtype, k
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    assert (got["input_ids"][:, 0] == (D.START if do_clean else D.NEXTCAPTION_START)).all()


def test_is_eoc_to_video_src_ids():
    chunks = [{"tokenized_cleaned_asr": [], "tokenized_raw_asr": [], "youtube_id": b"v", "chunk_num": i, "mean_time": 0.0,
               "is_eoc": e} for i, e in enumerate([0, 1, 0, 0, 1, 1, 0, 0])]
    for c in chunks:
        c.update({"image/encoded": b"", "image/height": 1, "image/width": 1})
    got = D.parse_text(parse_example(W.chunks_example(chunks)), 8, 4, True)
    # the last chunk always ends a video; a new video starts after every end
    assert got["is_eoc"].tolist() == [False, True, False, False, True, True, False, True]
    assert got["video_src_ids"].tolist() == [0, 0, 1, 1, 1, 2, 3, 3]


# ---- frame plan --------------------------------------------------------------------------------------------------------
def test_plan_matches_oracle_with_injected_draws():
    rng = np.random.default_rng(3)
    n = 400
    h = rng.integers(20, 900, n)
    w = rng.integers(20, 1600, n)
    h[:3], w[:3] = 288, 512  # what data/process.py writes
    out = (192, 352)
    dr = D.frame_draws(rng, n, {"random_scale_min": 0.5, "random_scale_max": 1.5, "augment_prob": 0.8})
    got = D.plan_frames(h, w, out, dr["scale"], dr["u_y"], dr["u_x"])
    for i in range(n):
        ref = O.resize_plan(h[i], w[i], out, dr["scale"][i], dr["u_y"][i], dr["u_x"][i])
        assert (got["scaled_h"][i], got["scaled_w"][i], got["offset_y"][i], got["offset_x"][i]) == ref, i
    assert {k: v.dtype for k, v in got.items()} == {k: np.dtype(np.int32) for k in got}


def test_frame_draws_ranges():
    d = D.frame_draws(np.random.default_rng(0), 4000, {"random_scale_min": 1.125, "random_scale_max": 1.5, "augment_prob": 0.8})
    assert d["scale"].dtype == np.float32 and (d["scale"] >= 1.125).all() and (d["scale"] < 1.5).all()
    assert set(np.unique(d["method"])) == {0, 1, 2, 3}
    assert set(np.unique(d["augment"])) == {0, 1, 2}
    assert abs((d["augment"] > 0).mean() - 0.8) < 0.03
    assert (d["factor"] >= np.float32(0.68)).all() and (d["factor"] < np.float32(1.32)).all()
    none = D.frame_draws(np.random.default_rng(0), 100, {})
    assert (none["augment"] == 0).all()  # augment_prob defaults to 0: no augmentation, no clip


# ---- input_fn_builder's host-side rules ---------------------------------------------------------------------------------
def _config(train_file, **data):
    d = {"train_file": train_file, "num_chunks": 4}
    d.update(data)
    return NeatConfig.from_dict({"data": d, "model": {"image_size": [32, 48], "num_chunks_in_group": 2},
                                 "optimizer": {}, "device": {"output_dir": "/tmp/unused", "train_batch_size": 4}})


def test_shard_files_by_rank():
    files = [f"f{i}" for i in range(7)]
    shards = [D.shard_files(files, r, 3) for r in range(3)]
    assert shards == [["f0", "f3", "f6"], ["f1", "f4"], ["f2", "f5"]]
    assert D.shard_files(files, 0, 1) == files


def test_fewer_files_than_ranks_raises(tmp_path):
    for i in range(2):
        W.write_records(tmp_path / f"t{i}.tfrecord", [b""])
    cfg = _config(str(tmp_path / "t*.tfrecord"))
    with pytest.raises(ValueError, match="at least one per rank"):
        D.input_fn_builder(cfg, True, rank=0, world=3)


def test_no_train_file_raises(tmp_path):
    with pytest.raises(ValueError, match="matches no file"):
        D.input_fn_builder(_config(str(tmp_path / "none*.tfrecord")), True)


def test_unbatch_size_raises(tmp_path):
    W.write_records(tmp_path / "t.tfrecord", [b""])
    with pytest.raises(NotImplementedError, match="unbatch_size"):
        D.input_fn_builder(_config(str(tmp_path / "t.tfrecord"), unbatch_size=2), True)


# ---- oracle KATs (derived by hand from the kernels' definitions) --------------------------------------------------------
def _img(h, w, seed=0):
    return (np.random.default_rng(seed).integers(0, 256, (h, w, 3)).astype(np.float32) * O.INV255).astype(np.float32)


@pytest.mark.parametrize("method", [0, 1, 2])
@pytest.mark.parametrize("hw", [(7, 11), (13, 5), (4, 4)])
def test_kat_align_corners_maps_corners_exactly(method, hw):
    img = _img(9, 10)
    out = O.RESIZE[method](img, *hw)
    for (oy, ox), (iy, ix) in [((0, 0), (0, 0)), ((0, -1), (0, -1)), ((-1, 0), (-1, 0)), ((-1, -1), (-1, -1))]:
        np.testing.assert_array_equal(out[oy, ox], img[iy, ix])


@pytest.mark.parametrize("method", [0, 1, 2, 3])
@pytest.mark.parametrize("hw", [(5, 9), (17, 23), (1, 1)])
def test_kat_constant_image_stays_constant(method, hw):
    img = np.full((8, 12, 3), np.float32(200) * O.INV255, np.float32)
    out = O.RESIZE[method](img, *hw)
    # bicubic and area weights sum to 1 up to float rounding; bilinear and nearest reproduce the value exactly
    tol = 1e-6 if method in (2, 3) else 0
    np.testing.assert_allclose(out, img[0, 0, 0], rtol=tol, atol=0)


@pytest.mark.parametrize("method", [0, 1, 2])
def test_kat_same_size_is_identity(method):
    img = _img(11, 14, seed=3)
    np.testing.assert_array_equal(O.RESIZE[method](img, 11, 14), img)


def test_kat_bilinear_reproduces_linear_ramp():
    h, w = 9, 17
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.repeat((0.25 * yy / (h - 1) + 0.5 * xx / (w - 1))[..., None], 3, -1).astype(np.float32)
    out = O.resize_bilinear(img, 25, 40)
    oy, ox = np.mgrid[0:25, 0:40].astype(np.float64)
    np.testing.assert_allclose(out[..., 0], 0.25 * oy / 24 + 0.5 * ox / 39, atol=2e-7)


def test_kat_plan_floor_and_padding():
    # a wide 40 x 400 frame asked for 192 x 352 at scale 1: min(352/400, 192/40) = 0.88 gives 35 rows, below the 64-pixel
    # floor, so image_scale = 64/40 = 1.6 -> 64 x 640, the crop keeps 64 rows and the other 128 are zero padding
    sh, sw, oy, ox = O.resize_plan(40, 400, (192, 352), 1.0, 0.5, 0.5)
    assert (sh, sw, oy) == (64, 640, 0) and ox == int(np.float32(640 - 352) * np.float32(0.5))
    got = D.plan_frames([40], [400], (192, 352), [1.0], [0.5], [0.5])
    assert (got["scaled_h"][0], got["scaled_w"][0], got["offset_y"][0], got["offset_x"][0]) == (sh, sw, oy, ox)
    u8 = np.random.default_rng(0).integers(1, 256, (40, 400, 3)).astype(np.uint8)
    out, _ = O.load_and_resize_img(u8, (192, 352), 1.0, 0.5, 0.5, 1, 0, [1, 1, 1])
    assert (out[64:] == 0).all() and (out[:64] > 0).all()
