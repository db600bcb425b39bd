"""TensorFlow V2 checkpoint writer and the `checkpoint` state file (CPU only): round trips through the reader, byte-level checks
of the leveldb table and the bundle protos made independently of the writer's helpers, and the crash-safety order of a save."""
import os
import struct

import numpy as np
import pytest
import torch

from merlot_b200 import tf_checkpoint as T
from tests.test_tf_checkpoint import _write_checkpoint


def _raw(t):
    return t.contiguous().view(torch.uint8).numpy().tobytes() if t.dtype == torch.bfloat16 else t.contiguous().numpy().tobytes()


_DT = {torch.float32: T.DT_FLOAT, torch.bfloat16: T.DT_BFLOAT16, torch.int64: T.DT_INT64}


def _entries(tensors, with_crc=True):
    return [(n, _DT[t.dtype], tuple(t.shape), _raw(t), T.crc32c(_raw(t)) if with_crc else None) for n, t in tensors.items()]


def _tensors(seed=0, n_shared=300):
    g = torch.Generator().manual_seed(seed)
    out = {
        "encoder/layer00/query_layer/kernel": torch.randn(8, 8, generator=g),
        "encoder/layer00/query_layer/kernel/adam_m": torch.randn(8, 8, generator=g).bfloat16(),
        "encoder/layer00/query_layer/kernel/adam_v": -torch.rand(8, 8, generator=g).bfloat16(),
        "global_step": torch.tensor(460000, dtype=torch.int64),
        "vision_backbone/vision_transformer/conv2d/kernel": torch.randn(2, 2, 3, 8, generator=g),
        "empty/fp32": torch.zeros(0, 4),
        "empty/fp32_b": torch.zeros(3, 0),
        "odd/bf16": torch.randn(7, generator=g).bfloat16(),   # puts the next tensor at a 2-byte offset
    }
    stem = "vision_backbone/vision_transformer/resnet50lite/block_group3/" + "x" * 60
    for i in range(n_shared):  # hundreds of names sharing a long prefix
        out[f"{stem}/conv2d_{i}/kernel"] = torch.randn(1 + i % 5, generator=g)
    return out


# ---- independent parsing of the files ---------------------------------------------------------------------------
def _uvarint(buf, pos):
    v, s = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << s
        s += 7
        if b < 0x80:
            return v, pos


def _blocks(index_bytes):
    """Footer -> (metaindex handle, index handle); every block's trailer crc checked; returns the data block handles."""
    footer = index_bytes[-48:]
    assert struct.unpack("<Q", footer[40:])[0] == 0xDB4775248B80FB57
    mo, p = _uvarint(footer, 0)
    ms, p = _uvarint(footer, p)
    io, p = _uvarint(footer, p)
    isz, p = _uvarint(footer, p)
    assert footer[p:40] == bytes(40 - p)

    def block(off, size):
        raw, ctype = index_bytes[off:off + size], index_bytes[off + size]
        assert ctype == 0
        assert struct.unpack_from("<I", index_bytes, off + size + 1)[0] == T.mask_crc(T.crc32c(raw + b"\x00"))
        return raw

    assert block(mo, ms) == struct.pack("<II", 0, 1)  # empty metaindex: one restart point
    handles = [v for _, v in T._block_entries(block(io, isz))]
    data = []
    end = 0
    for h in handles:
        off, p = _uvarint(h, 0)
        size, _ = _uvarint(h, p)
        assert off == end  # blocks tile the file up to the metaindex
        data.append(block(off, size))
        end = off + size + 5
    assert end == mo and mo + ms + 5 == io and io + isz + 5 == len(index_bytes) - 48
    return data


def test_write_bundle_round_trips_and_is_well_formed(tmp_path):
    tensors = _tensors()
    prefix = str(tmp_path / "model.ckpt-3")
    T.write_bundle(prefix, _entries(tensors), block_size=4096)
    assert sorted(os.listdir(tmp_path)) == ["model.ckpt-3.data-00000-of-00001", "model.ckpt-3.index"]  # no temporary left
    got = T.load_checkpoint(prefix, names=list(tensors))
    assert set(got) == set(tensors)
    for n, t in tensors.items():
        assert got[n].dtype == t.dtype and list(got[n].shape) == list(t.shape) and torch.equal(got[n], t), n
    assert T.list_variables(prefix) == sorted((n, list(t.shape)) for n, t in tensors.items())

    index = open(prefix + ".index", "rb").read()
    data = open(prefix + ".data-00000-of-00001", "rb").read()
    blocks = _blocks(index)
    assert len(blocks) >= 4  # several data blocks
    keys = [k for b in blocks for k, _ in T._block_entries(b)]
    assert keys == sorted(keys) and keys[0] == b"" and len(keys) == len(tensors) + 1
    # prefix compression is in use: the shared-prefix names take far less than their full length
    assert len(index) < sum(len(k) for k in keys) // 2
    vals = {k: v for b in blocks for k, v in T._block_entries(b)}
    # header: num_shards 1, endianness absent (LITTLE), version { producer 1 }
    assert vals[b""] == bytes([0x08, 0x01, 0x1A, 0x02, 0x08, 0x01])
    spans = []
    for n, t in tensors.items():
        e = T.parse_entry(vals[n.encode()])
        raw = _raw(t)
        assert e["dtype"] == _DT[t.dtype] and e["shape"] == list(t.shape) and e["shard_id"] == 0
        assert data[e["offset"]:e["offset"] + e["size"]] == raw
        assert e["crc32c"] == T.mask_crc(T.crc32c(raw)), n
        spans.append((e["offset"], e["size"]))
    spans.sort()
    pos = 0
    for off, size in spans:  # the offsets tile the data file exactly
        assert off == pos
        pos += size
    assert pos == len(data)


def test_writer_and_reference_writer_read_identically(tmp_path):
    """The reader gives the same tensors for a bundle of the new writer and one of the test suite's independent writer."""
    tensors = _tensors(seed=1, n_shared=40)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    T.write_bundle(a, _entries(tensors, with_crc=False))  # crc computed by the writer
    _write_checkpoint(b, tensors)
    ga, gb = T.load_checkpoint(a, names=list(tensors)), T.load_checkpoint(b, names=list(tensors))
    assert set(ga) == set(gb) == set(tensors)
    for n in tensors:
        assert ga[n].dtype == gb[n].dtype and torch.equal(ga[n], gb[n]), n
    assert T.load_checkpoint(a).keys() == T.load_checkpoint(b).keys()  # same default (slot-skipping) view


def test_write_bundle_rejects_bad_entries(tmp_path):
    good = ("a", T.DT_FLOAT, (2,), np.zeros(2, np.float32).tobytes(), None)
    with pytest.raises(ValueError, match="bytes for shape"):
        T.write_bundle(str(tmp_path / "x"), [("a", T.DT_FLOAT, (3,), np.zeros(2, np.float32).tobytes(), None)])
    with pytest.raises(ValueError, match="duplicate"):
        T.write_bundle(str(tmp_path / "x"), [good, good])
    with pytest.raises(ValueError, match="dtype"):
        T.write_bundle(str(tmp_path / "x"), [("a", 3, (2,), np.zeros(2, np.int32).tobytes(), None)])
    assert not os.listdir(tmp_path)


def test_checkpoint_state_file(tmp_path):
    d = tmp_path / "out"
    d.mkdir()
    assert T.latest_checkpoint(str(d)) is None  # no state file
    for step in (2, 4):
        T.write_bundle(str(d / f"model.ckpt-{step}"), [("global_step", T.DT_INT64, (), np.int64(step).tobytes(), None)])
        T.update_checkpoint_state(str(d), str(d / f"model.ckpt-{step}"))
    text = (d / "checkpoint").read_text()
    assert text == ('model_checkpoint_path: "model.ckpt-4"\n'
                    'all_model_checkpoint_paths: "model.ckpt-2"\nall_model_checkpoint_paths: "model.ckpt-4"\n')
    assert T.latest_checkpoint(str(d)) == str(d / "model.ckpt-4")
    # an absolute path, as other writers may leave it
    (d / "checkpoint").write_text(f'model_checkpoint_path: "{d / "model.ckpt-2"}"\n')
    assert T.latest_checkpoint(str(d)) == str(d / "model.ckpt-2")
    # a checkpoint outside the directory is recorded by its absolute path
    other = tmp_path / "elsewhere.ckpt-9"
    T.write_bundle(str(other), [("global_step", T.DT_INT64, (), np.int64(9).tobytes(), None)])
    T.update_checkpoint_state(str(d), str(other))
    assert T.latest_checkpoint(str(d)) == str(other)
    # a state file naming a checkpoint whose index is gone
    (d / "checkpoint").write_text('model_checkpoint_path: "model.ckpt-77"\n')
    assert T.latest_checkpoint(str(d)) is None


def test_failed_save_leaves_the_previous_checkpoint_latest(tmp_path, monkeypatch):
    """A save that dies after the data file is in place but before the index is renamed leaves no index under the new prefix,
    no temporary file, and the state file still naming the previous checkpoint."""
    d = str(tmp_path)

    def save(step):
        prefix = os.path.join(d, f"model.ckpt-{step}")
        T.write_bundle(prefix, [("global_step", T.DT_INT64, (), np.int64(step).tobytes(), None),
                                ("w", T.DT_FLOAT, (4,), np.full(4, step, np.float32).tobytes(), None)])
        T.update_checkpoint_state(d, prefix)

    save(2)
    real_replace = os.replace

    def replace(src, dst):
        if str(dst).endswith(".index"):
            raise OSError("disk gone")
        return real_replace(src, dst)

    monkeypatch.setattr(os, "replace", replace)
    with pytest.raises(OSError, match="disk gone"):
        save(4)
    monkeypatch.setattr(os, "replace", real_replace)
    assert os.path.exists(os.path.join(d, "model.ckpt-4.data-00000-of-00001"))
    assert not os.path.exists(os.path.join(d, "model.ckpt-4.index"))
    assert not [f for f in os.listdir(d) if "tempstate" in f]
    latest = T.latest_checkpoint(d)
    assert latest == os.path.join(d, "model.ckpt-2")
    assert int(T.load_checkpoint(latest, names=["global_step"])["global_step"]) == 2
