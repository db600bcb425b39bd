"""TFRecord files and tf.train.Example records, read without TensorFlow -- what tf.data.TFRecordDataset and
tf.io.parse_single_example do for the pretraining input pipeline (model/dataloader.py:33-53,174-176).

  record   uint64 length | uint32 masked_crc32c(length) | data[length] | uint32 masked_crc32c(data)   (little endian;
           tensorflow/core/lib/io/record_reader.cc).  Both checksums are verified; a mismatch or a truncated file raises.
  Example  Example{features=1: Features{feature=1: map<string, Feature>}}, Feature{bytes_list=1 | float_list=2 | int64_list=3}
           (tensorflow/core/example/example.proto, feature.proto); numeric lists may be packed or not.

The varint, CRC-32C and protobuf field walkers are those of the checkpoint reader (tf_checkpoint.py).
"""
from __future__ import annotations

import os
import struct
from typing import Callable, Dict, Iterator, List, Optional, Union

import numpy as np

from .tf_checkpoint import _proto_fields, _signed64, crc32c, mask_crc, read_varint

FeatureValue = Union[List[bytes], np.ndarray]


class RecordFormatError(ValueError):
    pass


def read_records(path: str, keep: Optional[Callable[[], bool]] = None) -> Iterator[Optional[bytes]]:
    """The serialized records of one TFRecord file (uncompressed), in file order.

    With `keep`, it is asked before each record's data is read.  A record it declines has its 12-byte header read and its
    length checksum verified, then its data and data checksum are skipped by seeking: they are never read or checksummed,
    and None is yielded in the record's place.  A skipped record that runs past the end of the file still raises."""
    with open(path, "rb") as f:
        size = os.fstat(f.fileno()).st_size if keep is not None else 0
        while True:
            head = f.read(12)
            if not head:
                return
            if len(head) < 12:
                raise RecordFormatError(f"{path}: truncated record header")
            if struct.unpack("<I", head[8:])[0] != mask_crc(crc32c(head[:8])):
                raise RecordFormatError(f"{path}: record length checksum mismatch")
            (length,) = struct.unpack("<Q", head[:8])
            if keep is not None and not keep():
                if f.seek(length + 4, os.SEEK_CUR) > size:
                    raise RecordFormatError(f"{path}: truncated record")
                yield None
                continue
            data = f.read(length)
            tail = f.read(4)
            if len(data) < length or len(tail) < 4:
                raise RecordFormatError(f"{path}: truncated record")
            if struct.unpack("<I", tail)[0] != mask_crc(crc32c(data)):
                raise RecordFormatError(f"{path}: record data checksum mismatch")
            yield data


def _int64s(wire: int, v) -> List[int]:
    if wire == 0:
        return [_signed64(v)]
    out, pos = [], 0
    while pos < len(v):
        x, pos = read_varint(v, pos)
        out.append(_signed64(x))
    return out


def _feature(buf: bytes) -> FeatureValue:
    for kind, _, lst in _proto_fields(buf):
        if kind == 1:  # BytesList{repeated bytes value = 1}
            return [bytes(v) for f, _, v in _proto_fields(lst) if f == 1]
        if kind == 2:  # FloatList{repeated float value = 1}: packed (wire 2) or one fixed32 per field (wire 5)
            raw = b"".join(bytes(v) for f, _, v in _proto_fields(lst) if f == 1)
            return np.frombuffer(raw, dtype="<f4").astype(np.float32)
        if kind == 3:  # Int64List{repeated int64 value = 1}: packed (wire 2) or one varint per field (wire 0)
            return np.array([x for f, w, v in _proto_fields(lst) if f == 1 for x in _int64s(w, v)], dtype=np.int64)
    return []  # a Feature with no list set reads as an empty bytes list


def parse_example(buf: bytes) -> Dict[str, FeatureValue]:
    """tf.train.Example -> {feature key: list of bytes (bytes_list) | int64 array (int64_list) | float32 array (float_list)}."""
    out = {}
    for f, _, features in _proto_fields(buf):
        if f != 1:
            continue
        for g, _, entry in _proto_fields(features):
            if g != 1:
                continue
            key, value = None, b""
            for h, _, v in _proto_fields(entry):
                if h == 1:
                    key = bytes(v).decode("utf-8")
                elif h == 2:
                    value = v
            if key is None:
                raise RecordFormatError("Example feature map entry without a key")
            out[key] = _feature(value)
    return out
