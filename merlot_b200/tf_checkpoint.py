"""Reader for TensorFlow "tensor bundle" (V2) checkpoints -- SURVEY.md 8(f) next-row 2.

The reference initialises from a checkpoint by NAME (utils/model_utils.py:388-413 `get_assignment_map_from_checkpoint`:
every checkpoint variable whose name also exists in the graph is loaded, the rest keep their initialisers) through
`tf.train.list_variables` / `tf.train.init_from_checkpoint` (model/modeling.py:724-740).  TensorFlow is not installable
here, so this module reads the on-disk format directly:

  <prefix>.index                    a leveldb-format table (SSTable): key "" -> BundleHeaderProto, key <variable name> ->
                                    BundleEntryProto {dtype, shape, shard_id, offset, size, crc32c}
  <prefix>.data-SSSSS-of-NNNNN      the raw little-endian tensor bytes, addressed by (shard_id, offset, size)

`list_variables(prefix)` mirrors tf.train.list_variables; `load_checkpoint(prefix)` returns {name: torch.Tensor};
`ParamStore.load_tf_dict(..., strict=False)` applies the reference's by-name semantics.  `write_bundle` writes the same
format (what ParamStore.save_checkpoint uses), and `update_checkpoint_state` / `latest_checkpoint` keep the `checkpoint`
state file of a model directory.

UNPINNED against TensorFlow-written files: no checkpoint and no TensorFlow exist in this environment; the reader follows
the published formats (leveldb table_format.md, tensorflow/core/protobuf/tensor_bundle.proto, tensor_shape.proto, snappy
format_description.txt) and is tested against a writer of the same formats in tests/ plus known-answer vectors for the
varint, CRC-32C and Snappy pieces.
"""
from __future__ import annotations

import os
import struct
from typing import Dict, Iterable, List, Optional, Tuple

import numpy as np
import torch

TABLE_MAGIC = 0xDB4775248B80FB57  # leveldb kTableMagicNumber
FOOTER_LEN = 48                    # two block handles padded to 40 bytes + 8-byte magic

# tensorflow/core/framework/types.proto
_DTYPES = {1: np.dtype("<f4"), 2: np.dtype("<f8"), 3: np.dtype("<i4"), 4: np.dtype("u1"), 5: np.dtype("<i2"), 6: np.dtype("i1"),
           9: np.dtype("<i8"), 10: np.dtype("?"), 17: np.dtype("<u2"), 19: np.dtype("<f2"), 22: np.dtype("<u4"), 23: np.dtype("<u8")}
DT_BFLOAT16 = 14


class CheckpointFormatError(ValueError):
    pass


# ---------------------------------------------------------------------------------------------------------------
# primitives
# ---------------------------------------------------------------------------------------------------------------
def read_varint(buf: bytes, pos: int) -> Tuple[int, int]:
    """LEB128 unsigned varint (protobuf / leveldb): returns (value, next position)."""
    result, shift = 0, 0
    while True:
        if pos >= len(buf):
            raise CheckpointFormatError("truncated varint")
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7
        if shift > 63:
            raise CheckpointFormatError("varint longer than 64 bits")


def _crc32c_table() -> List[int]:
    tab = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        tab.append(c)
    return tab


_CRC_TABLE = _crc32c_table()


def _crc32c_scalar(data, c: int) -> int:  # raw register update (no init / final xor)
    for b in data:
        c = _CRC_TABLE[(c ^ b) & 0xFF] ^ (c >> 8)
    return c


_CRC_LANE = 4096  # bytes per lane of the vectorised path
_CRC_NP = None    # (byte table as uint32 array, 4 x 256 "advance the register by _CRC_LANE zero bytes" tables)


def _crc32c_np_tables():
    global _CRC_NP
    if _CRC_NP is None:
        tab = np.array(_CRC_TABLE, dtype=np.uint32)
        # the register update is linear over GF(2): advance the 32 basis registers through _CRC_LANE zero bytes ...
        basis = (np.uint32(1) << np.arange(32, dtype=np.uint32)).astype(np.uint32)
        for _ in range(_CRC_LANE):
            basis = tab[basis & np.uint32(0xFF)] ^ (basis >> np.uint32(8))
        # ... and fold them into one 256-entry table per register byte
        shift = np.zeros((4, 256), dtype=np.uint32)
        for byte in range(4):
            for v in range(256):
                acc = np.uint32(0)
                for bit in range(8):
                    if v >> bit & 1:
                        acc ^= basis[8 * byte + bit]
                shift[byte, v] = acc
        _CRC_NP = (tab, shift)
    return _CRC_NP


def crc32c(data, crc: int = 0) -> int:
    """CRC-32C (Castagnoli), the checksum of leveldb blocks and bundle entries.  crc32c(b"123456789") == 0xE3069283.
    Buffers of 64 KiB and more take a vectorised path: the buffer is cut into lanes of 4 KiB whose registers advance together
    (one table lookup per byte position for ALL lanes), and the lane results are chained with the precomputed linear map
    "advance a register through 4 KiB of zeros" -- ~65 MB/s in NumPy against ~5 MB/s for the byte loop, which matters for
    the ~1 GB of variables in a MERLOT checkpoint."""
    c = crc ^ 0xFFFFFFFF
    n = len(data)
    if n < (1 << 16):
        return _crc32c_scalar(bytes(data), c) ^ 0xFFFFFFFF
    tab, shift = _crc32c_np_tables()
    buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data.reshape(-1).view(np.uint8)
    lanes = n // _CRC_LANE
    cols = np.ascontiguousarray(buf[:lanes * _CRC_LANE].reshape(lanes, _CRC_LANE).T)  # [_CRC_LANE, lanes]: one row per byte position
    reg = np.zeros(lanes, dtype=np.uint32)
    m = np.uint32(0xFF)
    e = np.uint32(8)
    for j in range(_CRC_LANE):
        reg = tab[(reg ^ cols[j]) & m] ^ (reg >> e)
    for p in reg.tolist():  # chain: register after lane i = advance(register before) ^ lane-local register
        c = int(shift[0, c & 0xFF] ^ shift[1, (c >> 8) & 0xFF] ^ shift[2, (c >> 16) & 0xFF] ^ shift[3, c >> 24]) ^ p
    return _crc32c_scalar(buf[lanes * _CRC_LANE:].tobytes(), c) ^ 0xFFFFFFFF


def mask_crc(crc: int) -> int:
    """leveldb / TensorFlow store crcs "masked": rotate right by 15 and add a constant."""
    return ((((crc >> 15) | (crc << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def snappy_uncompress(data: bytes) -> bytes:
    """Raw Snappy block decoder (leveldb compression type 1): varint length, then literal / copy elements."""
    n, pos = read_varint(data, 0)
    out = bytearray()
    while pos < len(data):
        tag = data[pos]
        pos += 1
        kind = tag & 3
        if kind == 0:  # literal
            ln = tag >> 2
            if ln >= 60:
                nb = ln - 59
                ln = int.from_bytes(data[pos:pos + nb], "little")
                pos += nb
            ln += 1
            out += data[pos:pos + ln]
            pos += ln
            continue
        if kind == 1:  # copy, 1-byte offset
            ln = ((tag >> 2) & 7) + 4
            off = ((tag >> 5) << 8) | data[pos]
            pos += 1
        elif kind == 2:  # copy, 2-byte offset
            ln = (tag >> 2) + 1
            off = int.from_bytes(data[pos:pos + 2], "little")
            pos += 2
        else:  # copy, 4-byte offset
            ln = (tag >> 2) + 1
            off = int.from_bytes(data[pos:pos + 4], "little")
            pos += 4
        if off == 0 or off > len(out):
            raise CheckpointFormatError("snappy: bad copy offset")
        for _ in range(ln):  # copies may overlap their own output
            out.append(out[-off])
    if len(out) != n:
        raise CheckpointFormatError(f"snappy: expected {n} bytes, produced {len(out)}")
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------
# leveldb table
# ---------------------------------------------------------------------------------------------------------------
def _read_block(buf: bytes, offset: int, size: int, verify: bool) -> bytes:
    if offset + size + 5 > len(buf):
        raise CheckpointFormatError("block handle points past the end of the index file")
    raw = buf[offset:offset + size]
    ctype = buf[offset + size]
    if verify:
        stored = struct.unpack_from("<I", buf, offset + size + 1)[0]
        if stored != mask_crc(crc32c(buf[offset:offset + size + 1])):
            raise CheckpointFormatError("block checksum mismatch")
    if ctype == 0:
        return raw
    if ctype == 1:
        return snappy_uncompress(raw)
    raise CheckpointFormatError(f"unknown block compression type {ctype}")


def _block_entries(block: bytes) -> Iterable[Tuple[bytes, bytes]]:
    """(key, value) pairs of one block: prefix-compressed entries followed by the restart array."""
    if len(block) < 4:
        raise CheckpointFormatError("block too small")
    num_restarts = struct.unpack_from("<I", block, len(block) - 4)[0]
    end = len(block) - 4 - 4 * num_restarts
    if end < 0:
        raise CheckpointFormatError("bad restart array")
    pos, key = 0, b""
    while pos < end:
        shared, pos = read_varint(block, pos)
        non_shared, pos = read_varint(block, pos)
        vlen, pos = read_varint(block, pos)
        if shared > len(key) or pos + non_shared + vlen > end:
            raise CheckpointFormatError("corrupt block entry")
        key = key[:shared] + block[pos:pos + non_shared]
        pos += non_shared
        yield key, block[pos:pos + vlen]
        pos += vlen


def read_table(path: str, verify_checksums: bool = True) -> List[Tuple[bytes, bytes]]:
    """All (key, value) pairs of a leveldb-format table file, in key order."""
    with open(path, "rb") as f:
        buf = f.read()
    if len(buf) < FOOTER_LEN:
        raise CheckpointFormatError(f"{path}: too short for a table footer")
    footer = buf[-FOOTER_LEN:]
    if struct.unpack_from("<Q", footer, 40)[0] != TABLE_MAGIC:
        raise CheckpointFormatError(f"{path}: not a leveldb table (bad magic) -- is this a V1 checkpoint?")
    pos = 0
    _, pos = read_varint(footer, pos)  # metaindex offset
    _, pos = read_varint(footer, pos)  # metaindex size
    idx_off, pos = read_varint(footer, pos)
    idx_size, pos = read_varint(footer, pos)
    out: List[Tuple[bytes, bytes]] = []
    for _, handle in _block_entries(_read_block(buf, idx_off, idx_size, verify_checksums)):
        off, p = read_varint(handle, 0)
        size, _ = read_varint(handle, p)
        out.extend(_block_entries(_read_block(buf, off, size, verify_checksums)))
    return out


# ---------------------------------------------------------------------------------------------------------------
# protobuf messages of tensor_bundle.proto (hand-decoded: the generated classes ship with TensorFlow only)
# ---------------------------------------------------------------------------------------------------------------
def _proto_fields(buf: bytes) -> Iterable[Tuple[int, int, object]]:
    pos = 0
    while pos < len(buf):
        tag, pos = read_varint(buf, pos)
        field, wire = tag >> 3, tag & 7
        if wire == 0:
            v, pos = read_varint(buf, pos)
        elif wire == 1:
            v = buf[pos:pos + 8]
            pos += 8
        elif wire == 2:
            ln, pos = read_varint(buf, pos)
            v = buf[pos:pos + ln]
            pos += ln
        elif wire == 5:
            v = buf[pos:pos + 4]
            pos += 4
        else:
            raise CheckpointFormatError(f"unsupported protobuf wire type {wire}")
        yield field, wire, v


def _signed64(v: int) -> int:
    return v - (1 << 64) if v >= (1 << 63) else v


def parse_header(buf: bytes) -> Dict[str, int]:
    """BundleHeaderProto: num_shards = 1, endianness = 2 (0 little), version = 3."""
    h = {"num_shards": 0, "endianness": 0}
    for field, _, v in _proto_fields(buf):
        if field == 1:
            h["num_shards"] = int(v)
        elif field == 2:
            h["endianness"] = int(v)
    return h


def parse_entry(buf: bytes) -> Dict[str, object]:
    """BundleEntryProto: dtype = 1, shape = 2 (TensorShapeProto{dim = 2 {size = 1}}), shard_id = 3, offset = 4, size = 5,
    crc32c = 6 (fixed32), slices = 7."""
    e: Dict[str, object] = {"dtype": 0, "shape": [], "shard_id": 0, "offset": 0, "size": 0, "crc32c": None, "slices": 0}
    for field, wire, v in _proto_fields(buf):
        if field == 1:
            e["dtype"] = int(v)
        elif field == 2:
            dims = []
            for f2, _, v2 in _proto_fields(v):
                if f2 == 2:  # Dim
                    size = 0
                    for f3, _, v3 in _proto_fields(v2):
                        if f3 == 1:
                            size = _signed64(int(v3))
                    dims.append(size)
                elif f2 == 3 and int(v2):
                    raise CheckpointFormatError("tensor of unknown rank in checkpoint")
            e["shape"] = dims
        elif field == 3:
            e["shard_id"] = int(v)
        elif field == 4:
            e["offset"] = _signed64(int(v))
        elif field == 5:
            e["size"] = _signed64(int(v))
        elif field == 6 and wire == 5:
            e["crc32c"] = struct.unpack("<I", v)[0]
        elif field == 7:
            e["slices"] = int(e["slices"]) + 1
    return e


# ---------------------------------------------------------------------------------------------------------------
# public API
# ---------------------------------------------------------------------------------------------------------------
def _index(prefix: str, verify: bool):
    path = prefix + ".index"
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path}: no V2 checkpoint index (pass the checkpoint PREFIX, e.g. .../model.ckpt-460000)")
    header, entries = None, {}
    for key, value in read_table(path, verify):
        if key == b"":
            header = parse_header(value)
        else:
            entries[key.decode("utf-8")] = parse_entry(value)
    if header is None:
        raise CheckpointFormatError(f"{path}: missing bundle header")
    if header["endianness"] != 0:
        raise CheckpointFormatError("big-endian checkpoints are not supported")
    return header, entries


def list_variables(prefix: str, verify_checksums: bool = True) -> List[Tuple[str, List[int]]]:
    """tf.train.list_variables: [(name, shape)] sorted by name."""
    _, entries = _index(prefix, verify_checksums)
    return [(n, list(e["shape"])) for n, e in sorted(entries.items())]


def load_checkpoint(prefix: str, names: Optional[Iterable[str]] = None, verify_checksums: bool = True,
                    skip_optimizer_slots: bool = True) -> Dict[str, torch.Tensor]:
    """{variable name: tensor}.  `names` restricts the read; Adam slots (`.../adam_m`, `.../adam_v`) and `global_step` are
    skipped by default -- the reference only restores model variables that exist in the graph (model_utils.py:388-413)."""
    header, entries = _index(prefix, verify_checksums)
    want = set(names) if names is not None else None
    shards: Dict[int, np.memmap] = {}
    out: Dict[str, torch.Tensor] = {}
    for name, e in sorted(entries.items()):
        if want is not None and name not in want:
            continue
        if want is None and skip_optimizer_slots and (name.endswith("/adam_m") or name.endswith("/adam_v") or name == "global_step"):
            continue
        if e["slices"]:
            raise NotImplementedError(f"{name}: partitioned (sliced) variables are not supported")
        dt = int(e["dtype"])
        if dt != DT_BFLOAT16 and dt not in _DTYPES:
            continue  # strings / resources / variants: nothing a parameter arena can hold
        sid = int(e["shard_id"])
        if sid not in shards:
            shards[sid] = np.memmap(f"{prefix}.data-{sid:05d}-of-{header['num_shards']:05d}", dtype=np.uint8, mode="r")
        raw = shards[sid][int(e["offset"]):int(e["offset"]) + int(e["size"])].tobytes()
        if len(raw) != int(e["size"]):
            raise CheckpointFormatError(f"{name}: data shard is shorter than the index says")
        if verify_checksums and e["crc32c"] is not None and mask_crc(crc32c(raw)) != e["crc32c"]:
            raise CheckpointFormatError(f"{name}: tensor checksum mismatch")
        shape = [int(d) for d in e["shape"]]
        if dt == DT_BFLOAT16:
            t = torch.frombuffer(bytearray(raw), dtype=torch.bfloat16).reshape(shape)
        else:
            arr = np.frombuffer(raw, dtype=_DTYPES[dt]).reshape(shape)
            t = torch.from_numpy(arr.copy())
        out[name] = t
    return out


# ---------------------------------------------------------------------------------------------------------------
# writer (the same formats; what tf.train.Saver writes for a single-shard V2 checkpoint)
# ---------------------------------------------------------------------------------------------------------------
DT_FLOAT = 1
DT_INT64 = 9
_ITEMSIZE = {DT_FLOAT: 4, DT_BFLOAT16: 2, DT_INT64: 8}
BLOCK_SIZE = 262144       # TensorFlow's table::Options.block_size: a data block is closed once it reaches this many bytes
RESTART_INTERVAL = 16     # table::Options.block_restart_interval


def _varint(v: int) -> bytes:
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _pb(field: int, wire: int, payload: bytes) -> bytes:
    return _varint((field << 3) | wire) + payload


def _pb_bytes(field: int, payload: bytes) -> bytes:
    return _pb(field, 2, _varint(len(payload)) + payload)


def _header_proto() -> bytes:
    """BundleHeaderProto{num_shards: 1, endianness: LITTLE (0, the proto3 default, not serialised), version{producer: 1}}."""
    return _pb(1, 0, _varint(1)) + _pb_bytes(3, _pb(1, 0, _varint(1)))


def _entry_proto(dtype: int, shape, offset: int, size: int, masked_crc: int) -> bytes:
    """BundleEntryProto of shard 0; proto3 leaves zero scalars out, the crc32c is always written."""
    dims = b"".join(_pb_bytes(2, _pb(1, 0, _varint(d)) if d else b"") for d in shape)
    out = _pb(1, 0, _varint(dtype)) + _pb_bytes(2, dims)
    if offset:
        out += _pb(4, 0, _varint(offset))
    if size:
        out += _pb(5, 0, _varint(size))
    return out + _pb(6, 5, struct.pack("<I", masked_crc))


def _block(items: List[Tuple[bytes, bytes]], restart_interval: int) -> bytes:
    """leveldb block: prefix-compressed entries with a full key every `restart_interval` entries, then the restart array."""
    buf, restarts, last = bytearray(), [], b""
    for i, (k, v) in enumerate(items):
        shared = 0
        if i % restart_interval == 0:
            restarts.append(len(buf))
        else:
            n = min(len(k), len(last))
            while shared < n and k[shared] == last[shared]:
                shared += 1
        buf += _varint(shared) + _varint(len(k) - shared) + _varint(len(v)) + k[shared:] + v
        last = k
    for r in restarts or [0]:  # an empty block still has one restart point (leveldb BlockBuilder)
        buf += struct.pack("<I", r)
    buf += struct.pack("<I", len(restarts or [0]))
    return bytes(buf)


def table_bytes(items: List[Tuple[bytes, bytes]], block_size: int = BLOCK_SIZE) -> bytes:
    """A leveldb table of (key, value) pairs in strictly increasing key order: uncompressed data blocks, an empty metaindex
    block, an index block whose keys are each data block's last key, every block followed by its type byte and masked CRC,
    and the 48-byte footer."""
    out = bytearray()

    def emit(block: bytes) -> bytes:
        off = len(out)
        out.extend(block)
        out.append(0)  # kNoCompression
        out.extend(struct.pack("<I", mask_crc(crc32c(block + b"\x00"))))
        return _varint(off) + _varint(len(block))

    index, pending, size = [], [], 0
    for i, (k, v) in enumerate(items):
        if i and k <= items[i - 1][0]:
            raise ValueError(f"table keys must be strictly increasing: {items[i - 1][0]!r} then {k!r}")
        pending.append((k, v))
        size += len(k) + len(v) + 8
        if size >= block_size:
            index.append((pending[-1][0], emit(_block(pending, RESTART_INTERVAL))))
            pending, size = [], 0
    if pending:
        index.append((pending[-1][0], emit(_block(pending, RESTART_INTERVAL))))
    meta = emit(_block([], 1))
    idx = emit(_block(index, 1))
    footer = meta + idx
    return bytes(out) + footer + b"\x00" * (40 - len(footer)) + struct.pack("<Q", TABLE_MAGIC)


def _fsync_dir(path: str) -> None:
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def write_bundle(prefix: str, entries, block_size: int = BLOCK_SIZE) -> None:
    """Write the single-shard V2 checkpoint `<prefix>.data-00000-of-00001` + `<prefix>.index`.

    `entries`: (name, dtype, shape, data, crc32c) with dtype DT_FLOAT, DT_BFLOAT16 or DT_INT64, `data` the tensor's
    little-endian bytes (bytes or any buffer, e.g. a slice of a pinned host array) and `crc32c` its unmasked CRC-32C or None
    to compute it here.  The data file holds the tensors back to back in the given order; the index lists them by name.
    Both files are written under temporary names and fsynced; the data file is renamed into place first and the index last,
    so an interrupted write never leaves an index that points into a missing or partial data file."""
    d = os.path.dirname(os.path.abspath(prefix))
    data_path, index_path = f"{prefix}.data-00000-of-00001", f"{prefix}.index"
    items, offset, names = [(b"", _header_proto())], 0, set()
    for name, dtype, shape, data, crc in entries:
        if dtype not in _ITEMSIZE:
            raise ValueError(f"{name}: unsupported dtype {dtype}")
        if name == "" or name in names:
            raise ValueError(f"duplicate or empty tensor name {name!r}")
        names.add(name)
        size = memoryview(data).nbytes
        if size != _ITEMSIZE[dtype] * int(np.prod(shape, dtype=np.int64)):
            raise ValueError(f"{name}: {size} bytes for shape {list(shape)} of dtype {dtype}")
        if crc is None:
            crc = crc32c(data)
        items.append((name.encode("utf-8"), _entry_proto(dtype, [int(s) for s in shape], offset, size, mask_crc(int(crc)))))
        offset += size
    items.sort(key=lambda kv: kv[0])
    index = table_bytes(items, block_size)
    tag = f".tempstate{os.getpid()}"
    try:
        with open(data_path + tag, "wb") as f:
            for _, _, _, data, _ in entries:
                f.write(data)
            f.flush()
            os.fsync(f.fileno())
        with open(index_path + tag, "wb") as f:
            f.write(index)
            f.flush()
            os.fsync(f.fileno())
        os.replace(data_path + tag, data_path)
        os.replace(index_path + tag, index_path)
    finally:
        for p in (data_path + tag, index_path + tag):
            if os.path.exists(p):
                os.remove(p)
    _fsync_dir(d)


# ---------------------------------------------------------------------------------------------------------------
# the `checkpoint` state file (tf.train.CheckpointState as a text proto)
# ---------------------------------------------------------------------------------------------------------------
STATE_FILE = "checkpoint"


def _quote(s: str) -> str:
    return '"' + s.replace("\\", "\\\\").replace('"', '\\"') + '"'


def _read_state(directory: str) -> Tuple[Optional[str], List[str]]:
    path = os.path.join(directory, STATE_FILE)
    if not os.path.exists(path):
        return None, []
    latest, every = None, []
    with open(path, "r", encoding="utf-8") as f:
        for line in f:
            key, sep, val = line.strip().partition(":")
            val = val.strip()
            if not sep or len(val) < 2 or val[0] != '"' or val[-1] != '"':
                continue
            val = val[1:-1].replace('\\"', '"').replace("\\\\", "\\")
            if key == "model_checkpoint_path":
                latest = val
            elif key == "all_model_checkpoint_paths":
                every.append(val)
    return latest, every


def update_checkpoint_state(directory: str, prefix: str) -> None:
    """Name `prefix` the latest checkpoint of `directory` and append it to all_model_checkpoint_paths (every earlier one is
    kept).  Paths inside `directory` are written relative to it.  The file is replaced atomically: call this only once the
    bundle itself is durable, so that a crash during a save leaves the previous checkpoint as the latest."""
    d = os.path.abspath(directory)
    p = os.path.abspath(prefix)
    rel = os.path.relpath(p, d) if os.path.commonpath([d, p]) == d else p
    _, every = _read_state(d)
    every = [x for x in every if x != rel] + [rel]
    text = f"model_checkpoint_path: {_quote(rel)}\n" + "".join(f"all_model_checkpoint_paths: {_quote(x)}\n" for x in every)
    path = os.path.join(d, STATE_FILE)
    tmp = path + f".tmp{os.getpid()}"
    with open(tmp, "w", encoding="utf-8") as f:
        f.write(text)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)
    _fsync_dir(d)


def latest_checkpoint(directory: str) -> Optional[str]:
    """tf.train.latest_checkpoint: the prefix the state file names (relative paths are taken relative to `directory`), or
    None when there is no state file or its checkpoint has no index file."""
    latest, _ = _read_state(directory)
    if not latest:
        return None
    p = latest if os.path.isabs(latest) else os.path.join(directory, latest)
    return p if os.path.exists(p + ".index") else None


def checkpoint_prefixes(directory: str) -> List[str]:
    """Every checkpoint the state file of `directory` names (all_model_checkpoint_paths, then model_checkpoint_path), once
    each and resolved like latest_checkpoint, that still has its index file."""
    latest, every = _read_state(directory)
    out = []
    for p in every + ([latest] if latest else []):
        p = p if os.path.isabs(p) else os.path.join(directory, p)
        if p not in out and os.path.exists(p + ".index"):
            out.append(p)
    return out
