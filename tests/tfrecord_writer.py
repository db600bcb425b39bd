"""TEST INFRASTRUCTURE ONLY: a writer of the published TFRecord and tf.train.Example formats (record_writer.cc, example.proto,
feature.proto) and of pretraining examples with the reference's chunk_k2f schema (data/process.py:236-256), so that the
reader and the input pipeline are tested on files built from a seed -- nothing binary is committed."""
import io
import struct

import numpy as np

from merlot_b200.tf_checkpoint import crc32c, mask_crc


def varint(v: int) -> bytes:
    v &= (1 << 64) - 1  # negative int64 -> two's complement, ten bytes
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def field(num: int, wire: int, payload: bytes) -> bytes:
    if wire == 2:
        return varint(num << 3 | 2) + varint(len(payload)) + payload
    return varint(num << 3 | wire) + payload


def feature(kind: str, values, packed: bool = True) -> bytes:
    if kind == "bytes":
        return field(1, 2, b"".join(field(1, 2, v) for v in values))
    if kind == "float":
        vals = [struct.pack("<f", v) for v in values]
        body = field(1, 2, b"".join(vals)) if packed else b"".join(field(1, 5, v) for v in vals)
        return field(2, 2, body)
    body = field(1, 2, b"".join(varint(int(v)) for v in values)) if packed else \
        b"".join(field(1, 0, varint(int(v))) for v in values)
    return field(3, 2, body)


def example(features: dict) -> bytes:
    """{key: (kind, values[, packed])} -> serialized tf.train.Example."""
    entries = b"".join(field(1, 2, field(1, 2, k.encode()) + field(2, 2, feature(*spec))) for k, spec in features.items())
    return field(1, 2, entries)


def write_records(path, records):
    with open(path, "wb") as f:
        for r in records:
            head = struct.pack("<Q", len(r))
            f.write(head + struct.pack("<I", mask_crc(crc32c(head))) + r + struct.pack("<I", mask_crc(crc32c(r))))


def jpeg(rng, h: int, w: int, gray: bool = False) -> bytes:
    """A smooth random frame (gradients + noise) as a quality-95 JPEG, like pil_image_to_jpgstring."""
    from PIL import Image
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(yy * rng.uniform(0.5, 2) + xx * rng.uniform(0.5, 2) + rng.uniform(0, 255)) % 256 for _ in range(3)], -1)
    img = np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)
    im = Image.fromarray(img[..., 0] if gray else img, mode="L" if gray else "RGB")
    buf = io.BytesIO()
    im.save(buf, format="JPEG", quality=95)
    return buf.getvalue()


def video_chunks(rng, num_chunks: int, frame_hw=(48, 64), max_caption: int = 40, video: str = "vid", vocab: int = 50000):
    """One example's chunks as plain values (what the oracle's parser takes), frames as JPEG bytes."""
    chunks = []
    for i in range(num_chunks):
        h, w = frame_hw if not callable(frame_hw) else frame_hw(i)
        chunks.append({
            "image/encoded": jpeg(rng, h, w, gray=(i == 1)),
            "image/height": h, "image/width": w,
            "youtube_id": f"{video}{int(rng.integers(1 << 30)):x}".encode(),
            "tokenized_cleaned_asr": rng.integers(7, vocab, int(rng.integers(0, max_caption))).tolist(),
            "tokenized_raw_asr": rng.integers(7, vocab, int(rng.integers(0, max_caption))).tolist(),
            "is_eoc": int(rng.random() < 0.3), "mean_time": float(np.float32(rng.uniform(0, 600))), "chunk_num": i,
        })
    return chunks


def chunks_example(chunks) -> bytes:
    """The c{i:02d}/ keys of data/process.py:236-256."""
    feats = {}
    for i, c in enumerate(chunks):
        p = f"c{i:02d}/"
        feats.update({
            p + "image/encoded": ("bytes", [c["image/encoded"]]),
            p + "image/height": ("int64", [c["image/height"]]),
            p + "image/width": ("int64", [c["image/width"]]),
            p + "image/key/sha256": ("bytes", [b"0" * 64]),
            p + "image/format": ("bytes", [b"jpeg"]),
            p + "youtube_id": ("bytes", [c["youtube_id"]]),
            p + "tokenized_cleaned_asr": ("int64", c["tokenized_cleaned_asr"]),
            p + "tokenized_raw_asr": ("int64", c["tokenized_raw_asr"], i % 2 == 0),
            p + "is_eoc": ("int64", [c["is_eoc"]]),
            p + "mean_time": ("float", [c["mean_time"]]),
            p + "chunk_num": ("int64", [c["chunk_num"]]),
        })
    return example(feats)
