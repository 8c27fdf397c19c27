"""numpy restatement of the checkpoint delta format (include/bevy_ggrs_b200.h "checkpoint deltas"), built on the
checkpoint restatement (checkpoint_codec.py): block b's vectors are canon(target) XOR canon(base), coded exactly as a
checkpoint's blocks, over ceil(max(rows, base_rows) / 512) blocks.  The GPU encoder's deltas are compared with
``encode`` byte for byte; ``decode`` refuses every malformed delta the engine refuses before its digest check.

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

import struct
from typing import Tuple

import numpy as np

import checkpoint_codec as cc
from checkpoint_codec import BLOCK, CodecError

MAGIC, VERSION = 0x44524742, 1
HEADER = struct.Struct("<IIQiIiIIIIIQQ4QQQQ")   # bgr_checkpoint_delta_header, 120 bytes
HEADER_FIELDS = ("magic", "version", "layout", "frame", "rows", "base_frame", "base_rows", "words", "n_blocks",
                 "n_columns", "fps", "active", "elapsed_ns", "rng", "digest_root", "base_root", "payload_bytes")
assert HEADER.size == 120


def n_blocks_of(rows: int, base_rows: int) -> int:
    return -(-max(rows, base_rows) // BLOCK)


def widen(planes: np.ndarray, mask: np.ndarray, n: int) -> Tuple[np.ndarray, np.ndarray]:
    """A world's blocks followed by zero blocks up to ``n``."""
    extra = n - mask.shape[0]
    return (np.concatenate([planes, np.zeros((extra,) + planes.shape[1:], np.uint32)]),
            np.concatenate([mask, np.zeros((extra, BLOCK), np.uint8)]))


def xor_worlds(target, base, n: int):
    (tp, tm), (bp, bm) = widen(*target, n), widen(*base, n)
    return tp ^ bp, tm ^ bm


def encode(target, base, **header) -> bytes:
    """The delta of two canonical worlds (planes, mask), each with its own block count.  ``header`` gives every field
    but magic, version, words, n_blocks and payload_bytes."""
    n = n_blocks_of(header["rows"], header["base_rows"])
    planes, mask = xor_worlds(target, base, n)
    blocks = [cc.encode_block(planes[b], mask[b]) for b in range(n)]
    offsets = np.concatenate([[0], np.cumsum([len(b) for b in blocks], dtype=np.uint64)]).astype("<u8")
    h = dict(header, magic=MAGIC, version=VERSION, words=planes.shape[1], n_blocks=n, payload_bytes=int(offsets[-1]))
    return pack_header(h) + offsets.tobytes() + b"".join(blocks)


def encoded_size(target, base, rows: int, base_rows: int) -> int:
    """The delta's size, computed per vector without building it (fast at 1M rows)."""
    planes, mask = xor_worlds(target, base, n_blocks_of(rows, base_rows))
    return cc.encoded_size(planes, mask) - cc.HEADER.size + HEADER.size


def pack_header(h: dict) -> bytes:
    vals = [h[f] for f in HEADER_FIELDS]
    rng = vals.pop(HEADER_FIELDS.index("rng"))
    vals[HEADER_FIELDS.index("rng"):HEADER_FIELDS.index("rng")] = list(rng)
    return HEADER.pack(*vals)


def unpack_header(blob: bytes) -> dict:
    if len(blob) < HEADER.size:
        raise CodecError("truncated: shorter than the header")
    v = list(HEADER.unpack_from(blob))
    i = HEADER_FIELDS.index("rng")
    v[i:i + 4] = [tuple(v[i:i + 4])]
    return dict(zip(HEADER_FIELDS, v))


def decode(delta: bytes, base_header: dict, base_planes: np.ndarray, base_mask: np.ndarray, absent: np.ndarray,
           pad: np.ndarray, mask_bits: int) -> Tuple[dict, np.ndarray, np.ndarray]:
    """(header, planes, mask) of the target: ``delta`` applied to the decoded base checkpoint.  Checks everything the
    engine checks before its digest comparison except the layout and fps: the header against the base's, the offsets
    and blocks as a checkpoint's, and the target's canonical form (``pad``: the bits past each plane's element bytes;
    ``mask_bits``: the alive bit and the registered absent bits)."""
    h = unpack_header(delta)
    if h["magic"] != MAGIC:
        raise CodecError("bad magic")
    if h["version"] != VERSION:
        raise CodecError("bad version")
    if h["words"] != base_header["words"]:
        raise CodecError("word count differs")
    if (h["base_frame"], h["base_rows"], h["base_root"]) != (base_header["frame"], base_header["rows"],
                                                             base_header["digest_root"]):
        raise CodecError("another base")
    words, n = h["words"], h["n_blocks"]
    if n != n_blocks_of(h["rows"], h["base_rows"]):
        raise CodecError("n_blocks != ceil(max(rows, base_rows) / 512)")
    prefix = HEADER.size + 8 * (n + 1)
    if len(delta) < prefix:
        raise CodecError("truncated: shorter than the offsets")
    if len(delta) - prefix != h["payload_bytes"]:
        raise CodecError("truncated or overlong")
    off = np.frombuffer(delta, "<u8", n + 1, HEADER.size).astype(np.int64)
    max_block = 4 * ((words + 1 + 3) // 4 + words * BLOCK + cc.MASK_WORDS)
    min_block = 4 * ((words + 1 + 3) // 4 + words + 1)
    d = np.diff(off)
    if off[0] != 0 or off[-1] != h["payload_bytes"] or (d < min_block).any() or (off % 4).any() or (d > max_block).any():
        raise CodecError("bad offsets")
    planes, mask = widen(base_planes, base_mask, n)
    for b in range(n):
        dp, dm = cc.decode_block(delta[prefix + int(off[b]): prefix + int(off[b + 1])], words)
        planes[b] ^= dp
        mask[b] ^= dm
    canon_planes, canon_mask = cc.canonical(planes, mask, h["rows"], absent)
    if not np.array_equal(canon_mask, mask):
        raise CodecError("a mask byte of a row that does not exist")
    if (mask.astype(np.uint32) & ~np.uint32(mask_bits)).any():
        raise CodecError("a presence bit this registration does not use")
    if not np.array_equal(canon_planes, planes):
        raise CodecError("a word of a row that does not exist or lacks the column")
    if (planes & pad[None, :, None]).any():
        raise CodecError("bits past an element's bytes")
    own = -(-h["rows"] // BLOCK)
    return h, planes[:own], mask[:own]
