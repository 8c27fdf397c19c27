"""numpy restatement of the world checkpoint format (include/bevy_ggrs_b200.h "world checkpoints"): canonicalisation,
encoding and decoding.  The GPU encoder's blobs are compared with ``encode`` byte for byte; ``decode`` refuses every
malformed blob the engine refuses before its digest check.

A world here is ``planes`` [n_blocks, words, 512] u32 and ``mask`` [n_blocks, 512] u8, tile by tile as the engine
stores it (kernels.cuh: per tile the word planes, then one mask byte per row).

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

import struct
from typing import List, Optional, Sequence, Tuple

import numpy as np

BLOCK = 512
MASK_WORDS = BLOCK // 4
MAGIC, VERSION = 0x43524742, 1
CONST, SPARSE, RAW = 0, 1, 2
HEADER = struct.Struct("<IIQiIIIIIQQ4QQQ")   # bgr_checkpoint_header, 104 bytes
HEADER_FIELDS = ("magic", "version", "layout", "frame", "rows", "words", "n_blocks", "n_columns", "fps", "active",
                 "elapsed_ns", "rng", "digest_root", "payload_bytes")
assert HEADER.size == 104


class CodecError(ValueError):
    """A malformed blob (BGR_ERR_INVALID_ARGUMENT in the engine)."""


def plane_absent(elem_bytes: Sequence[int], optional: Sequence[bool]) -> np.ndarray:
    """The absent bit of the column each word plane belongs to: planes are laid out in registration order, optional
    column k (counting optional columns only) has mask bit 1 + k."""
    out, k = [], 0
    for eb, opt in zip(elem_bytes, optional):
        bit = (2 << k) if opt else 0
        k += 1 if opt else 0
        out += [bit] * ((eb + 3) // 4)
    return np.array(out, np.uint32)


def tiles_from_image(image: np.ndarray, words: int) -> Tuple[np.ndarray, np.ndarray]:
    """Tile-planar image bytes (n_blocks * 512 * (4 * words + 1)) -> (planes, mask)."""
    t = image.reshape(-1, BLOCK * (4 * words + 1))
    planes = t[:, : 4 * words * BLOCK].copy().view("<u4").reshape(-1, words, BLOCK)
    return planes, t[:, 4 * words * BLOCK:].copy()


def canonical(planes: np.ndarray, mask: np.ndarray, rows: int, absent: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Zero every word of a row that does not exist or lacks the column, and the mask byte of a row that does not
    exist (r >= rows or alive bit clear)."""
    n_blocks = mask.shape[0]
    r = np.arange(n_blocks * BLOCK).reshape(n_blocks, BLOCK)
    exists = (r < rows) & ((mask & 1) != 0)
    m = np.where(exists, mask, 0).astype(np.uint8)
    keep = exists[:, None, :] & ((m[:, None, :].astype(np.uint32) & absent[None, :, None]) == 0)
    return np.where(keep, planes, 0).astype(np.uint32), m


def vectors(planes_b: np.ndarray, mask_b: np.ndarray) -> List[np.ndarray]:
    """The words + 1 vectors of one block: its word planes, then the mask plane as 128 little-endian u32."""
    return [planes_b[w] for w in range(planes_b.shape[0])] + [mask_b.view("<u4").copy()]


def kind_of(v: np.ndarray) -> int:
    n = v.size
    if (v == v[0]).all():
        return CONST
    return SPARSE if np.count_nonzero(v) < n - n // 32 else RAW


def encode_block(planes_b: np.ndarray, mask_b: np.ndarray) -> bytes:
    vs = vectors(planes_b, mask_b)
    kinds = [kind_of(v) for v in vs]
    head = bytes(kinds) + bytes(-len(kinds) % 4)
    body = []
    for k, v in zip(kinds, vs):
        if k == CONST:
            body.append(v[:1])
        elif k == RAW:
            body.append(v)
        else:
            bits = (v != 0).reshape(-1, 32)
            bitmap = (bits.astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
            body += [bitmap, v[v != 0]]
    return head + b"".join(b.astype("<u4").tobytes() for b in body)


def encoded_size(planes: np.ndarray, mask: np.ndarray) -> int:
    """The blob's size for a canonical world, computed per vector without building it (fast at 1M rows)."""
    n_blocks, words = planes.shape[0], planes.shape[1]
    total = HEADER.size + 8 * (n_blocks + 1)
    vecs = [planes[:, w, :] for w in range(words)] + [np.ascontiguousarray(mask).view("<u4").reshape(n_blocks, MASK_WORDS)]
    body = 4 * ((words + 1 + 3) // 4) * n_blocks
    for v in vecs:
        n = v.shape[1]
        const = (v == v[:, :1]).all(axis=1)
        nnz = np.count_nonzero(v, axis=1)
        size = np.where(const, 1, np.where(nnz < n - n // 32, n // 32 + nnz, n))
        body += 4 * int(size.sum())
    return total + body


def encode(planes: np.ndarray, mask: np.ndarray, **header) -> bytes:
    """The blob of a canonical world.  ``header`` gives every field but magic, version, n_blocks, words and
    payload_bytes, which follow from the data."""
    n_blocks, words = mask.shape[0], planes.shape[1]
    blocks = [encode_block(planes[b], mask[b]) for b in range(n_blocks)]
    offsets = np.concatenate([[0], np.cumsum([len(b) for b in blocks], dtype=np.uint64)]).astype("<u8")
    h = dict(header, magic=MAGIC, version=VERSION, words=words, n_blocks=n_blocks, payload_bytes=int(offsets[-1]))
    return pack_header(h) + offsets.tobytes() + b"".join(blocks)


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


def decode_block(buf: bytes, words: int) -> Tuple[np.ndarray, np.ndarray]:
    """One block's bytes -> (planes [words, 512], mask [512]), as written (not canonicalised)."""
    a = np.frombuffer(buf, "<u4")
    kw = (words + 1 + 3) // 4
    if a.size < kw:
        raise CodecError("block shorter than its kind bytes")
    kb = a[:kw].view(np.uint8)
    kinds, pad = kb[: words + 1], kb[words + 1:]
    if (kinds > RAW).any():
        raise CodecError("kind byte > 2")
    if pad.any():
        raise CodecError("non-zero padding")
    pos, vs = kw, []
    for i, k in enumerate(kinds):
        n = BLOCK if i < words else MASK_WORDS
        if k == CONST:
            if pos + 1 > a.size:
                raise CodecError("block shorter than its kinds imply")
            vs.append(np.full(n, a[pos], np.uint32))
            pos += 1
        elif k == RAW:
            if pos + n > a.size:
                raise CodecError("block shorter than its kinds imply")
            vs.append(a[pos:pos + n].astype(np.uint32))
            pos += n
        else:
            if pos + n // 32 > a.size:
                raise CodecError("bitmap outside the block")
            bm = a[pos:pos + n // 32]
            bits = ((bm[:, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(-1)
            nnz = int(bits.sum())
            if pos + n // 32 + nnz > a.size:
                raise CodecError("block shorter than its bitmaps imply")
            v = np.zeros(n, np.uint32)
            v[bits] = a[pos + n // 32: pos + n // 32 + nnz]
            vs.append(v)
            pos += n // 32 + nnz
    if pos != a.size:
        raise CodecError("block longer than its kinds and bitmaps imply")
    return np.stack(vs[:words]) if words else np.zeros((0, BLOCK), np.uint32), vs[words].astype("<u4").view(np.uint8)


def decode(blob: bytes, words: Optional[int] = None) -> Tuple[dict, np.ndarray, np.ndarray]:
    """(header, planes, mask) of a blob; ``words``: the word count the reader expects.  Checks everything the engine
    checks before its digest comparison, except the layout and fps, which need an engine."""
    h = unpack_header(blob)
    if h["magic"] != MAGIC:
        raise CodecError("bad magic")
    if h["version"] != VERSION:
        raise CodecError("bad version")
    if words is not None and h["words"] != words:
        raise CodecError("word count differs")
    words, n = h["words"], h["n_blocks"]
    if n != -(-h["rows"] // BLOCK):
        raise CodecError("n_blocks != ceil(rows / 512)")
    prefix = HEADER.size + 8 * (n + 1)
    if len(blob) < prefix:
        raise CodecError("truncated: shorter than the offsets")
    if len(blob) - prefix != h["payload_bytes"]:
        raise CodecError("truncated or overlong")
    off = np.frombuffer(blob, "<u8", n + 1, HEADER.size).astype(np.int64)
    max_block = 4 * ((words + 1 + 3) // 4 + words * BLOCK + MASK_WORDS)
    min_block = 4 * ((words + 1 + 3) // 4 + words + 1)   # every vector CONST
    d = np.diff(off)
    if off[0] != 0 or off[-1] != h["payload_bytes"] or (d < min_block).any() or (off % 4).any() or (d > max_block).any():
        raise CodecError("bad offsets")
    planes = np.zeros((n, words, BLOCK), np.uint32)
    mask = np.zeros((n, BLOCK), np.uint8)
    for b in range(n):
        planes[b], mask[b] = decode_block(blob[prefix + int(off[b]): prefix + int(off[b + 1])], words)
    return h, planes, mask
