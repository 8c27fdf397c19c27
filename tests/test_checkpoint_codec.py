"""CPU: the world checkpoint format restated in numpy (checkpoint_codec.py) round-trips, picks each vector's kind at the
documented thresholds, refuses malformed blobs, and the header's ctypes layout matches the C header."""
import ctypes as C
import struct

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.stress import synth_particles
import checkpoint_codec as cc

HDR = dict(layout=0x1234, frame=17, rows=0, n_columns=3, fps=60, active=0, elapsed_ns=99, rng=(1, 2, 3, 4), digest_root=7)


def _world(rng, rows, words, absent, dead=0.1, fill=0.5):
    n = -(-rows // cc.BLOCK)
    planes = np.where(rng.random((n, words, cc.BLOCK)) < fill, rng.integers(1, 2**32, (n, words, cc.BLOCK)), 0).astype(np.uint32)
    mask = (rng.random((n, cc.BLOCK)) >= dead).astype(np.uint8)
    mask |= (rng.integers(0, 4, (n, cc.BLOCK)) << 1).astype(np.uint8)   # absent bits of two optional columns
    return cc.canonical(planes, mask, rows, absent)


def _roundtrip(planes, mask, rows):
    blob = cc.encode(planes, mask, **{**HDR, "rows": rows})
    assert len(blob) == cc.encoded_size(planes, mask)
    h, p2, m2 = cc.decode(blob, planes.shape[1])
    assert h["rows"] == rows and h["rng"] == HDR["rng"] and h["n_blocks"] == mask.shape[0]
    np.testing.assert_array_equal(p2, planes)
    np.testing.assert_array_equal(m2, mask)
    return blob


def test_header_layout_matches_the_c_header():
    assert C.sizeof(capi.bgr_checkpoint_header) == 104 == cc.HEADER.size
    offs = {"magic": 0, "version": 4, "layout": 8, "frame": 16, "rows": 20, "words": 24, "n_blocks": 28, "n_columns": 32,
            "fps": 36, "active": 40, "elapsed_ns": 48, "rng": 56, "digest_root": 88, "payload_bytes": 96}
    assert [f for f, _ in capi.bgr_checkpoint_header._fields_] == list(offs) == list(cc.HEADER_FIELDS)
    for f, o in offs.items():
        assert getattr(capi.bgr_checkpoint_header, f).offset == o, f
    h = capi.bgr_checkpoint_header(magic=cc.MAGIC, version=1, frame=-3, rows=5, rng=(C.c_uint64 * 4)(9, 8, 7, 6), payload_bytes=44)
    d = cc.unpack_header(bytes(h))
    assert d["frame"] == -3 and d["rows"] == 5 and d["rng"] == (9, 8, 7, 6) and d["payload_bytes"] == 44
    assert cc.pack_header(d) == bytes(h)


@pytest.mark.parametrize("rows", [0, 1, 511, 512, 513, 1400, 3 * 512])
@pytest.mark.parametrize("words", [1, 3, 15])
def test_random_worlds_roundtrip(rows, words):
    rng = np.random.default_rng(rows * 31 + words)
    absent = cc.plane_absent([4 * words], [False]) if words < 3 else cc.plane_absent([4, 4, 4 * (words - 2)], [False, True, True])
    planes, mask = _world(rng, rows, words, absent)
    _roundtrip(planes, mask, rows)


def test_canonical_form_zeroes_what_the_digest_does_not_cover():
    absent = cc.plane_absent([8, 4], [False, True])   # planes 0-1 always, plane 2 optional (bit 2)
    planes = np.full((1, 3, cc.BLOCK), 7, np.uint32)
    mask = np.ones((1, cc.BLOCK), np.uint8)
    mask[0, 5] = 0          # dead row
    mask[0, 6] = 1 | 2      # exists, optional column absent
    mask[0, 7] = 2          # dead with a stale absent bit
    p, m = cc.canonical(planes, mask, 300, absent)
    assert (p[0, :, 5] == 0).all() and (m[0, 5] == 0)
    assert (p[0, :2, 6] == 7).all() and p[0, 2, 6] == 0 and m[0, 6] == 3
    assert m[0, 7] == 0 and (p[0, :, 7] == 0).all()
    assert (p[0, :, 300:] == 0).all() and (m[0, 300:] == 0).all() and (p[0, :, :300][:, m[0, :300] == 1] == 7).all()


@pytest.mark.parametrize("n_vec", ["plane", "mask"])
def test_kind_thresholds(n_vec):
    n = cc.BLOCK if n_vec == "plane" else cc.MASK_WORDS
    lim = n - n // 32
    rng = np.random.default_rng(n)

    def vec(nnz):
        v = np.zeros(n, np.uint32)
        v[rng.choice(n, nnz, replace=False)] = rng.integers(1, 2**32, nnz)
        return v
    assert cc.kind_of(np.zeros(n, np.uint32)) == cc.CONST
    assert cc.kind_of(np.full(n, 5, np.uint32)) == cc.CONST
    assert cc.kind_of(vec(lim - 1)) == cc.SPARSE
    assert cc.kind_of(vec(lim)) == cc.RAW
    assert cc.kind_of(vec(1)) == cc.SPARSE
    for nnz, body in ((lim - 1, n // 32 + lim - 1), (lim, n)):
        v = vec(nnz)
        if n_vec == "plane":
            planes, mask = v.reshape(1, 1, n), np.zeros((1, cc.BLOCK), np.uint8)
        else:
            planes, mask = np.zeros((1, 1, cc.BLOCK), np.uint32), v.astype("<u4").view(np.uint8).reshape(1, cc.BLOCK)
        blk = cc.encode_block(planes[0], mask[0])
        assert len(blk) == 4 * (1 + body + 1)    # kind bytes, this vector, the other one CONST
        p2, m2 = cc.decode_block(blk, 1)
        np.testing.assert_array_equal(p2, planes[0])
        np.testing.assert_array_equal(m2, mask[0])


def test_all_equal_all_zero_and_partial_last_blocks():
    absent = cc.plane_absent([8], [False])
    planes = np.zeros((2, 2, cc.BLOCK), np.uint32)
    planes[:, 1] = 3
    mask = np.ones((2, cc.BLOCK), np.uint8)
    p, m = cc.canonical(planes, mask, 700, absent)
    blob = _roundtrip(p, m, 700)
    off = np.frombuffer(blob, "<u8", 3, cc.HEADER.size)
    assert int(off[1]) == 4 * (1 + 3)        # block 0: every vector CONST
    assert int(off[2] - off[1]) == 4 * (1 + 1 + (16 + 188) + (4 + 47))   # 188 rows remain: plane 1 and the mask SPARSE


def _blob():
    rng = np.random.default_rng(2)
    absent = cc.plane_absent([8, 4], [False, True])
    planes, mask = _world(rng, 1100, 3, absent, fill=0.3)
    return cc.encode(planes, mask, **{**HDR, "rows": 1100})


def _patch(blob, at, fmt, value):
    b = bytearray(blob)
    struct.pack_into(fmt, b, at, value)
    return bytes(b)


def _payload_at(blob, block):
    h = cc.unpack_header(blob)
    off = np.frombuffer(blob, "<u8", h["n_blocks"] + 1, cc.HEADER.size)
    return cc.HEADER.size + 8 * (h["n_blocks"] + 1) + int(off[block])


def malformed_cases(blob, words):
    """(name, blob) of every malformed case the codec and the engine refuse before decoding."""
    h = cc.unpack_header(blob)
    n = h["n_blocks"]
    off0 = cc.HEADER.size
    p1 = _payload_at(blob, 1)
    first_sparse = next(i for i, k in enumerate(blob[p1:p1 + words + 1]) if k == cc.SPARSE)
    return [
        ("bad magic", _patch(blob, 0, "<I", 0x12345678)),
        ("bad version", _patch(blob, 4, "<I", 2)),
        ("n_blocks", _patch(blob, 28, "<I", n + 1)),
        ("rows", _patch(blob, 20, "<I", h["rows"] + 512)),
        ("truncated header", blob[:50]),
        ("truncated offsets", blob[:off0 + 8]),
        ("truncated payload", blob[:-4]),
        ("overlong", blob + b"\0\0\0\0"),
        ("payload_bytes", _patch(blob, 96, "<Q", h["payload_bytes"] + 4)),
        ("first offset", _patch(blob, off0, "<Q", 4)),
        ("unaligned offset", _patch(blob, off0 + 8, "<Q", int(np.frombuffer(blob, "<u8", 1, off0 + 8)[0]) + 2)),
        ("descending offsets", _patch(blob, off0 + 8, "<Q", int(np.frombuffer(blob, "<u8", 1, off0 + 16)[0]) + 4)),
        ("kind byte 3", _patch(blob, p1, "<B", 3)),
        ("padding", _patch(blob, p1 + words + 1, "<B", 1)),
        ("implied length", _patch(blob, p1 + first_sparse, "<B", cc.RAW)),
        ("bitmap bit", _patch(blob, p1 + 4 * ((words + 1 + 3) // 4) + 0, "<B", blob[p1 + 4 * ((words + 1 + 3) // 4)] ^ 0x10)
         if blob[p1] == cc.SPARSE else _patch(blob, p1, "<B", cc.SPARSE)),
    ]


def test_codec_refuses_malformed_blobs():
    blob = _blob()
    cc.decode(blob, 3)
    with pytest.raises(cc.CodecError):
        cc.decode(blob, 4)                   # words that do not match
    for name, bad in malformed_cases(blob, 3):
        with pytest.raises(cc.CodecError):
            cc.decode(bad, 3)
            pytest.fail(name)


def test_rows_zero():
    p, m = np.zeros((0, 2, cc.BLOCK), np.uint32), np.zeros((0, cc.BLOCK), np.uint8)
    blob = _roundtrip(p, m, 0)
    assert len(blob) == 104 + 8


def test_particles_world_of_a_million_rows_is_counted():
    """The stress schema's 1M-row synthetic world: ten of the fifteen word planes (translation.z, rotation, scale,
    velocity.z, ttl.hi) and the mask plane are CONST in every tile, the other five RAW: 10 300 B per tile."""
    n = 1 << 20
    tf, vel, ttl = synth_particles(n, 3, 40, 400)
    rows = np.concatenate([tf.view("<u4"), vel.view("<u4"), ttl.view("<u4").reshape(n, 2)], axis=1)   # [n, 15]
    planes = np.ascontiguousarray(rows.reshape(n // cc.BLOCK, cc.BLOCK, 15).transpose(0, 2, 1))
    mask = np.ones((n // cc.BLOCK, cc.BLOCK), np.uint8)
    size = cc.encoded_size(planes, mask)
    assert size == 104 + 8 * 2049 + 2048 * 10300 == 21_110_896
    assert cc.encode_block(planes[5], mask[5]).__len__() == 10300
    raw = n * 61
    assert 2.9 < raw / size < 3.1
