"""CPU: the checkpoint delta format restated in numpy (checkpoint_delta_codec.py) round-trips random pairs of worlds
with differing row counts, optional columns and sub-word elements, codes unchanged blocks as CONST zero, refuses
malformed deltas and non-canonical targets, and the delta header has one layout in the C header, capi.py, the
restatement and the Rust #[repr(C)] mirror."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
import checkpoint_codec as cc
import checkpoint_delta_codec as dc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_delta_header_layout_matches_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    fields = list(dc.HEADER_FIELDS)
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "bevy_ggrs_b200.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(bgr_checkpoint_delta_header));']
    lines += [f'printf("{f} %zu\\n", offsetof(bgr_checkpoint_delta_header, {f}));' for f in fields]
    lines += ['printf("magic_value %u\\n", BGR_CHECKPOINT_DELTA_MAGIC);', "return 0;", "}"]
    src.write_text("\n".join(lines))
    exe = str(tmp_path / "layout")
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = dict(l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    cls = capi.bgr_checkpoint_delta_header
    assert int(got["size"]) == C.sizeof(cls) == dc.HEADER.size == 120
    assert int(got["magic_value"]) == capi.BGR_CHECKPOINT_DELTA_MAGIC == dc.MAGIC
    assert [f for f, _ in cls._fields_] == fields
    for f in fields:
        assert int(got[f]) == getattr(cls, f).offset, f
    h = cls(magic=dc.MAGIC, version=1, frame=-3, rows=5, base_frame=-9, base_rows=700, rng=(C.c_uint64 * 4)(9, 8, 7, 6),
            base_root=0xABCDEF, payload_bytes=44)
    d = dc.unpack_header(bytes(h))
    assert (d["frame"], d["base_frame"], d["base_rows"], d["rng"], d["base_root"]) == (-3, -9, 700, (9, 8, 7, 6), 0xABCDEF)
    assert dc.pack_header(d) == bytes(h)


def test_rust_delta_header_has_the_c_layout():
    rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200_sys", "src", "checkpoint.rs")).read()
    body = re.search(r"#\[repr\(C\)\]\s*#\[derive\([^)]*\)\]\s*pub struct bgr_checkpoint_delta_header \{(.*?)\}", rs, re.S).group(1)
    size = {"u32": 4, "i32": 4, "u64": 8, "[u64; 4]": 32}
    align = {"u32": 4, "i32": 4, "u64": 8, "[u64; 4]": 8}
    off, layout = 0, []
    for name, ty in re.findall(r"pub (\w+): ([^,\n]+),", body):
        off = (off + align[ty] - 1) // align[ty] * align[ty]
        layout.append((name, off))
        off += size[ty]
    cls = capi.bgr_checkpoint_delta_header
    assert layout == [(f, getattr(cls, f).offset) for f, _ in cls._fields_]
    assert off == C.sizeof(cls)
    assert re.search(r"pub const BGR_CHECKPOINT_DELTA_MAGIC: u32 = 0x44524742;", rs)
    assert "pub fn save_delta(" in rs and "pub fn restore_delta(" in rs


# ---- the codec ----
# a registration: element bytes and optional flags per column (a 5-byte and a 2-byte column are sub-word)
SCHEMAS = {
    "stress": ([40, 12, 8], [False, False, False]),
    "optional_subword": ([5, 4, 2, 12], [False, True, True, False]),
}


def _schema(name):
    eb, opt = SCHEMAS[name]
    absent = cc.plane_absent(eb, opt)
    pad = []
    for e in eb:
        pad += [0] * ((e + 3) // 4 - 1) + [(0xFFFFFFFF << (8 * (e % 4))) & 0xFFFFFFFF if e % 4 else 0]
    mask_bits = 1 | sum(2 << k for k in range(sum(opt)))
    return absent, np.array(pad, np.uint32), mask_bits


def _world(rng, rows, absent, pad, mask_bits, like=None, p_change=1.0):
    """A canonical world of ``rows`` rows; with ``like``, one whose rows differ from it with probability p_change."""
    n = -(-rows // cc.BLOCK)
    planes = rng.integers(0, 2**32, (n, len(absent), cc.BLOCK), dtype=np.uint32) & ~pad[None, :, None]
    mask = (rng.integers(0, 256, (n, cc.BLOCK)) & mask_bits).astype(np.uint8)
    mask[rng.random((n, cc.BLOCK)) < 0.1] &= 0xFE   # despawned rows
    if like is not None:
        lp, lm = dc.widen(*like, max(n, like[1].shape[0]))
        keep = rng.random((n, cc.BLOCK)) >= p_change
        planes = np.where(keep[:, None, :], lp[:n], planes)
        mask = np.where(keep, lm[:n], mask)
    return cc.canonical(planes, mask, rows, absent)


def _roundtrip(target, base, rows, base_rows, absent, pad, mask_bits):
    bh = dict(frame=10, rows=base_rows, words=len(absent), digest_root=77)
    fields = dict(layout=5, frame=12, rows=rows, base_frame=10, base_rows=base_rows, n_columns=3, fps=60, active=1,
                  elapsed_ns=9, rng=(1, 2, 3, 4), digest_root=88, base_root=77)
    blob = dc.encode(target, base, **fields)
    assert len(blob) == dc.encoded_size(target, base, rows, base_rows)
    h, planes, mask = dc.decode(blob, bh, *base, absent, pad, mask_bits)
    assert np.array_equal(planes, target[0]) and np.array_equal(mask, target[1])
    assert h["n_blocks"] == -(-max(rows, base_rows) // cc.BLOCK)
    return blob, bh, fields


@pytest.mark.parametrize("schema", list(SCHEMAS))
@pytest.mark.parametrize("rows,base_rows", [(1400, 1400), (900, 1400), (1400, 600), (0, 700), (700, 0), (513, 512)])
def test_random_pairs_roundtrip(schema, rows, base_rows):
    absent, pad, mask_bits = _schema(schema)
    rng = np.random.default_rng(rows * 7 + base_rows)
    base = _world(rng, base_rows, absent, pad, mask_bits)
    for p in (0.0, 0.01, 0.3, 1.0):
        target = _world(rng, rows, absent, pad, mask_bits, like=base, p_change=p)
        _roundtrip(target, base, rows, base_rows, absent, pad, mask_bits)


def test_an_unchanged_block_codes_as_const_zero():
    absent, pad, mask_bits = _schema("stress")
    rng = np.random.default_rng(1)
    base = _world(rng, 2048, absent, pad, mask_bits)
    blob = dc.encode(base, base, layout=0, frame=1, rows=2048, base_frame=1, base_rows=2048, n_columns=3, fps=60, active=0,
                     elapsed_ns=0, rng=(0, 0, 0, 0), digest_root=0, base_root=0)
    # 16 vectors: 16 kind bytes and one zero u32 each, 80 bytes per block
    assert len(blob) == 120 + 8 * 5 + 4 * 80
    assert not any(blob[120 + 8 * 5:])
    # k changed rows of one plane: that vector SPARSE, 16 bitmap words plus k values
    target = (base[0].copy(), base[1].copy())
    live = np.nonzero(base[1][0] & 1)[0][:5]
    target[0][0, 3, live] ^= 0x10
    blob2 = dc.encode(target, base, **{**dc.unpack_header(blob), "payload_bytes": 0})
    assert len(blob2) == len(blob) + 4 * (16 + 5) - 4


def test_refusals():
    absent, pad, mask_bits = _schema("optional_subword")
    rng = np.random.default_rng(3)
    base = _world(rng, 1000, absent, pad, mask_bits)
    target = _world(rng, 800, absent, pad, mask_bits, like=base, p_change=0.05)
    blob, bh, fields = _roundtrip(target, base, 800, 1000, absent, pad, mask_bits)

    def refused(bad):
        with pytest.raises(cc.CodecError):
            dc.decode(bad, bh, *base, absent, pad, mask_bits)
    h = dc.unpack_header(blob)
    for field, val in (("magic", cc.MAGIC), ("version", 2), ("base_frame", 11), ("base_rows", 999), ("base_root", 78),
                       ("n_blocks", 1), ("rows", 1100)):
        refused(dc.pack_header({**h, field: val}) + blob[120:])
    refused(blob[:-4])
    refused(blob + bytes(4))
    refused(blob[:50])

    def with_target(planes, mask):
        return dc.encode((planes, mask), base, **fields)
    tp, tm = dc.widen(*target, 2)
    dead = int(np.nonzero((tm[0] & 1) == 0)[0][0])
    p2 = tp.copy(); p2[0, 0, dead] = 1
    refused(with_target(p2, tm))                                        # a word of a row that does not exist
    m2 = tm.copy(); m2[1, 900 - 512] = 1
    refused(with_target(tp, m2))                                        # a row past the target's rows
    live = int(np.nonzero(tm[0] == 1)[0][0])
    m3 = tm.copy(); m3[0, live] |= 0x80
    refused(with_target(tp, m3))                                        # a presence bit the registration lacks
    p4 = tp.copy(); p4[0, 1, live] |= np.uint32(1 << 8)
    refused(with_target(p4, tm))                                        # a bit past the 5-byte column's element
    lacks = int(np.nonzero((tm[0] & 3) == 3)[0][0])                     # alive, optional column absent
    col_plane = int(np.nonzero(absent == 2)[0][0])
    p5 = tp.copy(); p5[0, col_plane, lacks] = 7
    refused(with_target(p5, tm))                                        # a word of a column the row lacks
