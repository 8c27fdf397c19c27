"""Desync reports on random registrations, against the oracle's restatements (tests/oracle_p2p.py, oracle_desync.py).

The other desync tests run two fixed registrations.  Here the schemas come from schema_util.random_schema: element
sizes with sub-word tails (1, 2, 3, 5, 7 B) and up to 1024 B, up to seven optional columns (every bit of the mask byte),
checksum ranges that are none, whole-element or unaligned and partial, rows of 24 / 25 and 49 / 50 words, populations
on either side of a 512-row block, and an order_base above 2^32.  Every tick-path case runs on the generic one-launch
program (interpreter, NVRTC whole tile, NVRTC quarter tile) and on the stepwise path (TMA, flat, two TMA stages).

- digest parity: bgr_frame_digest of every queued and retained frame equals the oracle's restatement, bit for bit,
  under host edits (remove, insert, spawn, despawn) and rollbacks across spawns, including frames of 0 rows;
- fold: the words of whole-element checksummed columns fold (bgr_fold_partials) to the frame's checksum;
- remote diff: two peers with seeded divergences and different row counts exchange digests and blocks as
  INTEGRATION.md documents, in both directions; digest_mismatch and diff_remote equal the oracle's;
- capture diff: bgr_desync_diff of a SyncTest re-simulation that diverges equals CaptureOracleWorld's report;
- limits and refusals of the digest and the blob.
"""
import ctypes as C

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine, digest_mismatch
from bevy_ggrs_b200.session import SAVE, SESSION_NONE, P2PTraceSession, Request, SyncTestSession
from oracle_desync import CaptureOracleWorld
from oracle_p2p import RetainOracleWorld, two_world_diff
from schema_util import WIDE_PATHS, expected_kind, path_env, random_schema

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
BLOCK = capi.BGR_DIGEST_BLOCK_ROWS
CAP = capi.BGR_CFG_DESYNC_CAPTURE
LIB = capi.load_library()
BIG_BASE = (1 << 32) + 12345   # RollbackOrdered indices above 2^32: the digest hashes order_base + row as a u64

# name: random_schema arguments, population (None: random), order_base, tick of the first spawn, P(no rollback).
# An engine with order_base != 0 is one shard of a larger world and refuses spawns after its initial population, so
# those cases get no host spawns.  empty_frames: frames 0..2 hold 0 rows; its trace has no rollback, which would undo
# the population spawned at tick 3.
CASES = {
    "tails_all_optional": (dict(sizes=[1, 2, 3, 5, 7, 8, 12, 40], n_opt=7), 513, 0, 0, 0.3),
    "w24_big_base": (dict(words=24), 1025, BIG_BASE, 0, 0.3),
    "w25": (dict(words=25), 512, 0, 0, 0.3),
    "w49": (dict(words=49, n_opt=7), 511, 0, 0, 0.3),
    "w50": (dict(words=50), None, BIG_BASE, 0, 0.3),
    "elem1024": (dict(sizes=[1024, 3, 8], n_opt=1), 1, 0, 0, 0.3),
    "empty_frames": (dict(words=12, n_opt=3), 600, 0, 3, 1.0),
}


def _seed(name):
    return 7000 + list(CASES).index(name)


def _populate(worlds, spec, rng, n):
    if n == 0:
        return
    data = spec.values(rng, n)
    removes = [(i, int(r)) for i, o in enumerate(spec.optional) if o for r in rng.choice(n, min(n, 5), replace=False)]
    for w in worlds:
        first = w.spawn(n)
        for i, d in enumerate(data):
            w.write_component(i, first, d)
        for i, r in removes:
            w.remove_component(i, first + r)


def _edit(worlds, spec, rng, max_entities, spawn=True):
    """Host edits between ticks, the same on every world: remove / insert optional components, despawn, spawn."""
    orc = worlds[-1]
    rows = orc.row_count()
    alive = np.flatnonzero(orc.read_alive(0, rows)) if rows else np.zeros(0, np.int64)
    opt = [i for i, o in enumerate(spec.optional) if o]
    if opt and alive.size:
        for r in rng.choice(alive, size=min(2, alive.size), replace=False):
            i, r = int(rng.choice(opt)), int(r)
            if orc.has_component(i, r, 1)[0]:
                for w in worlds:
                    w.remove_component(i, r)
            else:
                v = rng.integers(0, 256, spec.sizes[i], dtype=np.uint8)
                for w in worlds:
                    w.insert_component(i, r, v)
    if alive.size > 1 and rng.random() < 0.3:
        r = int(rng.choice(alive))
        for w in worlds:
            w.despawn(r)
    if spawn and rng.random() < 0.3 and rows + 8 < max_entities:
        _populate(worlds, spec, rng, int(rng.integers(1, 6)))


def _p2p_twins(name, flags, generic_kernel, path, ticks=24, retain=(2, 6)):
    """Engine and RetainOracleWorld of one CASES entry on the same P2P trace with host edits between ticks.  Yields
    after every tick (for checks mid-run); the checksum of every frame the engine returned, latest first wins."""
    args, n, order_base, spawn_tick, p_clean = CASES[name]
    rng = np.random.default_rng(_seed(name))
    spec = random_schema(rng, **args)
    n = int(rng.integers(2, 1400)) if n is None else n
    cap = n + 64
    eng = Engine(max_entities=cap, max_depth=8, flags=flags, order_base=order_base)
    orc = RetainOracleWorld(max_entities=cap, max_depth=8, order_base=order_base)
    for w in (eng, orc):
        spec.register(w)
        w.retain_confirmed(*retain)
        w.build()
    if spawn_tick == 0:
        _populate((eng, orc), spec, rng, n)
    kind = expected_kind(path, spec.words, len(spec.systems), spec.nvrtc_ranges, generic_kernel)
    sess, latest = P2PTraceSession(2, 6, seed=_seed(name), p_clean=p_clean), {}
    for t in range(ticks):
        if t == spawn_tick and t:
            _populate((eng, orc), spec, rng, n)
        elif t:
            _edit((eng, orc), spec, rng, cap, spawn=order_base == 0)
        for h in range(2):
            sess.add_local_input(h, 0)
        reqs = sess.advance_frame()
        out = eng.handle_requests(sess.info(), reqs)
        assert orc.handle_requests(sess.info(), reqs) == out, f"checksums differ at tick {t}"
        assert eng.last_kernel().kind == kind, t
        for f, c in out:
            sess.save_cell(f, c)
            latest[f] = c
        yield eng, orc, spec, latest, t


def _digests_equal(eng, orc, n_cols):
    assert eng.snapshot_frames() == orc.snapshot_frames()
    assert eng.retained_frames() == orc.retained_frames()
    rows_seen = []
    for f in eng.snapshot_frames() + eng.retained_frames():
        h, words = eng.frame_digest(f)
        rows, active, expect = orc.frame_digest(f)
        assert (h.frame, h.rows, h.active, h.n_blocks, h.n_columns) == (f, rows, active, -(-rows // BLOCK), n_cols), f
        assert np.array_equal(words, expect), f
        assert h.root == LIB.bgr_seahash(words.tobytes(), words.nbytes)
        rows_seen.append(rows)
    return rows_seen


@pytest.mark.parametrize("path", list(WIDE_PATHS))
@pytest.mark.parametrize("name", list(CASES))
def test_digest_equals_the_oracle_on_random_schemas(monkeypatch, generic_kernel, name, path):
    flags = path_env(monkeypatch, path, generic_kernel)
    rows_seen = []
    for eng, orc, spec, _, t in _p2p_twins(name, flags, generic_kernel, path):
        if t in (CASES[name][3], 12, 23):   # while frames of 0 rows are queued (empty_frames), mid-run, at the end
            rows_seen += _digests_equal(eng, orc, len(spec.sizes))
    assert eng.retained_frames()
    if name == "empty_frames":
        assert 0 in rows_seen and max(rows_seen) > 0
    # after rollbacks across spawns a slot holds a frame with fewer rows than the frame it held before: its stale rows
    # past the row count are not data (the digests above equal the oracle's, which has no such rows)
    if CASES[name][2] == 0:
        assert len(set(rows_seen)) > 1


FOLD_CASES = {"optional_big_base": (dict(sizes=[1, 3, 5, 7, 8, 12, 40, 2], n_opt=7, ranges=("whole",)), 1300,
                                    BIG_BASE),
              "w24_whole": (dict(words=24, ranges=("whole",)), 700, 3)}


@pytest.mark.parametrize("path", list(WIDE_PATHS))
@pytest.mark.parametrize("case", list(FOLD_CASES))
def test_digest_words_fold_to_the_frames_checksum(monkeypatch, generic_kernel, case, path):
    """Columns checksummed over the whole element: the XOR of a column's words over all blocks is its checksum partial,
    so the words fold through bgr_fold_partials to the checksum the tick returned for that frame."""
    flags = path_env(monkeypatch, path, generic_kernel)
    args, n, order_base = FOLD_CASES[case]
    rng = np.random.default_rng(31 + len(case))
    spec = random_schema(rng, **args)
    assert spec.cks and all(off == 0 and ln == spec.sizes[i] for i, off, ln in spec.cks)
    eng = Engine(max_entities=n + 64, max_depth=8, flags=flags, order_base=order_base)
    spec.register(eng)
    eng.retain_confirmed(3, 4)
    eng.build()
    _populate((eng,), spec, rng, n)
    sess, latest = P2PTraceSession(2, 8, seed=5, p_clean=0.3), {}
    for t in range(20):
        if t:
            _edit((eng,), spec, rng, n + 64, spawn=order_base == 0)
        for h in range(2):
            sess.add_local_input(h, 0)
        for f, c in eng.handle_requests(sess.info(), sess.advance_frame()):
            sess.save_cell(f, c)
            latest[f] = c
    assert eng.last_kernel().kind == expected_kind(path, spec.words, len(spec.systems), spec.nvrtc_ranges, generic_kernel)
    frames = eng.snapshot_frames() + eng.retained_frames()
    assert len(frames) > 4
    for f in frames:
        h, words = eng.frame_digest(f)
        x = np.bitwise_xor.reduce(words, axis=0) if len(words) else np.zeros(words.shape[1], np.uint64)
        p = capi.bgr_partial()
        p.frame, p.n_columns, p.active, p.total = f, len(spec.cks), h.active, h.rows
        for k, (i, _, _) in enumerate(spec.cks):   # checksum slots follow column order
            p.xor_[k] = int(x[i])
        cs = capi.bgr_checksum()
        assert LIB.bgr_fold_partials(C.byref(p), C.byref(cs)) == 0
        assert cs.lo == latest[f], f


# ---- two peers: the documented exchange (digest -> mismatched blocks the peer has -> export -> diff_remote) ----
def _remote_schema(rng):
    """Column 0 (16 B) is checksummed over [3, 8): word 2 is the first word past a range that ends on a word boundary
    inside the element.  Column 1 is 7 B: its last word holds 3 bytes.  Columns 2..4 are optional."""
    spec = random_schema(rng, sizes=[16, 7, 3, 12, 5, 8])
    spec.optional = [False, False, True, True, True, False]
    spec.cks = sorted([(0, 3, 5)] + [c for c in spec.cks if c[0] != 0][:5])
    spec.systems = [(capi.BGR_SYS_U32_ADD, [3], [4, 1])]
    return spec


def _diverge(w, spec, data, m):
    """Peer B's seeded divergences, all in rows both peers have (m = the smaller population)."""
    def flip(col, row, byte):
        v = data[col][row].copy()
        v[byte] ^= 0x5A
        w.write_component(col, row, v)
    flip(0, 5, 5)                 # a word inside the checksummed range
    flip(0, 40, 9)                # the word right past it
    flip(1, 300, 6)               # the last word of a 7-byte element
    w.remove_component(2, m - 2)  # presence: removed on B only ...
    w.insert_component(3, 7, data[3][7])   # ... and inserted on B only (row 7 of column 3 is removed on both first)
    w.despawn(100)
    w.despawn(m - 3)


def _remote_peers(n_a, n_b, flags):
    rng = np.random.default_rng(n_a * 7 + n_b)
    spec = _remote_schema(rng)
    data = spec.values(rng, max(n_a, n_b))
    peers = []
    for rows, seed in ((n_a, 100), (n_b, 200)):
        eng = Engine(max_entities=max(n_a, n_b) + 64, max_depth=8, flags=flags)
        orc = RetainOracleWorld(max_entities=max(n_a, n_b) + 64, max_depth=8)
        for w in (eng, orc):
            spec.register(w)
            w.retain_confirmed(5, 4)
            w.build()
            w.spawn(rows)
            for i, d in enumerate(data):
                w.write_component(i, 0, d[:rows])
            w.remove_component(3, 7)
            if seed == 200:
                _diverge(w, spec, data, min(n_a, n_b))
        peers.append((eng, orc, P2PTraceSession(2, 8, seed=seed, p_clean=0.3)))
    for _ in range(30):
        for eng, orc, sess in peers:
            for h in range(2):
                sess.add_local_input(h, 0)
            reqs = sess.advance_frame()
            out = eng.handle_requests(sess.info(), reqs)
            assert orc.handle_requests(sess.info(), reqs) == out
            for f, c in out:
                sess.save_cell(f, c)
    for eng, orc, _ in peers:
        assert eng.retained_frames() == orc.retained_frames()
    (a, oa, _), (b, ob, _) = peers
    f = sorted(set(a.retained_frames()) & set(b.retained_frames()))[0]
    return (a, oa), (b, ob), f


def _same_report(rep, expect, what):
    assert rep.summary_tuple() == expect.summary_tuple(), what
    assert rep.columns == expect.columns, what
    assert rep.records.dtype == expect.records.dtype and np.array_equal(rep.records, expect.records), what


def _exchange(local, remote, f):
    """The INTEGRATION.md exchange with `local` diffing `remote`'s blocks; every step against the oracle twins."""
    (le, lo), (re_, ro) = local, remote
    dl, dr = le.frame_digest(f), re_.frame_digest(f)
    wl, wr = lo.frame_digest(f)[2], ro.frame_digest(f)[2]
    assert np.array_equal(dl[1], wl) and np.array_equal(dr[1], wr)
    common = min(len(wl), len(wr))
    blocks, host = digest_mismatch(dl, dr)
    assert blocks == [b for b in range(max(len(wl), len(wr))) if b >= common or (wl[b] != wr[b]).any()]
    assert host == 0
    want = [b for b in blocks if b < dr[0].n_blocks]
    blob = re_.export_blocks(f, want)
    full = two_world_diff(lo, ro, f, want, 1 << 30)
    # the blocks whose digests agree hold no difference: the exchange finds every differing row
    everything = two_world_diff(lo, ro, f, range(dr[0].n_blocks), 1 << 30)
    assert full.summary_tuple() == everything.summary_tuple() and np.array_equal(full.records, everything.records)
    total = len(full.records)
    for cap in sorted({0, 1, 31, 32, 33, 511, 512, 513, total, total + 1}):
        _same_report(le.diff_remote(f, blob, cap), two_world_diff(lo, ro, f, want, cap), cap)
    return full


@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
@pytest.mark.parametrize("n_a,n_b", [(1400, 1450), (512, 513), (1025, 2100)])
def test_remote_diff_equals_the_oracle_in_both_directions(n_a, n_b, flags):
    a, b, f = _remote_peers(n_a, n_b, flags)
    ab, ba = _exchange(a, b, f), _exchange(b, a, f)
    for rep in (ab, ba):
        assert rep.rows_differing > 0 and rep.columns[0].rows == 2 and rep.columns[0].rows_in_checksum == 1
        assert rep.columns[1].rows == 1 and rep.columns[2].presence == 1 and rep.columns[3].presence == 1
    # B holds n_b - n_a rows A does not have (minus none: B's despawns are all below n_a): every one is an existence
    # record of B's report, whichever side exports
    extra = n_b - n_a
    assert ba.existence_differing == ab.existence_differing == extra + 2
    # the peer that has fewer blocks exports subsets of its blocks; the local-only blocks are diffed with every one
    for (le, lo), (re_, ro) in ((b, a), (a, b)):
        nb = re_.frame_digest(f)[0].n_blocks
        for subset in ([0, nb - 1] if nb > 2 else [0], [nb - 1], []):
            blob = re_.export_blocks(f, subset)
            expect = two_world_diff(lo, ro, f, subset, 1 << 30)
            for cap in (0, 1, 33, len(expect.records), len(expect.records) + 1):
                _same_report(le.diff_remote(f, blob, cap), two_world_diff(lo, ro, f, subset, cap), (subset, cap))


# ---- SyncTest capture diff on random schemas ----
CAPTURE_CASES = {"tails_all_optional": (dict(sizes=[8, 1, 2, 3, 5, 7, 12, 40], n_opt=7), 513),
                 "w25": (dict(words=25), 1025),
                 "w50": (dict(words=50), 600)}


@pytest.mark.parametrize("path", list(WIDE_PATHS))
@pytest.mark.parametrize("case", list(CAPTURE_CASES))
def test_capture_diff_equals_the_oracle_on_random_schemas(monkeypatch, generic_kernel, case, path):
    """A U32_STORE_CALL_COUNT system makes every re-simulated frame differ from its first image; host edits between
    ticks add presence and existence differences the re-simulation's Load undoes."""
    flags = path_env(monkeypatch, path, generic_kernel)
    args, n = CAPTURE_CASES[case]
    rng = np.random.default_rng(400 + list(CAPTURE_CASES).index(case))
    spec = random_schema(rng, store_call_count=True, **args)
    eng = Engine(max_entities=n + 64, max_depth=8, flags=flags | CAP)
    orc = CaptureOracleWorld(max_entities=n + 64, max_depth=8)
    for w in (eng, orc):
        spec.register(w)
        w.build()
    _populate((eng, orc), spec, rng, n)
    kind = expected_kind(path, spec.words, len(spec.systems), spec.nvrtc_ranges, generic_kernel)
    sess = SyncTestSession(1, 3, 8)
    for t in range(12):
        if t:
            _edit((eng, orc), spec, rng, n + 64)
        sess.add_local_input(0, 0)
        reqs = sess.advance_frame()
        out = eng.handle_requests(sess.info(), reqs)
        assert orc.handle_requests(sess.info(), reqs) == out
        assert eng.last_kernel().kind == kind
        for f, _ in out:   # the edits are undone by the re-simulations: keep the request shape, skip the check
            sess.save_cell(f, 0)
    frames = eng.desync_frames()
    assert frames and frames == orc.desync_frames()
    for f in frames[:2]:
        total = len(orc.desync_diff(f, 1 << 30).records)
        assert total > 0
        for cap in sorted({0, 1, 31, 32, 33, 511, 512, 513, total, total + 1}):
            _same_report(eng.desync_diff(f, cap), orc.desync_diff(f, cap), (f, cap))


# ---- limits and refusals ----
def _saved(eng_or_orc, n_rows, values=None):
    w = eng_or_orc
    w.build()
    w.set_depth(2)
    w.spawn(n_rows)
    for i, v in enumerate(values or []):
        w.write_component(i, 0, v)
    return w.handle_requests((SESSION_NONE, 0, 0, 0), [Request(SAVE, 0)])


def test_digest_of_382_one_byte_columns_and_refusal_at_383():
    """The kernel's shared memory holds 16 warps x (columns + 1) words: 382 columns fit in 48 KB, 383 do not."""
    rng = np.random.default_rng(382)
    values = [rng.integers(0, 256, (600, 1), dtype=np.uint8) for _ in range(383)]
    eng, orc = Engine(max_entities=608, max_depth=4), RetainOracleWorld(max_entities=608, max_depth=4)
    for w in (eng, orc):
        for c in range(382):
            w.rollback_component(f"B{c}", 1)
        w.checksum_component(381, 0, 1)
    assert _saved(eng, 600, values[:382]) == _saved(orc, 600, values[:382])
    h, words = eng.frame_digest(0)
    rows, active, expect = orc.frame_digest(0)
    assert (h.rows, h.active, h.n_blocks, h.n_columns) == (rows, active, 2, 382) and words.shape == (2, 383)
    assert np.array_equal(words, expect)
    big = Engine(max_entities=608, max_depth=4)
    for c in range(383):
        big.rollback_component(f"B{c}", 1)
    _saved(big, 600, values)
    with pytest.raises(BgrError) as ei:
        big.frame_digest(0)
    assert ei.value.status == capi.BGR_ERR_UNSUPPORTED and "382" in str(ei.value)


def _small_world(max_entities, rows, order_base=0):
    w = Engine(max_entities=max_entities, max_depth=4, order_base=order_base)
    w.rollback_component("A", 5)
    w.rollback_component("B", 4, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)
    w.checksum_component(0, 1, 3)
    _saved(w, rows, [np.full((rows, 5), 3, np.uint8), np.full((rows, 4), 9, np.uint8)])
    return w


def test_peers_whose_order_base_differs_above_bit_32_are_refused():
    a, b = _small_world(700, 600, 77), _small_world(700, 600, 77 + (1 << 32))
    with pytest.raises(BgrError) as ei:
        digest_mismatch(a.frame_digest(0), b.frame_digest(0))
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and "layout" in str(ei.value)
    with pytest.raises(BgrError) as ei:
        a.diff_remote(0, b.export_blocks(0, [0]))
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and "layout" in str(ei.value)


def test_a_blob_of_more_blocks_than_the_local_capacity_is_refused():
    small, big = _small_world(600, 600), _small_world(2000, 1100)   # 2 blocks of capacity; a 3-block frame
    assert small.diff_remote(0, small.export_blocks(0, [1])).rows_differing == 0
    with pytest.raises(BgrError) as ei:
        small.diff_remote(0, big.export_blocks(0, [0]))
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    assert "the blob's row and block counts are inconsistent or exceed this engine's capacity" in str(ei.value)
