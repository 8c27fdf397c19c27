"""P2P desync reports on the H100: retaining confirmed frames changes nothing observable, the frame digest equals the
oracle's restatement (tests/oracle_p2p.py) bit for bit and folds to the frame's checksum, and two peers find, export and
diff exactly the blocks where their worlds differ, as the oracle's two-world diff says.  Generic one-launch program (generic_kernel fixture), the stepwise path, and the
particles bundle."""
import ctypes as C
import struct

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.desync import NO_INDEX, RECORD_DTYPE
from bevy_ggrs_b200.engine import Engine, digest_mismatch
from bevy_ggrs_b200.session import ADVANCE, SAVE, SESSION_P2P, P2PTraceSession, Request
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_p2p import RetainOracleWorld, two_world_diff

pytestmark = pytest.mark.gpu
PATHS = [0, capi.BGR_CFG_FORCE_STEPWISE]
BLOCK = capi.BGR_DIGEST_BLOCK_ROWS
OPT = capi.BGR_STRATEGY_OPTIONAL
LIB = capi.load_library()


def _presence_engine(n, flags=0, retain=(10, 4), tweak=None, max_depth=8, oracle=False):
    """Score (optional, +1 per frame), Health (optional, -1 per frame, despawns at 0), Tag (12 B, no system); on the
    engine, or on the oracle (oracle=True)."""
    eng = (RetainOracleWorld if oracle else Engine)(max_entities=n + 8, max_depth=max_depth, flags=flags)
    score = eng.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = eng.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = eng.rollback_component("Tag", 12)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        eng.checksum_component(c, 0, ln)
    eng.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    eng.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    if retain:
        eng.retain_confirmed(*retain)
    eng.build()
    eng.spawn(n)
    rng = np.random.default_rng(5)
    eng.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    eng.write_component(health, 0, rng.integers(30, 400, n, dtype=np.uint32))
    eng.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in range(3, n, 97):
        eng.remove_component(score, r)
    if tweak:
        tweak(eng)
    return eng


def _drive(eng, sess, ticks, edit=None):
    """Runs a P2P trace; returns every returned checksum (frame -> latest) and the per-tick outputs."""
    latest, outs = {}, []
    for t in range(ticks):
        if edit:
            edit(eng, t)
        for h in range(sess.num_players()):
            sess.add_local_input(h, 0)
        reqs = sess.advance_frame()
        out = eng.handle_requests(sess.info(), reqs)
        for f, c in out:
            sess.save_cell(f, c)
            latest[f] = c
        outs.append(out)
    return latest, outs


def _observe(eng, n_cols, rows):
    peeks = {}
    for f in eng.snapshot_frames():
        for c in range(n_cols):
            data, alive = eng.peek(f, c, 0, rows)
            peeks[(f, c)] = (data[alive.astype(bool)].tobytes(), alive.tobytes())
    return eng.snapshot_frames(), peeks, eng.launch_count()


# ---- nothing changes ----
@pytest.mark.usefixtures("generic_kernel")
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("depth", [1, 3, 8])
def test_retention_changes_nothing_on_p2p_traces(path, depth):
    def run(retain):
        eng = _presence_engine(1400, path, retain, max_depth=8)
        sess = P2PTraceSession(2, depth, seed=11 + depth, p_clean=0.3)
        _, outs = _drive(eng, sess, 60)
        return outs, _observe(eng, 3, 1400), eng
    a, b = run(None), run((2, 5))
    assert a[0] == b[0] and a[1][:2] == b[1][:2]
    # At depth 1 a plain ring hands the evicted base slot of a deferred live image straight to the next Save, which
    # then writes the live image first; a retained base slot is not reused, so retention saves some of those launches.
    # The stepwise path defers nothing: equal counts there.
    if depth == 1 and not path:
        assert b[1][2] < a[1][2]
    else:
        assert a[1][2] == b[1][2]
    assert b[2].retained_frames() and not a[2].retained_frames()


def _particles_engine(n, retain, seed=3, spawn_seed=None, flags=0):
    eng = Engine(max_entities=n + 64, max_depth=8, flags=flags)
    cols = register_particles(eng, spawn_rate=4 if spawn_seed is not None else 0, rng_seed=spawn_seed or 0)
    if retain:
        eng.retain_confirmed(*retain)
    eng.build()
    populate(eng, cols, *synth_particles(n, seed, 40, 400))
    return eng


@pytest.mark.parametrize("retain", [(1, 3), (10, 4)])
def test_retention_changes_nothing_on_the_bundle(retain):
    def run(r):
        eng = _particles_engine(3000, r)
        _, outs = _drive(eng, P2PTraceSession(2, 8, seed=5, p_clean=0.3), 50)
        assert eng.last_kernel().kind == "bundle"
        return outs, _observe(eng, 3, 3000), eng
    a, b = run(None), run(retain)
    assert a[:2] == b[:2]
    assert b[2].retained_frames()


def test_deferred_live_reads_a_base_slot_its_own_save_retained():
    """Depth 1: every Save evicts the previous frame from the old end, so with interval 1 the deferred live image's base
    slot becomes a retained frame at the next Save.  A retained slot is never written again: identical results."""
    def run(retain):
        eng = _particles_engine(2000, retain)
        sess = P2PTraceSession(2, 1, seed=9, p_clean=1.0)
        _, outs = _drive(eng, sess, 30)
        assert eng.last_kernel().deferred_live
        return outs, eng.read_component(0, 0, 2000).tobytes(), eng.launch_count()
    a, b = run(None), run((1, 6))
    assert a[:2] == b[:2] and b[2] < a[2]  # the retained base slot is not overwritten: fewer live-image writes


# ---- the digest, restated from bgr_peek ----
def _seahash_2xu64(a, b):
    return LIB.bgr_seahash(struct.pack("<QQ", a, b), 16)


def _image(eng, frame, elem_bytes, absent_bits):
    """Rows of a queued or retained frame from its export blob (tile bytes as stored): (rows, mask bytes of existing
    rows else 0, per column the element bytes of rows that hold it else None)."""
    h, _ = eng.frame_digest(frame)
    blob = eng.export_blocks(frame, range(h.n_blocks))
    hdr = capi.bgr_frame_blob_header.from_buffer_copy(blob)
    words = hdr.words
    tile_bytes = BLOCK * (4 * words + 1)
    first = np.cumsum([0] + [(e + 3) // 4 for e in elem_bytes])
    mask = np.zeros(hdr.rows, np.uint32)
    elems = [[None] * hdr.rows for _ in elem_bytes]
    for i in range(hdr.n_exported):
        off = C.sizeof(hdr) + i * (8 + tile_bytes)
        b = struct.unpack_from("<I", blob, off)[0]
        tile = np.frombuffer(blob, np.uint8, tile_bytes, off + 8)
        planes = tile[: words * BLOCK * 4].reshape(words, BLOCK, 4)
        for k in range(BLOCK):
            r = b * BLOCK + k
            if r >= hdr.rows or not tile[words * BLOCK * 4 + k] & 1:
                continue
            m = int(tile[words * BLOCK * 4 + k])
            mask[r] = m
            for c, eb in enumerate(elem_bytes):
                if not m & absent_bits[c]:
                    elems[c][r] = planes[first[c]:first[c + 1], k, :].reshape(-1)[:eb].tobytes()
    return hdr.rows, mask, elems


def test_export_of_a_queued_frame_matches_peek():
    eng = _presence_engine(1400, 0, (5, 4))
    _drive(eng, P2PTraceSession(2, 8, seed=3, p_clean=0.3), 20)
    f = eng.snapshot_frames()[0]
    rows, mask, elems = _image(eng, f, [4, 4, 12], [2, 4, 0])
    for c in range(3):
        data, has = eng.peek(f, c, 0, rows)
        assert [e is not None for e in elems[c]] == has.astype(bool).tolist()
        assert all(data[r].tobytes() == elems[c][r] for r in range(rows) if has[r])


def _drive_twins(worlds, sess, ticks):
    """One P2P trace replayed on several worlds (engine and oracle): every world gets the same request vectors."""
    for _ in range(ticks):
        for h in range(sess.num_players()):
            sess.add_local_input(h, 0)
        reqs = sess.advance_frame()
        outs = [w.handle_requests(sess.info(), reqs) for w in worlds]
        assert all(o == outs[0] for o in outs), "the engine's checksums differ from the oracle's"
        for f, c in outs[0]:
            sess.save_cell(f, c)


def _die_in_window(eng):  # rows whose Health reaches 0 inside the window of the frames checked below
    for r, h in ((1, 24), (2, 29), (5, 31)):
        if r < eng_rows(eng):
            eng.write_component(1, r, np.array([h], np.uint32))


def eng_rows(eng):
    return eng.row_count()


@pytest.mark.usefixtures("generic_kernel")
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n", [6, 1400])
def test_digest_equals_the_oracle_on_queued_and_retained_frames(path, n):
    eng = _presence_engine(n, path, (3, 4), _die_in_window)
    orc = _presence_engine(n, 0, (3, 4), _die_in_window, oracle=True)
    _drive_twins([eng, orc], P2PTraceSession(2, 6, seed=21, p_clean=0.3), 40)
    assert eng.retained_frames() == orc.retained_frames() and len(eng.retained_frames()) == 4
    for f in eng.snapshot_frames() + eng.retained_frames():
        h, words = eng.frame_digest(f)
        rows, active, expect = orc.frame_digest(f)
        assert h.frame == f and h.n_columns == 3 and h.rows == rows and h.n_blocks == (rows + BLOCK - 1) // BLOCK
        assert np.array_equal(words, expect), f
        assert h.active == active and h.elapsed_ns == f * 1_000_000_000 // 60
        assert h.root == LIB.bgr_seahash(words.tobytes(), words.nbytes)
        assert list(h.rng) == [0, 0, 0, 0]
    assert any(orc.frame_digest(f)[1] < n for f in eng.retained_frames()) or n < 6


def test_digest_of_the_particles_world_with_spawn_on_the_bundle():
    eng = _particles_engine(700, (2, 4), spawn_seed=77)
    orc = RetainOracleWorld(max_entities=700 + 64, max_depth=8)
    cols = register_particles(orc, spawn_rate=4, rng_seed=77)
    orc.retain_confirmed(2, 4)
    orc.build()
    populate(orc, cols, *synth_particles(700, 3, 40, 400))
    _drive_twins([eng, orc], P2PTraceSession(2, 8, seed=4, p_clean=0.3), 30)
    assert eng.last_kernel().kind == "bundle"
    assert eng.retained_frames() == orc.retained_frames()
    for f in eng.snapshot_frames()[::3] + eng.retained_frames():
        h, words = eng.frame_digest(f)
        rows, active, expect = orc.frame_digest(f)
        assert np.array_equal(words, expect), f
        assert h.rows == rows and h.active == active


def test_rng_is_in_the_header_and_not_in_the_blocks():
    """Two spawn-registered engines whose seeds differ and that never spawn: equal blocks, different ParticleRng."""
    def run(seed):
        eng = _particles_engine(1500, (1, 4), spawn_seed=seed)
        for t in range(12):
            reqs = [Request(SAVE, t), Request(ADVANCE, 0, [0, 0], [0, 0])]
            eng.handle_requests((SESSION_P2P, 8, 0, t - 2), reqs)
        return eng
    a, b = run(1), run(2)
    f = a.retained_frames()[0]
    da, db = a.frame_digest(f), b.frame_digest(f)
    assert np.array_equal(da[1], db[1]) and list(da[0].rng) != list(db[0].rng)
    assert digest_mismatch(da, db) == ([], 1)
    rep = a.diff_remote(f, b.export_blocks(f, range(da[0].n_blocks)))
    assert rep.host_state_differs & 1 and rep.rows_differing == 0 and len(rep.records) == 0


@pytest.mark.parametrize("n", [1400, 1_000_000])
def test_digest_folds_to_the_frames_checksum(n):
    eng = _presence_engine(n, 0, (5, 3))
    latest, _ = _drive(eng, P2PTraceSession(2, 8, seed=2, p_clean=0.3), 30 if n < 10**5 else 20)
    frames = eng.snapshot_frames() + eng.retained_frames()
    assert frames
    for f in frames:
        h, words = eng.frame_digest(f)
        p = capi.bgr_partial()
        p.frame, p.n_columns, p.active, p.total = f, 3, h.active, h.rows
        x = np.bitwise_xor.reduce(words, axis=0)
        p.xor_[0], p.xor_[1], p.xor_[2] = int(x[0]), int(x[1]), int(x[2])   # ck slots follow column order
        cs = capi.bgr_checksum()
        assert LIB.bgr_fold_partials(C.byref(p), C.byref(cs)) == 0
        assert cs.lo == latest[f], f


# ---- two peers ----
def _edit_b(eng):
    eng.write_component(2, 7, np.array([[1, 2, 3]], np.uint32))       # block 0: a word of Tag (no system writes it)
    eng.write_component(1, 2 * BLOCK + 11, np.array([1], np.uint32))  # block 2: Health 1, despawned by the first Advance
    eng.remove_component(1, 2 * BLOCK + 40)                              # block 2: a removed optional component


def _peers(b_tweak=None, b_edit=None, p_clean=0.3, flags=0, twins=False, round_trip=3, ticks=40):
    """Peers A and B (and, with twins, their oracle twins) on differently seeded P2P traces with desync detection every
    5 frames.  The run stops `round_trip` ticks after the first frame whose reported checksums differ, as GGRS raises
    DesyncDetected a round trip after the frame was confirmed.  Returns (a, b, reports_a, reports_b, oracles, frame)."""
    a, b = _presence_engine(1400, flags, (5, 4)), _presence_engine(1400, flags, (5, 4), b_tweak)
    oa = ob = None
    if twins:
        oa, ob = _presence_engine(1400, 0, (5, 4), oracle=True), _presence_engine(1400, 0, (5, 4), b_tweak, oracle=True)
    sa = P2PTraceSession(2, 8, seed=100, p_clean=p_clean, desync_interval=5)
    sb = P2PTraceSession(2, 8, seed=200, p_clean=p_clean, desync_interval=5)
    ra, rb, detected, left = {}, {}, None, None
    for t in range(ticks):
        for eng, orc, sess in ((a, oa, sa), (b, ob, sb)):
            if b_edit and eng is b:
                b_edit(eng, t)
                if orc is not None:
                    b_edit(orc, t)
            for h in range(2):
                sess.add_local_input(h, 0)
            reqs = sess.advance_frame()
            out = eng.handle_requests(sess.info(), reqs)
            if orc is not None:
                assert orc.handle_requests(sess.info(), reqs) == out
            for f, c in out:
                sess.save_cell(f, c)
        ra.update(sa.checksum_reports())
        rb.update(sb.checksum_reports())
        if detected is None:
            bad = sorted(f for f in set(ra) & set(rb) if ra[f] != rb[f])
            if bad:
                detected, left = bad[0], round_trip
        elif left is not None:
            left -= 1
            if left == 0:
                break
    return a, b, ra, rb, (oa, ob), detected


@pytest.mark.usefixtures("generic_kernel")
@pytest.mark.parametrize("path", PATHS)
def test_deterministic_peers_have_equal_digests(path):
    a, b, ra, rb, _, detected = _peers(flags=path)
    assert ra == rb and ra and detected is None
    common = set(a.retained_frames()) & set(b.retained_frames())
    assert len(common) >= 3
    for f in common:
        da, db = a.frame_digest(f), b.frame_digest(f)
        assert da[0].root == db[0].root
        assert digest_mismatch(da, db) == ([], 0)


def test_peers_with_a_different_initial_population_mismatch_in_exactly_those_blocks():
    a, b, ra, rb, (oa, ob), f = _peers(b_tweak=_edit_b, twins=True)
    assert f is not None and f in a.retained_frames() and f in b.retained_frames()  # still held when the report lands
    da, db = a.frame_digest(f), b.frame_digest(f)
    wa, wb = oa.frame_digest(f)[2], ob.frame_digest(f)[2]
    assert np.array_equal(da[1], wa) and np.array_equal(db[1], wb)
    oracle_blocks = [int(k) for k in np.nonzero((wa != wb).any(axis=1))[0]]
    blocks, host = digest_mismatch(da, db)
    assert blocks == oracle_blocks == [0, 2] and host == 0
    for g in set(a.retained_frames()) & set(b.retained_frames()):
        assert digest_mismatch(a.frame_digest(g), b.frame_digest(g))[0] == [0, 2], g
    blob = b.export_blocks(f, blocks)
    for cap in (1, 2, 3, 31, 32, 33, 100000):
        rep, expect = a.diff_remote(f, blob, cap), two_world_diff(oa, ob, f, blocks, cap)
        assert rep.summary_tuple() == expect.summary_tuple(), cap
        assert rep.columns == expect.columns
        assert np.array_equal(rep.records, expect.records), cap
    assert rep.by_name["Tag"].rows == 1 and rep.by_name["Health"].presence == 1
    again = a.diff_remote(f, blob, 33)
    assert again.summary_tuple() == a.diff_remote(f, blob, 33).summary_tuple()
    assert np.array_equal(again.records, a.diff_remote(f, blob, 33).records)


def test_a_mid_session_edit_mismatches_later_frames_only():
    def edit(eng, t):
        if t == 22:
            eng.write_component(2, BLOCK + 5, np.array([[9, 9, 9]], np.uint32))
    a, b, ra, rb, _, detected = _peers(b_edit=edit, p_clean=1.0, round_trip=None)
    assert detected == 25 and all(ra[f] == rb[f] for f in ra if f < 22)
    for f in set(a.retained_frames()) & set(b.retained_frames()):
        blocks, _ = digest_mismatch(a.frame_digest(f), b.frame_digest(f))
        assert blocks == ([1] if f >= 22 else []), f


# ---- refusals ----
def test_retention_refusals():
    e = Engine(max_entities=64, max_depth=8)
    e.rollback_component("A", 4)
    with pytest.raises(BgrError) as ei:
        e.retain_confirmed(0, 2)
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    with pytest.raises(BgrError) as ei:
        e.retain_confirmed(3, 0)
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    e.build()
    with pytest.raises(BgrError) as ei:
        e.retain_confirmed(3, 2)
    assert ei.value.status == capi.BGR_ERR_STATE
    s = Engine(max_entities=64, max_depth=8, flags=capi.BGR_CFG_SHARDED)
    with pytest.raises(BgrError) as ei:
        s.retain_confirmed(3, 2)
    assert ei.value.status == capi.BGR_ERR_UNSUPPORTED
    big = Engine(max_entities=64, max_depth=30, flags=capi.BGR_CFG_DESYNC_CAPTURE)
    big.rollback_component("A", 4)
    big.retain_confirmed(1, 5)
    with pytest.raises(BgrError) as ei:
        big.build()
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and "60" in str(ei.value) and "65" in str(ei.value)


def test_blob_refusals_and_unknown_frames():
    a, b, _, _, _, _ = _peers()
    f = a.retained_frames()[0]
    assert a.frame_digest(10**6) is None and a.export_blocks(10**6, [0]) is None
    blob = bytearray(b.export_blocks(f, [0, 2]))
    hdr = C.sizeof(capi.bgr_frame_blob_header)
    tile = (len(blob) - hdr) // 2

    def refused(data, frame=f):
        with pytest.raises(BgrError) as ei:
            a.diff_remote(frame, bytes(data))
        assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
        return str(ei.value)

    bad = bytearray(blob); bad[0] ^= 1
    assert "magic" in refused(bad)
    bad = bytearray(blob); bad[4] = 9
    assert "version" in refused(bad)
    bad = bytearray(blob); bad[8] ^= 1
    assert "layout" in refused(bad)
    assert "frame" in refused(blob, f + 1)
    assert "truncated" in refused(blob[:-1])
    assert "truncated" in refused(blob[:10])
    bad = bytearray(blob); struct.pack_into("<I", bad, hdr + tile, 99)
    assert ">=" in refused(bad)
    bad = bytearray(blob); struct.pack_into("<I", bad, hdr + tile, 0)
    assert "unsorted" in refused(bad)
    bad = bytearray(blob); struct.pack_into("<I", bad, hdr, 2); struct.pack_into("<I", bad, hdr + tile, 0)
    assert "unsorted" in refused(bad)
    other = Engine(max_entities=1408, max_depth=8)
    other.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    other.rollback_component("Health", 8, capi.BGR_STRATEGY_CLONE | OPT)
    other.rollback_component("Tag", 12)
    other.retain_confirmed(5, 4)
    other.build()
    other.spawn(1400)
    _drive(other, P2PTraceSession(2, 8, seed=100, p_clean=0.3), 40)
    with pytest.raises(BgrError) as ei:
        a.diff_remote(f, other.export_blocks(f, [0]))
    assert "layout" in str(ei.value)
    with pytest.raises(BgrError) as ei:
        digest_mismatch(a.frame_digest(f), other.frame_digest(f))
    assert "layout" in str(ei.value)
    with pytest.raises(BgrError) as ei:
        a.export_blocks(f, [2, 0])
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    with pytest.raises(BgrError) as ei:
        a.export_blocks(f, [3])
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT


def test_reset_session_releases_retained_frames():
    a, _, _, _, _, _ = _peers()
    assert a.retained_frames()
    a.reset_session()
    assert a.retained_frames() == []


def test_exported_rows_past_the_row_count_are_zero():
    a, _, _, _, _, _ = _peers()
    f = a.retained_frames()[0]
    blob = a.export_blocks(f, [2])
    hdr = C.sizeof(capi.bgr_frame_blob_header)
    tile = np.frombuffer(blob[hdr + 8:], np.uint8)
    words = 5
    planes = tile[: words * BLOCK * 4].reshape(words, BLOCK, 4)
    r0 = 1400 - 2 * BLOCK
    assert not planes[:, r0:].any() and not tile[words * BLOCK * 4 + r0:].any()
    assert tile[words * BLOCK * 4: words * BLOCK * 4 + r0].any()
