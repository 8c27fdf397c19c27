"""-m gpu: stable-plane elision of the bundle kernel's active planes (content stamps, engine.cu HostState).

A warp stores an active plane of its 64-row segment into a slot or the live image only when the image does not already
hold that content.  Each case runs the same calls on the default engine, on an engine created with BGR_TUNE_BUNDLE=0
(the generic one-launch program or the stepwise path: whole images, no stamps) and on the oracle.  Checksums are equal on
every tick.  The live world and every snapshot hold the oracle's bytes on every live row, and the whole-image engine's
passive bytes on every row below the row count.  Row counts are not multiples of 64 or 512.  The engine elides on
grids of several waves only; BGR_TUNE_PASSIVE_EARLY=0 gives these small worlds that configuration."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import SAVE, P2PTraceSession, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
PASSIVE = slice(12, 40)
SPAWN, NOOP = 1 << 4, 1 << 5
SEG_ROWS, TILE_ROWS = 64, 512


def _no_finite(w, t, v):   # the example's checksums without the finite assertion: NaN rows are allowed
    w.checksum_component(v, 0, 12, 0)
    w.checksum_component(t, 0, 12, 0)


def _population(n, edges, nan):
    """The stress population with z != 0 on a fifth of the rows; `edges` adds velocity.x = -0.0 and subnormals, ttl
    values that cross 2^32 and ttl values that reach 0 inside the window; `nan` puts NaNs into velocity.y."""
    tf, vel, ttl = synth_particles(n, 41, 30, 60, z_fraction=0.2)
    tf[:, 3:10] = np.random.default_rng(n).uniform(-2.0, 2.0, (n, 7))
    if edges:
        vel[5::97, 0] = np.float32(-0.0)
        vel[7::101, 0] = np.float32(1e-40)
        vel[9::103, 2] = np.float32(-1e-42)
        ttl[11::89] = (1 << 32) + np.arange(len(ttl[11::89]), dtype=np.uint64) % 6
        ttl[13::53] = 2 + np.arange(len(ttl[13::53]), dtype=np.uint64) % 5
    if nan:
        vel[3::71, 1] = np.float32(np.nan)
        vel[4::73, 1] = np.frombuffer(np.uint32(0x7FC12345).tobytes(), dtype=np.float32)[0]
    return tf, vel, ttl


def _build(w, n, spawn_rate, optional, retain, edges, nan):
    if optional:
        t = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
        v = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY | OPT)
        l = w.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY | OPT)
        w.checksum_component(v, 0, 12, FIN)
        w.checksum_component(t, 0, 12, FIN)
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        cols = (t, v, l)
    else:
        cols = register_particles(w, spawn_rate=spawn_rate, spawn_ttl=9, checksums=_no_finite if nan else None)
    if retain:
        w.retain_confirmed(*retain)
    w.build()
    populate(w, cols, *_population(n, edges, nan))
    return cols


class Worlds:
    """The default engine `g`, the whole-image engine `s` (BGR_TUNE_BUNDLE=0) and the oracle `o`, built identically."""

    def __init__(self, monkeypatch, n, spawn_rate=0, optional=False, flags=0, retain=None, extra_rows=0, edges=True,
                 nan=False, multi_wave=True):
        with monkeypatch.context() as m:
            if multi_wave:
                m.setenv("BGR_TUNE_PASSIVE_EARLY", "0")
            self.g = Engine(max_entities=n + extra_rows, max_depth=9, flags=flags)
        with monkeypatch.context() as m:
            m.setenv("BGR_TUNE_BUNDLE", "0")
            self.s = Engine(max_entities=n + extra_rows, max_depth=9, flags=flags)
        self.o = OracleWorld()
        for w in self.all():
            self.cols = _build(w, n, spawn_rate, optional, retain if w is not self.o else None, edges, nan)
        self.rng = np.random.default_rng(7)

    def all(self):
        return (self.g, self.s, self.o)

    def tick(self, info, reqs, elide=True):
        out = [w.handle_requests(info, reqs) for w in self.all()]
        assert out[0] == out[1] == out[2], reqs
        k = self.g.last_kernel()
        assert k.kind == "bundle" and self.s.last_kernel().kind != "bundle"
        assert elide is None or k.stable_planes == elide
        return k

    def _same(self, got, ref, orc, c):
        (vg, hg), (vs, hs), (vo, ho) = got, ref, orc
        m = ho.astype(bool)
        assert np.array_equal(hg.astype(bool), m) and np.array_equal(hs.astype(bool), m), c
        assert np.array_equal(vg[m], np.asarray(vo)[m]) and np.array_equal(vs[m], np.asarray(vo)[m]), c
        if c == self.cols[0]:
            assert np.array_equal(vg[:, PASSIVE], vs[:, PASSIVE])

    def check(self):
        g, s, o = self.all()
        n = g.row_count()
        assert s.row_count() == o.row_count() == n
        frames = g.snapshot_frames()
        assert frames == s.snapshot_frames() == o.snapshot_frames()
        assert np.array_equal(g.read_alive(0, n).astype(bool), o.read_alive(0, n).astype(bool))
        for c in self.cols:
            self._same((g.read_component(c, 0, n), g.has_component(c, 0, n)),
                       (s.read_component(c, 0, n), s.has_component(c, 0, n)), o.read_component_alive(c, 0, n), c)
        for f in frames:
            rows = g.frame_digest(f)[0].rows
            assert s.frame_digest(f)[0].rows == rows
            for c in self.cols:
                self._same(g.peek(f, c, 0, rows), s.peek(f, c, 0, rows), o.peek(f, c, 0, rows), c)

    def close(self):
        for w in self.all():
            w.close()


def _vectors(session, ticks, spawn=False, seed=0xB200, d=8):
    sess = SyncTestSession(2, d, 9, input_delay=2) if session == "synctest" else P2PTraceSession(2, 8, 2, seed=seed)
    out = []
    for t in range(ticks):
        sess.add_local_input(0, SPAWN if spawn and t % 7 in (2, 3) else 0)
        sess.add_local_input(1, NOOP if t % 3 == 0 else 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        out.append((sess.info(), reqs))
    return out


@pytest.mark.parametrize("session,n", [("synctest", 70_001), ("p2p", 9_001), ("synctest", 5_003)])
def test_stress_world_with_edge_values(monkeypatch, session, n):
    """SyncTest d=8 and the C4 P2P trace (rollbacks of varying depth) over z planes that move in some warps only,
    velocity.x = -0.0 and subnormals, ttl crossing 2^32 and reaching 0 (despawn, then rollbacks bring rows back)."""
    w = Worlds(monkeypatch, n)
    for t, (info, reqs) in enumerate(_vectors(session, 30)):
        w.tick(info, reqs)
        if t in (4, 12):
            w.check()
    w.check()
    w.close()


def test_spawning_world(monkeypatch):
    rate, ticks = 24, 40
    w = Worlds(monkeypatch, 6_001, spawn_rate=rate, extra_rows=rate * ticks)
    for t, (info, reqs) in enumerate(_vectors("p2p", ticks, spawn=True)):
        w.tick(info, reqs)
        if t == 20:
            w.check()
    assert w.g.row_count() > 6_001 + rate
    w.check()
    w.close()


def test_host_writers_between_ticks(monkeypatch):
    """After the ring is full: every host writer of the live image between two ticks — translation.z and velocity.x
    writes, despawn, spawn, the startup system — then ticks whose Loads go back to frames from before the write."""
    n, rate = 9_001, 16
    w = Worlds(monkeypatch, n, spawn_rate=rate, extra_rows=4096)
    t_col, v_col, _ = w.cols
    vectors = _vectors("synctest", 40)
    for t, (info, reqs) in enumerate(vectors):
        if t == 12:   # translation.z of a band of rows
            vals = w.g.read_component(t_col, 100, 3000).view(np.float32).copy()
            vals[:, 2] = w.rng.uniform(-9.0, 9.0, 3000)
            for x in w.all():
                x.write_component(t_col, 100, vals)
        if t == 15:   # velocity.x = -0.0 on scattered rows
            vals = w.g.read_component(v_col, 2000, 500).view(np.float32).copy()
            vals[::3, 0] = np.float32(-0.0)
            for x in w.all():
                x.write_component(v_col, 2000, vals)
        if t == 18:
            for r in (0, 63, 64, 4097, n - 1):
                for x in w.all():
                    x.despawn(r)
        if t == 21:
            for x in w.all():
                x.spawn(37)
        if t == 24:
            for x in w.all():
                x.run_startup_system(capi.BGR_SYS_PARTICLES_SPAWN)
        w.tick(info, reqs)
        if t in (13, 19, 25):
            w.check()
    w.check()
    w.close()


def test_mode2_remove_and_insert_between_ticks(monkeypatch):
    n = 6_007
    w = Worlds(monkeypatch, n, optional=True)
    _, v, l = w.cols
    for t, (info, reqs) in enumerate(_vectors("synctest", 28)):
        if t in (10, 11, 14):
            alive = w.o.read_alive(0, n).astype(bool)
            rows = [r for r in range(t * 7, n, 331) if alive[r]]
            for r in rows:
                col = v if r % 2 else l
                if t == 14:
                    value = w.g.read_component(col, r - 1, 1)[0]
                    for x in w.all():
                        x.insert_component(col, r, value)
                else:
                    for x in w.all():
                        x.remove_component(col, r)
        w.tick(info, reqs)
        if t in (12, 16):
            w.check()
    w.check()
    w.close()


@pytest.mark.parametrize("kind", ["capture", "retain"])
def test_capture_and_retention(monkeypatch, kind):
    """Desync capture hands witness slots out again, retention keeps confirmed frames: stamps follow the image index.
    The digest of a retained frame equals the whole-image engine's."""
    rate, ticks = 12, 70
    flags, retain = (capi.BGR_CFG_DESYNC_CAPTURE, None) if kind == "capture" else (0, (10, 4))
    w = Worlds(monkeypatch, 5_001, spawn_rate=rate, flags=flags, retain=retain, extra_rows=rate * ticks)
    for t, (info, reqs) in enumerate(_vectors("p2p", ticks, spawn=True)):
        w.tick(info, reqs)
    w.check()
    if kind == "capture":
        frames = w.g.desync_frames()
        assert frames and frames == w.s.desync_frames()
        for f in frames:
            rows = w.g.desync_diff(f).rows_first
            assert w.s.desync_diff(f).rows_first == rows
            for c in w.cols:
                (vg, hg), (vs, hs) = w.g.peek_first(f, c, 0, rows), w.s.peek_first(f, c, 0, rows)
                m = hs.astype(bool)
                assert np.array_equal(hg, hs) and np.array_equal(vg[m], vs[m])
    else:
        frames = w.g.retained_frames()
        assert frames and frames == w.s.retained_frames()
        for f in frames:
            (hg, dg), (hs, ds) = w.g.frame_digest(f), w.s.frame_digest(f)
            assert hg.rows == hs.rows and hg.root == hs.root and np.array_equal(dg, ds)
    w.close()


def test_reset_session_and_set_depth(monkeypatch):
    w = Worlds(monkeypatch, 4_099)
    for info, reqs in _vectors("synctest", 16):
        w.tick(info, reqs)
    frame = w.g.rollback_frame_count()
    for x in w.all():
        x.reset_session()
        x.set_rollback_frame_count(frame)
        x.set_depth(3)
    w.check()
    sess = P2PTraceSession(2, 8, 2, seed=0xC4)
    sess.current_frame = frame
    for t in range(30):
        sess.add_local_input(0, 0)
        sess.add_local_input(1, NOOP if t % 3 == 0 else 0)
        w.tick(sess.info(), sess.advance_frame())
    w.check()
    w.close()


def test_four_vectors_in_flight_then_synchronous(monkeypatch):
    """Overlapping launches (per-tile dependencies) read the stamps the previous launch wrote, then synchronous calls."""
    n, ticks = 120_001, 40
    w = Worlds(monkeypatch, n)
    vectors = _vectors("synctest", ticks)
    got, inflight = [], 0
    for info, reqs in vectors[:30]:
        w.g.submit_requests(info, reqs)
        inflight += 1
        if inflight == 4:
            got += w.g.collect()
            inflight -= 1
    while inflight:
        got += w.g.collect()
        inflight -= 1
    want = [w.o.handle_requests(info, reqs) for info, reqs in vectors[:30]]
    assert [w.s.handle_requests(info, reqs) for info, reqs in vectors[:30]] == want
    assert got == [c for out in want for c in out]
    for info, reqs in vectors[30:]:
        w.tick(info, reqs)
    w.check()
    w.close()


def test_steady_state_stores_four_planes_per_segment(monkeypatch):
    """Clean P2P ticks (Save, Advance) of a 2-D world with long ttl: a steady-state Save stores exactly translation.x/y,
    velocity.y and ttl.lo of every segment (4 x 4 units of 64 B; all nine planes are 33 units).  After a host write the first Save into each slot stores all nine planes
    (the live image's stamps are unknown); the tick right after the write also writes the live image whole."""
    n = 64 * TILE_ROWS
    segs = n // SEG_ROWS
    monkeypatch.setenv("BGR_TUNE_PASSIVE_EARLY", "0")
    w = Engine(max_entities=n, max_depth=8)
    cols = register_particles(w)
    w.build()
    tf, vel, ttl = synth_particles(n, 5, 100_000, 200_000)
    populate(w, cols, tf, vel, ttl)
    sess = P2PTraceSession(2, 8, 2, seed=1, p_clean=1.0)

    def run(ticks):
        w.trace_enable(ticks)
        kinds = []
        for _ in range(ticks):
            sess.add_local_input(0, 0)
            sess.add_local_input(1, 0)
            w.handle_requests(sess.info(), sess.advance_frame())
            kinds.append(w.last_kernel())
        tr = w.trace_read(ticks)
        w.trace_enable(0)
        assert all(k.kind == "bundle" and k.stable_planes for k in kinds)
        return [int(r[3]) for r in tr], kinds

    run(20)
    stored, kinds = run(8)
    assert all(k.deferred_live for k in kinds)
    assert stored == [16 * segs] * 8
    vals = w.read_component(cols[0], 0, 100).view(np.float32).copy()
    vals[:, 2] = 1.5
    w.write_component(cols[0], 0, vals)
    stored, kinds = run(24)
    assert not kinds[0].deferred_live and stored[0] == 33 * segs + 33 * segs
    full = [s for s in stored[1:] if s == 33 * segs]
    assert 1 <= len(full) <= 8 and stored[1:1 + len(full)] == full
    assert stored[1 + len(full):] == [16 * segs] * (23 - len(full))
    w.close()


def test_worlds_crossing_the_one_wave_size(monkeypatch):
    """A spawning P2P world around the one-wave size (3 blocks of 512 rows per SM): spawns take it to several waves
    (stamped launches), rollbacks to frames before them bring it back to one (launches without stamps, which leave the
    table stale), again and again.  Default configuration."""
    import torch
    edge = 3 * torch.cuda.get_device_properties(0).multi_processor_count * TILE_ROWS
    rate, ticks, n = 512, 40, edge - 700
    w = Worlds(monkeypatch, n, spawn_rate=rate, extra_rows=rate * ticks, multi_wave=False)
    sides = set()
    for t, (info, reqs) in enumerate(_vectors("p2p", ticks, spawn=True)):
        sides.add(w.tick(info, reqs, elide=None).stable_planes)
        if t in (12, 25):
            w.check()
    assert sides == {True, False}
    w.check()
    w.close()


def test_single_wave_grids_store_every_plane(monkeypatch):
    """A one-wave world runs the instance without stamps: whole active planes, as before the elision."""
    w = Worlds(monkeypatch, 20_011, multi_wave=False)
    for info, reqs in _vectors("synctest", 16):
        w.tick(info, reqs, elide=False)
    w.check()
    w.close()
