"""-m gpu: content-version elision of the passive planes on the default engine.

A Save into a slot that already holds the live image's passive planes (Transform.rotation / scale: no registered system
writes them) stores none of them, and a Load from such a slot rewrites none (engine.cu HostState::slot_passive_ver).
Each case runs the same calls on the default engine, on a BGR_CFG_FORCE_STEPWISE engine (whole-image copies, no
elision) and on the oracle.  Checksums equal the oracle's on every tick.  The live world and every snapshot hold the
oracle's bytes on every live row, and the stepwise engine's passive bytes on every row below the row count, dead rows
included.  Dead rows' active planes are not compared: the bundle kernel keeps stepping them, the stepwise systems do not,
and neither is observable."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import SAVE, P2PTraceSession, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
PASSIVE = slice(12, 40)   # Transform bytes: rotation 16 + scale 12
SPAWN, NOOP = 1 << 4, 1 << 5


def _build(w, n, spawn_rate, optional, retain):
    if optional:   # MODE 2: Velocity and Ttl can be removed from single entities
        t = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
        v = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY | OPT)
        l = w.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY | OPT)
        w.checksum_component(v, 0, 12, FIN)
        w.checksum_component(t, 0, 12, FIN)
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        cols = (t, v, l)
    else:
        cols = register_particles(w, spawn_rate=spawn_rate, spawn_ttl=9)
    if retain:
        w.retain_confirmed(*retain)
    w.build()
    tf, vel, ttl = synth_particles(n, 41, 3, 40, z_fraction=0.2)
    tf[:, 3:10] = np.random.default_rng(n).uniform(-2.0, 2.0, (n, 7))   # a distinct rotation / scale on every row
    populate(w, cols, tf, vel, ttl)
    return cols


class Worlds:
    """The default engine `g`, the stepwise engine `s` and the oracle `o`, built identically."""

    def __init__(self, n, spawn_rate=0, optional=False, flags=0, retain=None, extra_rows=0):
        self.g = Engine(max_entities=n + extra_rows, max_depth=8, flags=flags)
        self.s = Engine(max_entities=n + extra_rows, max_depth=8, flags=flags | capi.BGR_CFG_FORCE_STEPWISE)
        self.o = OracleWorld()
        for w in (self.g, self.s, self.o):
            self.cols = _build(w, n, spawn_rate, optional, retain if w is not self.o else None)
        self.rng = np.random.default_rng(7)

    def all(self):
        return (self.g, self.s, self.o)

    def tick(self, info, reqs):
        out = [w.handle_requests(info, reqs) for w in self.all()]
        assert out[0] == out[1] == out[2], reqs
        assert self.g.last_path_fused() and self.g.last_kernel().kind == "bundle"
        return self.g.last_kernel()

    def write_passive(self, first, count, part):
        """The host overwrites rotation (part 0) or scale (part 1) of `count` rows, translation kept."""
        t = self.cols[0]
        vals = self.g.read_component(t, first, count).view(np.float32).copy()
        cols = slice(3, 7) if part == 0 else slice(7, 10)
        vals[:, cols] = self.rng.uniform(-3.0, 3.0, (count, cols.stop - cols.start))
        for w in self.all():
            w.write_component(t, first, vals)

    def _same(self, got, ref, orc, c):
        (vg, hg), (vs, hs), (vo, ho) = got, ref, orc
        m = ho.astype(bool)
        assert np.array_equal(hg.astype(bool), m) and np.array_equal(hs.astype(bool), m), c
        assert np.array_equal(vg[m], np.asarray(vo)[m]), c
        if c == self.cols[0]:
            assert np.array_equal(vg[:, PASSIVE], vs[:, PASSIVE])   # every row, dead ones included

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


def _vectors(session, ticks, spawn=False, seed=0xB200):
    """Request vectors of a SyncTest (d=3) or C4 P2P session; with `spawn`, player 0 holds the spawn key now and then."""
    sess = SyncTestSession(2, 3, 8, input_delay=2) if session == "synctest" else P2PTraceSession(2, 8, 2, seed=seed)
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


@pytest.mark.parametrize("session,n", [("synctest", 4097), ("synctest", 250_000), ("p2p", 4097)])
def test_host_write_of_a_passive_column_between_ticks(session, n):
    """The host rewrites rotation, later scale, between ticks.  Later ticks roll back to frames saved before the write
    and save over slots that hold older versions; a later write lands while the ring is full of the earlier one."""
    w = Worlds(n)
    for t, (info, reqs) in enumerate(_vectors(session, 40)):
        if t in (12, 13, 25):
            w.write_passive(101 + 37 * t, min(n - 101 - 37 * t, 3000), t % 2)
        w.tick(info, reqs)
        if t in (14, 27):
            w.check()
    w.check()
    w.close()


def test_remove_and_insert_component_inside_the_window():
    """MODE 2: Velocity / Ttl removed from and inserted into single entities between ticks, inside the rollback
    window; Loads bring back frames from before each change."""
    n = 6000
    w = Worlds(n, optional=True)
    _, v, l = w.cols
    removed = {}
    for t, (info, reqs) in enumerate(_vectors("synctest", 30)):
        if 8 <= t < 20:
            alive = w.o.read_alive(0, n).astype(bool)
            if t % 3 == 2:   # put back what the previous tick removed
                for r in removed.pop(t - 1, []):
                    col = v if r % 2 else l
                    if alive[r]:
                        value = w.g.read_component(col, r - 1, 1)[0]
                        for x in w.all():
                            x.insert_component(col, r, value)
            else:
                removed[t] = [r for r in range(t * 5, n, 211) if alive[r]]
                for r in removed[t]:
                    for x in w.all():
                        x.remove_component(v if r % 2 else l, r)
        w.tick(info, reqs)
        if t == 15:
            w.check()
    w.check()
    w.close()


def test_spawns_under_four_pipelined_submits():
    """Spawns inside the window with four request vectors in flight on the default engine: a version bump falls
    between overlapping launches (per-tile dependencies), and the ticks after it store passive planes again."""
    n, ticks, rate = 120_000, 36, 24
    w = Worlds(n, spawn_rate=rate, extra_rows=rate * ticks)
    vectors = _vectors("synctest", ticks, spawn=True)
    got, inflight = [], 0
    for info, reqs in vectors:
        w.g.submit_requests(info, reqs)
        inflight += 1
        if inflight == 4:
            got += w.g.collect()
            inflight -= 1
    while inflight:
        got += w.g.collect()
        inflight -= 1
    want = [w.o.handle_requests(info, reqs) for info, reqs in vectors]
    assert [w.s.handle_requests(info, reqs) for info, reqs in vectors] == want
    assert got == [c for out in want for c in out]
    assert w.g.row_count() > n + rate
    w.check()
    w.close()


@pytest.mark.parametrize("kind", ["capture", "retain"])
def test_capture_and_retention_engines_on_the_p2p_trace(kind):
    """Desync capture hands first-image slots out again, retention keeps confirmed frames in slots of their own: the
    versions follow the slot index.  C4 P2P trace with spawns."""
    rate, ticks = 12, 90
    flags, retain = (capi.BGR_CFG_DESYNC_CAPTURE, None) if kind == "capture" else (0, (10, 4))
    w = Worlds(5000, spawn_rate=rate, flags=flags, retain=retain, extra_rows=rate * ticks)
    for t, (info, reqs) in enumerate(_vectors("p2p", ticks, spawn=True)):
        if t == 40:
            w.write_passive(300, 2000, 0)
        w.tick(info, reqs)
    w.check()
    t = w.cols[0]
    if kind == "capture":
        frames = w.g.desync_frames()
        assert frames and frames == w.s.desync_frames()
        for f in frames:
            rows = w.g.desync_diff(f).rows_first
            assert w.s.desync_diff(f).rows_first == rows
            (vg, hg), (vs, hs) = w.g.peek_first(f, t, 0, rows), w.s.peek_first(f, t, 0, rows)
            assert np.array_equal(hg, hs) and np.array_equal(vg[:, PASSIVE], vs[:, PASSIVE])
    else:
        frames = w.g.retained_frames()
        assert frames and frames == w.s.retained_frames()
        for f in frames:
            (hg, dg), (hs, ds) = w.g.frame_digest(f), w.s.frame_digest(f)
            assert hg.rows == hs.rows and hg.root == hs.root and np.array_equal(dg, ds)
    w.close()


def test_reset_session_then_a_new_session():
    """bgr_reset_session, a host write, then a new P2P session on the same engines: its first Saves go into slots
    that still hold the old session's versions."""
    w = Worlds(4097)
    for info, reqs in _vectors("synctest", 16):
        w.tick(info, reqs)
    frame = w.g.rollback_frame_count()
    for x in w.all():
        x.reset_session()
        x.set_rollback_frame_count(frame)   # Time<GgrsTime> only moves forward
    w.write_passive(50, 1500, 1)
    sess = P2PTraceSession(2, 8, 2, seed=0xC4)
    sess.current_frame = frame
    for t in range(30):
        sess.add_local_input(0, 0)
        sess.add_local_input(1, NOOP if t % 3 == 0 else 0)
        w.tick(sess.info(), sess.advance_frame())
    w.check()
    w.close()


def test_steady_state_ticks_move_no_passive_planes():
    """Elision is on by default: steady-state SyncTest ticks of a 250k world move no passive plane
    (BGR_KERNEL_PASSIVE_PLANES clear), though they launch the passive-TMA configuration.  The first tick after a host
    write of rotation moves them by TMA (its Load restores the slot's older planes into the live image); the ticks after
    it do not."""
    w = Worlds(250_000)
    vectors = _vectors("synctest", 24)
    for t, (info, reqs) in enumerate(vectors[:16]):
        k = w.tick(info, reqs)
    assert k.passive_tma and not k.passive_planes
    w.write_passive(1000, 5000, 0)
    k = w.tick(*vectors[16])
    assert k.passive_tma and k.passive_planes and not k.deferred_live
    for info, reqs in vectors[17:]:
        assert not w.tick(info, reqs).passive_planes
    w.check()
    w.close()
