"""Spawning worlds on the generic one-launch program: a world that registers spawn_particles but is not exactly the
particles bundle (a whole-Transform checksum, an extra column, BGR_TUNE_BUNDLE=0) ticks in ONE launch per request
vector on the interpreter and on the generated kernel (generic_kernel fixture), and its worlds can be batched.  Newborn
rows are written after the frame's systems and despawns, byte for byte what the oracle and the stepwise path write."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine, EngineBatch
from bevy_ggrs_b200.session import ADVANCE, SAVE, P2PTraceSession, Request, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld
from parity_util import compare_state, run_particles_synctest_pair

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
SPAWN = capi.BGR_INPUT_SPAWN


def whole_transform(w, t, v):
    """checksum_component_with_hash::<Transform> over all 40 bytes next to the example's Velocity checksum: not the
    bundle's checksum layout, so the world runs on the generic program."""
    w.checksum_component(v, 0, 12, FIN)
    w.checksum_component(t, 0, 40)


def kind_of(generic_kernel):
    return "generic_interpreter" if generic_kernel == "interpreter" else "generic_nvrtc"


def peeks_equal(eng, orc, cols):
    """Every ring snapshot of every column: presence and the bytes of every row that has the column."""
    n = eng.row_count()
    for f in eng.snapshot_frames():
        for c in cols:
            pe, po = eng.peek(f, c, 0, n), orc.peek(f, c, 0, n)
            if (pe is None) != (po is None):
                return False
            if pe is None:
                continue
            m = po[1].astype(bool)
            if not (np.array_equal(pe[1].astype(bool), m) and np.array_equal(pe[0][m], po[0][m])):
                return False
    return True


# ---- 1. oracle parity on SyncTest: whole-Transform checksum, and the bundle switched off ----
@pytest.mark.parametrize("n,rate,d,ticks", [(500, 40, 8, 16), (3000, 100, 3, 14), (1, 7, 6, 12)])
@pytest.mark.parametrize("setup", ["whole_transform", "bundle_off"])
def test_synctest_spawning_world_matches_the_oracle(monkeypatch, generic_kernel, setup, n, rate, d, ticks):
    """500 rows + 40 per spawning frame cross the first quarter tile and the first tile inside the window; every SyncTest
    tick rolls back over spawning frames, so rows are un-spawned and re-spawned from the rolled-back ParticleRng."""
    if setup == "bundle_off":
        monkeypatch.setenv("BGR_TUNE_BUNDLE", "0")
    r = run_particles_synctest_pair(n, d, ticks, seed=7 + n, ttl_lo=2, ttl_hi=30, spawn_rate=rate, spawn_ttl=9,
                                    startup_burst=True, peek_check=True, z_fraction=0.2,
                                    checksums=whole_transform if setup == "whole_transform" else None)
    assert r["fused"] and r["launches"] == ticks
    assert r["kernel"].kind == kind_of(generic_kernel)
    assert r["checksums_equal"] and r["state_equal"] and r["peek_equal"]
    assert r["rows"][0] == r["rows"][1] > n + rate
    assert r["ring"][0] == r["ring"][1] and r["active"][0] == r["active"][1]
    assert r["mismatch_events"] == (0, 0)


# ---- 2. P2P: rollbacks of random depth reach back before spawning frames ----
def _particles_pair(n, rate, ttl, seed, checksums=whole_transform, extra=False):
    """The engine and the oracle with the same spawning registration and seeded population."""
    eng = Engine(max_entities=n + rate * 64, max_depth=9)
    orc = OracleWorld()
    cols = None
    for w in (eng, orc):
        cols = register_particles(w, spawn_rate=rate, spawn_ttl=ttl, rng_seed=seed, checksums=checksums)
        if extra:
            cols = cols + (_add_score(w),)
        w.build()
        populate(w, cols[:3], *synth_particles(n, seed, 2, 40, 0.2))
    return eng, orc, cols


def _add_score(w):
    """An optional 4-byte Score (+1 per frame) behind the particles columns; spawned rows carry it, zeroed."""
    s = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    w.checksum_component(s, 0, 4)
    w.add_system(capi.BGR_SYS_U32_ADD, [s], [0, 1])
    return s


def _p2p_vectors(ticks, mp, seed):
    """Request vectors of a 2-peer P2P trace; player 0 presses INPUT_SPAWN on two ticks in five."""
    sess = P2PTraceSession(2, max_prediction=mp, input_delay=2, seed=seed, p_clean=0.3)
    out = []
    for t in range(ticks):
        sess.add_local_input(0, SPAWN if t % 5 in (1, 2) else 0)
        reqs = sess.advance_frame()
        for q in reqs:
            if q.kind == SAVE:
                sess.save_cell(q.frame, 0)
        out.append((sess.info(), reqs))
    return out


@pytest.mark.parametrize("n,rate", [(500, 40), (2000, 130)])
def test_p2p_rollbacks_before_a_spawn_match_the_oracle(generic_kernel, n, rate):
    eng, orc, cols = _particles_pair(n, rate, 11, seed=n)
    for info, reqs in _p2p_vectors(40, 6, seed=0x5A + n):
        l0 = eng.launch_count()
        assert eng.handle_requests(info, reqs) == orc.handle_requests(info, reqs)
        assert eng.launch_count() - l0 == 1 and eng.last_kernel().kind == kind_of(generic_kernel)
    rows = eng.row_count()
    assert rows == orc.row_count() > n + rate
    assert eng.active_count() == orc.active_count()
    assert eng.snapshot_frames() == orc.snapshot_frames()
    assert compare_state(eng, orc, cols, rows) and peeks_equal(eng, orc, cols)
    # every Transform word of every newborn row in every snapshot: ten words, rotation.w and scale 1
    for f in eng.snapshot_frames():
        pe, po = eng.peek(f, cols[0], n, rows - n), orc.peek(f, cols[0], n, rows - n)
        m = po[1].astype(bool)
        assert np.array_equal(pe[0][m].view(np.uint32), po[0][m].view(np.uint32))


# ---- 3. the stepwise twin: every column of every snapshot, the zeroed extra column and its presence ----
def test_stepwise_twin_is_byte_equal(generic_kernel):
    n, rate = 700, 60
    eng, orc, cols = _particles_pair(n, rate, 8, seed=3, extra=True)
    twin = Engine(max_entities=n + rate * 64, max_depth=9, flags=capi.BGR_CFG_FORCE_STEPWISE)
    register_particles(twin, spawn_rate=rate, spawn_ttl=8, rng_seed=3, checksums=whole_transform)
    _add_score(twin)
    twin.build()
    populate(twin, cols[:3], *synth_particles(n, 3, 2, 40, 0.2))
    score = np.arange(n, dtype=np.uint32)
    for w in (eng, twin, orc):
        w.write_component(cols[3], 0, score)
        for r in range(0, n, 7):
            w.remove_component(cols[3], r)
    sess = SyncTestSession(2, 6, 9, input_delay=2)
    for t in range(24):
        sess.add_local_input(0, SPAWN if t % 5 in (1, 2) else 0)
        sess.add_local_input(1, 0)
        reqs = sess.advance_frame()
        l0 = eng.launch_count()
        got = eng.handle_requests(sess.info(), reqs)
        assert eng.launch_count() - l0 == 1 and eng.last_kernel().kind == kind_of(generic_kernel)
        assert got == twin.handle_requests(sess.info(), reqs) == orc.handle_requests(sess.info(), reqs)
        assert twin.last_kernel().kind.startswith("stepwise")
        for q in reqs:
            if q.kind == SAVE:
                sess.save_cell(q.frame, 0)
    rows = eng.row_count()
    assert rows == twin.row_count() == orc.row_count() > n
    assert eng.snapshot_frames() == twin.snapshot_frames()
    for f in eng.snapshot_frames():
        alive = twin.peek(f, cols[0], 0, rows)[1].astype(bool)
        for c in cols:
            pe, pt = eng.peek(f, c, 0, rows), twin.peek(f, c, 0, rows)
            assert np.array_equal(pe[1], pt[1]), (f, c)
            assert np.array_equal(pe[0][alive], pt[0][alive]), (f, c)
        born = eng.peek(f, cols[3], n, rows - n)  # spawned rows carry the Score column (zero at birth, +1 per frame since)
        assert np.array_equal(born[1].astype(bool), alive[n:])
    # live image: the oracle on the columns every row has (compare_state reads alive, not presence), the twin on all
    assert compare_state(eng, orc, cols[:3], rows) and peeks_equal(eng, orc, cols)
    assert live_equal(eng, twin, cols, rows)


def live_equal(a, b, cols, rows):
    """Two engines' live images: the alive bytes, and every column on the rows that exist."""
    alive = a.read_alive(0, rows).astype(bool)
    if not np.array_equal(alive, b.read_alive(0, rows).astype(bool)):
        return False
    return all(np.array_equal(a.read_component(c, 0, rows)[alive], b.read_component(c, 0, rows)[alive]) for c in cols)


# ---- 4. a growable engine spawning past its capacity inside vectors, with vectors in flight ----
@pytest.mark.timeout(240)
@pytest.mark.parametrize("tiledep", ["0", "1"])
def test_growable_engine_with_queued_submits_matches_synchronous_calls(monkeypatch, generic_kernel, tiledep):
    monkeypatch.setenv("BGR_TUNE_JIT_TILEDEP", tiledep)
    n, rate = 900, 150

    def make():
        e = Engine(max_entities=1024, max_depth=9, flags=capi.BGR_CFG_GROWABLE)
        c = register_particles(e, spawn_rate=rate, spawn_ttl=40, rng_seed=9, checksums=whole_transform)
        e.build()
        populate(e, c, *synth_particles(n, 9, 20, 80, 0.2))
        return e, c
    (q, cols), (s, _) = make(), make()
    vectors = []
    sess = SyncTestSession(2, 4, 8, input_delay=2)
    for t in range(30):
        sess.add_local_input(0, SPAWN if t % 5 in (1, 2) else 0)
        sess.add_local_input(1, 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        vectors.append((sess.info(), reqs))
    got, want, inflight = [], [], 0
    for info, reqs in vectors:
        q.submit_requests(info, reqs)
        inflight += 1
        if inflight == 4:
            got += q.collect()
            inflight -= 1
        want += s.handle_requests(info, reqs)
        assert s.last_kernel().kind == kind_of(generic_kernel)
    while inflight:
        got += q.collect()
        inflight -= 1
    assert got == want and len(got) >= 30
    rows = q.row_count()
    assert rows == s.row_count() and q.capacity()[0] >= rows > 1024
    assert q.snapshot_frames() == s.snapshot_frames()
    assert live_equal(q, s, cols, rows)
    for f in q.snapshot_frames():
        for c in cols:
            pq, ps = q.peek(f, c, 0, rows), s.peek(f, c, 0, rows)
            m = ps[1].astype(bool)
            assert np.array_equal(pq[1], ps[1]) and np.array_equal(pq[0][m], ps[0][m])


# ---- 5. world batches of spawning worlds ----
@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


def spawn_world(n, depth, stream=None, seed=0, rate=25, ttl=12, flags=0, cap=None):
    """The particles columns with a whole-Transform checksum; spawn rate, ttl and seed per world."""
    w = Engine(max_entities=cap or n + rate * 48, max_depth=depth, flags=flags, stream=stream)
    c = register_particles(w, spawn_rate=rate, spawn_ttl=ttl, rng_seed=0xC0FFEE + seed, checksums=whole_transform)
    w.build()
    populate(w, c, *synth_particles(n, seed, 2, 30, 0.2))
    return w


class SyncDriver:
    def __init__(self, d, depth):
        self.sess, self.depth = SyncTestSession(2, d, depth, input_delay=2), depth

    def next(self, tick):
        self.sess.add_local_input(0, SPAWN if tick % 5 in (1, 2) else 0)
        self.sess.add_local_input(1, 0)
        return self.sess.info(), self.sess.advance_frame()

    def saved(self, checksums):
        for f, cs in checksums:
            self.sess.save_cell(f, cs)


class P2PDriver(SyncDriver):
    def __init__(self, mp, seed):
        self.sess, self.depth = P2PTraceSession(2, max_prediction=mp, input_delay=2, seed=seed, p_clean=0.3), mp + 1

    def next(self, tick):
        self.sess.add_local_input(0, SPAWN if tick % 5 in (1, 3) else 0)
        return self.sess.info(), self.sess.advance_frame()


def image(e):
    """Counters, ring, every stored frame's peek (rows that exist in it), the live image."""
    n = e.row_count()
    alive = e.read_alive(0, n).astype(bool)
    out = [e.rollback_frame_count(), e.confirmed_frame_count(), e.snapshot_frames(), n, e.active_count(), alive.tobytes()]
    for c in range(len(e.elem_bytes)):
        out.append(e.read_component(c, 0, n)[alive].tobytes())
        for f in e.snapshot_frames():
            p = e.peek(f, c, 0, n)
            m = p[1].astype(bool)
            out.append((f, p[0][m].tobytes(), p[1].tobytes()))
    return out


class Fleet:
    """Spawning members on one stream and their twins; rows, seeds, ttls, rates and sessions differ per world."""

    def __init__(self, stream, n_worlds, rows=(300, 600, 2000, 40)):
        self.drivers = [SyncDriver(1 + (3 * i) % 8, 9) if i % 2 == 0 else P2PDriver(3 + i % 5, 0xB200 + i) for i in range(n_worlds)]
        self.members, self.twins = [], []
        for i, d in enumerate(self.drivers):
            kw = dict(seed=i, rate=20 + 7 * (i % 3), ttl=6 + 5 * (i % 4), flags=capi.BGR_CFG_GROWABLE if i % 3 == 2 else 0)
            self.members.append(spawn_world(rows[i % len(rows)], d.depth, stream=stream, **kw))
            self.twins.append(spawn_world(rows[i % len(rows)], d.depth, **kw))
        self.batch = EngineBatch(self.members)
        self.tick_no = [0] * n_worlds

    def draw(self, worlds):
        calls = []
        for w in worlds:
            info, reqs = self.drivers[w].next(self.tick_no[w])
            self.tick_no[w] += 1
            calls.append((w, info, reqs))
        return calls

    def run(self, calls):
        res = self.batch.handle_requests(calls)
        for (w, info, reqs), (status, cs) in zip(calls, res):
            assert status == capi.BGR_OK
            assert cs == self.twins[w].handle_requests(info, reqs), f"world {w} tick {self.tick_no[w]}"
            self.drivers[w].saved(cs)
            lk = self.members[w].last_kernel()
            assert lk.batched == self.batch.specialised()
            if lk.batched:
                assert lk.kind == "generic_nvrtc"
        return res


def assert_fleet_equal(fl, worlds=None):
    for w in worlds if worlds is not None else range(len(fl.members)):
        assert image(fl.members[w]) == image(fl.twins[w]), f"world {w}"


def test_batched_spawning_worlds_match_their_twins(generic_kernel, stream):
    fl = Fleet(stream, 8)
    assert fl.batch.specialised() == (generic_kernel != "interpreter")
    for t in range(36):
        l0 = [m.launch_count() for m in fl.members]
        fl.run(fl.draw(range(8)))
        assert all(m.launch_count() - a == 1 for m, a in zip(fl.members, l0))
        if t % 12 == 11:
            assert_fleet_equal(fl)
    grown = [m for i, m in enumerate(fl.members) if i % 3 == 2]
    assert all(m.row_count() > 0 for m in fl.members)
    assert grown and all(m.capacity()[0] >= m.row_count() for m in grown)
    assert_fleet_equal(fl)


def test_over_capacity_member_refuses_the_whole_call(generic_kernel, stream):
    fl = Fleet(stream, 4, rows=(300, 600, 100))
    small = Engine(max_entities=320, max_depth=9, stream=stream)   # 300 rows, room for no spawn of 25
    c = register_particles(small, spawn_rate=25, spawn_ttl=5, rng_seed=1, checksums=whole_transform)
    small.build()
    populate(small, c, *synth_particles(300, 1, 2, 30))
    fl.batch.close()
    fl.batch = EngineBatch(fl.members + [small])
    for _ in range(6):
        fl.run(fl.draw(range(4)))
    calls = fl.draw(range(4))
    before = [image(m) for m in fl.members + [small]]   # reads launch kernels of their own
    launches = [m.launch_count() for m in fl.members + [small]]
    bad = (4, (capi.BGR_SESSION_NONE, 0, 0, 0), [Request(ADVANCE, 0, [SPAWN, 0])])
    with pytest.raises(BgrError) as ei:
        fl.batch.handle_requests(calls + [bad])
    assert ei.value.status == capi.BGR_ERR_CAPACITY and str(ei.value).startswith("world 4: ")
    assert [m.launch_count() for m in fl.members + [small]] == launches
    assert [image(m) for m in fl.members + [small]] == before
    fl.run(calls)                                    # the same vectors without the refused world
    for _ in range(8):
        fl.run(fl.draw(range(4)))
    assert_fleet_equal(fl)


def test_growable_member_grows_inside_a_batched_call(generic_kernel, stream):
    a = spawn_world(500, 9, stream=stream, seed=1, rate=200, flags=capi.BGR_CFG_GROWABLE, cap=512)
    b = spawn_world(300, 9, stream=stream, seed=2, rate=30)
    ta = spawn_world(500, 9, seed=1, rate=200, flags=capi.BGR_CFG_GROWABLE, cap=512)
    tb = spawn_world(300, 9, seed=2, rate=30)
    batch = EngineBatch([a, b])
    da, db = SyncDriver(3, 9), P2PDriver(4, 7)
    cap0 = a.capacity()[0]
    for t in range(12):
        (ia, ra), (ib, rb) = da.next(t), db.next(t)
        res = batch.handle_requests([(0, ia, ra), (1, ib, rb)])
        assert res[0][1] == ta.handle_requests(ia, ra) and res[1][1] == tb.handle_requests(ib, rb)
        da.saved(res[0][1])
        db.saved(res[1][1])
        assert a.last_kernel().batched == batch.specialised()
    assert a.row_count() > cap0 and a.capacity()[0] > cap0
    assert image(a) == image(ta) and image(b) == image(tb)
