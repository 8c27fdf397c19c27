"""-m gpu: the deferred live image (BGR_TUNE_DEFER_LIVE, engine.cu DeferredLive).

A fused program that ends in `Save(f), Advance` does not write image 0; the next program starts from f's slot, or with
its own Load, and every entry point that touches image 0 rebuilds it first.  Each case runs the same calls on an engine
that defers, on an engine created with BGR_TUNE_DEFER_LIVE=0 (every program writes image 0 itself, as before) and, for
request vectors, on the oracle.  The two engines must agree byte for byte on every row below the row count, dead rows
included, and on every snapshot; checksums must equal the oracle's.  Knobs fall back quietly, so each case also asserts
through Engine.last_kernel() that the vectors it targets deferred (or did not) and which kernel ran."""
import dataclasses

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, P2PTraceSession, Request, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
MULTI_WAVE = 250_000   # 489 tiles: several waves of the one-launch kernels on 132 SMs


def _particles(w, n, mode, spawn_rate=0):
    """The particles bundle: MODE 0 (one column without the finite assertion), 1 (the example's registration) or 2
    (Velocity and Ttl optional).  Ttl 4..60: entities die inside the runs."""
    if mode == 2:
        t = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
        v = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY | OPT)
        l = w.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY | OPT)
        w.checksum_component(v, 0, 12, FIN)
        w.checksum_component(t, 0, 12, FIN)
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        w.build()
        cols = (t, v, l)
    else:
        ck = None if mode == 1 else (lambda w_, t_, v_: (w_.checksum_component(v_, 0, 12, 0), w_.checksum_component(t_, 0, 12, FIN)))
        cols = register_particles(w, spawn_rate=spawn_rate, checksums=ck)
        w.build()
    populate(w, cols, *synth_particles(n, 17, 4, 60, z_fraction=0.2))
    if mode == 2:
        for r in range(0, n, 13):
            w.remove_component(cols[1 + (r // 13) % 2], r)
    return cols


def _scores(w, n):
    """A world the bundle does not cover: Score (optional, +1 per frame), Health (optional, saturating, despawns at 0),
    Tag (checksummed, untouched)."""
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = w.rollback_component("Tag", 12, capi.BGR_STRATEGY_COPY)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        w.checksum_component(c, 0, ln)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(5)
    w.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    w.write_component(health, 0, rng.integers(3, 40, n, dtype=np.uint32))
    w.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in range(0, n, 17):
        w.remove_component(score, r)
    return (score, health, tag)


# variant -> (environment, builder, kernel kind)
VARIANTS = {
    "bundle_mode0": ({}, lambda w, n, **k: _particles(w, n, 0, **k), "bundle"),
    "bundle_mode1": ({}, lambda w, n, **k: _particles(w, n, 1, **k), "bundle"),
    "bundle_mode2": ({}, lambda w, n, **k: _particles(w, n, 2, **k), "bundle"),
    "interpreter": ({"BGR_TUNE_JIT": "0"}, _scores, "generic_interpreter"),
    "nvrtc_tile": ({"BGR_TUNE_JIT": "2", "BGR_TUNE_JIT_ITEM": "512"}, _scores, "generic_nvrtc"),
    "nvrtc_quarter": ({"BGR_TUNE_JIT": "2"}, _scores, "generic_nvrtc"),
}
ALL = list(VARIANTS)
SOME = ["bundle_mode1", "bundle_mode2", "interpreter", "nvrtc_quarter"]


class Worlds:
    """The deferring engine `d`, the eager engine `e` and (optionally) the oracle, built identically."""

    def __init__(self, monkeypatch, variant, n, depth=8, flags=0, oracle=True, extra_rows=0, **kw):
        env, build, self.kind = VARIANTS[variant]
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        self.engines = []
        for defer in ("1", "0"):
            monkeypatch.setenv("BGR_TUNE_DEFER_LIVE", defer)
            eng = Engine(max_entities=n + extra_rows, max_depth=depth, flags=flags)
            self.cols = build(eng, n, **kw)
            self.engines.append(eng)
        monkeypatch.delenv("BGR_TUNE_DEFER_LIVE")
        self.orc = None
        if oracle:
            self.orc = OracleWorld()
            build(self.orc, n, **kw)
        self.d, self.e = self.engines

    def all(self):
        return self.engines + ([self.orc] if self.orc else [])

    def call(self, name, *args):
        """The same entry point on both engines; returns the deferring engine's result after checking they agree."""
        a, b = [getattr(w, name)(*args) for w in self.engines]
        assert np.array_equal(np.asarray(a), np.asarray(b)), name
        return a

    def tick(self, info, reqs):
        """One request vector everywhere; returns (deferring engine's last_kernel, its launches for the vector)."""
        l0 = self.d.launch_count()
        out = [w.handle_requests(info, reqs) for w in self.all()]
        launches = self.d.launch_count() - l0
        assert all(o == out[0] for o in out), reqs
        k = self.d.last_kernel()
        assert k.kind == self.kind and self.d.last_path_fused()
        assert not self.e.last_kernel().deferred_live and not self.e.last_kernel().from_deferred
        return k, launches

    def check(self):
        n = self.d.row_count()
        assert self.e.row_count() == n
        frames = self.d.snapshot_frames()
        assert frames == self.e.snapshot_frames()
        alive = self.call("read_alive", 0, n)
        self.call("active_count")
        for c in self.cols:
            raw = self.call("read_component", c, 0, n)           # every row below the row count, dead ones too
            for f in frames:
                (vd, hd), (ve, he) = self.d.peek(f, c, 0, n), self.e.peek(f, c, 0, n)
                assert np.array_equal(vd, ve) and np.array_equal(hd, he), (f, c)
            if self.orc is not None:
                vo, ho = self.orc.read_component_alive(c, 0, n)
                m = ho.astype(bool)
                assert np.array_equal(raw[m], np.asarray(vo).reshape(raw.shape)[m]), c
        if self.orc is not None:
            assert frames == self.orc.snapshot_frames()
            assert np.array_equal(alive.astype(bool), self.orc.read_alive(0, n).astype(bool))

    def close(self):
        for w in self.all():
            w.close()


def _synctest(d, ticks, maxp=8, inputs=lambda t, h: 0):
    sess = SyncTestSession(2, d, maxp, input_delay=2)
    out = []
    for t in range(ticks):
        for h in range(2):
            sess.add_local_input(h, inputs(t, h))
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        out.append((sess.info(), reqs))
    return out


def _p2p(ticks, maxp=8, seed=0xB200):
    sess = P2PTraceSession(2, maxp, 2, seed=seed)
    out = []
    for t in range(ticks):
        for h in range(2):
            sess.add_local_input(h, (1 << 5) if (t + h) % 3 == 0 else 0)
        reqs = sess.advance_frame()
        out.append((sess.info(), reqs, sess.last_rollback_depth))
    return out


@pytest.mark.parametrize("n", [300, 4097, MULTI_WAVE])
@pytest.mark.parametrize("variant", ALL)
def test_synctest_defers_every_tick_and_matches(monkeypatch, variant, n):
    """SyncTest d=4: every tick after the first ends in Save, Advance and defers; the ticks before the first rollback
    read the live image and start from the deferred base slot instead.  One launch per tick."""
    w = Worlds(monkeypatch, variant, n)
    prev = False
    for t, (info, reqs) in enumerate(_synctest(4, 12)):
        k, launches = w.tick(info, reqs)
        assert launches == 1
        # tick 0 follows the host's writes of the initial population: eager
        assert k.deferred_live == (t > 0)
        assert k.from_deferred == (prev and reqs[0].kind != LOAD)
        prev = k.deferred_live
    if n == 300 and variant.startswith("nvrtc"):
        assert w.d.last_kernel().item_rows == (512 if variant == "nvrtc_tile" else 128)
    w.check()
    w.close()


@pytest.mark.parametrize("variant", ALL)
def test_p2p_trace_reads_the_base_slot_on_clean_ticks(monkeypatch, variant):
    """The C4 P2P trace: clean ticks [Save, Advance] start from the previous tick's base slot, rollbacks of every depth
    start with their own Load; every tick defers.  Checked midway (reads go eager for one tick) and at the end."""
    w = Worlds(monkeypatch, variant, 4097)
    trace = _p2p(120)
    assert {depth for _, _, depth in trace} == set(range(9))
    prev = False
    for t, (info, reqs, depth) in enumerate(trace):
        k, launches = w.tick(info, reqs)
        assert launches == 1
        assert k.deferred_live == (t not in (0, 61))   # the first tick after the host wrote / read the live world is eager
        assert k.from_deferred == (depth == 0 and prev)
        prev = k.deferred_live
        if t == 60:
            w.check()
    w.check()
    w.close()


ENTRY_POINTS = ["read", "write", "alive", "has", "active", "remove_insert", "spawn", "despawn", "download", "startup",
                "reset", "set_depth", "confirm", "stepwise"]


@pytest.mark.parametrize("entry", ENTRY_POINTS)
@pytest.mark.parametrize("variant", SOME)
def test_entry_points_after_a_deferred_tick(monkeypatch, variant, entry):
    """Each entry point that touches image 0 (or the ring outside a program), called right after a tick that deferred,
    then more ticks: both engines stay byte-identical."""
    optional = variant != "bundle_mode1"
    if entry in ("has", "remove_insert") and not optional:
        pytest.skip("needs an optional column")
    if entry == "startup" and variant != "bundle_mode1":
        pytest.skip("needs spawn_particles")
    kw = {"spawn_rate": 8} if variant == "bundle_mode1" else {}
    n = 1300
    w = Worlds(monkeypatch, variant, n, oracle=False, extra_rows=64, **kw)
    vectors = _synctest(3, 12)
    for info, reqs in vectors[:6]:
        w.tick(info, reqs)
    assert w.d.last_kernel().deferred_live
    c0, c1, c2 = w.cols
    l0, le0 = w.d.launch_count(), w.e.launch_count()
    if entry == "read":
        w.call("read_component", c0, 0, n)
    elif entry == "write":
        vals = w.call("read_component", c2, 5, 7)
        w.call("write_component", c2, 700, vals)
    elif entry == "alive":
        w.call("read_alive", 0, n)
    elif entry == "has":
        w.call("has_component", c1, 0, n)
    elif entry == "active":
        w.call("active_count")
    elif entry == "remove_insert":
        value = w.call("read_component", c1, 20, 1)[0]
        w.call("remove_component", c1, 7)
        w.call("insert_component", c1, 9, value)
    elif entry == "spawn":
        w.call("spawn", 5)
    elif entry == "despawn":
        w.call("despawn", 3)
    elif entry == "download":
        ln = 12 if w.kind == "bundle" else 4   # Transform.translation / Score
        bufs = [eng.host_alloc(n, ln) for eng in w.engines]
        for eng, b in zip(w.engines, bufs):
            eng.download_wait(eng.download_begin(c0, 0, ln, 0, n, b))
        assert np.array_equal(bufs[0], bufs[1])
    elif entry == "startup":
        w.call("run_startup_system", capi.BGR_SYS_PARTICLES_SPAWN)
    elif entry == "reset":
        frame = w.d.rollback_frame_count()
        w.call("reset_session")
        w.call("set_rollback_frame_count", frame)   # the same session goes on (Time<GgrsTime> only moves forward)
    elif entry == "set_depth":
        w.call("set_depth", 8)
    elif entry == "confirm":
        w.call("confirm", w.d.rollback_frame_count() - 3)   # keeps the frame the next SyncTest Load needs
    elif entry == "stepwise":
        w.call("save_world")
        k = w.d.last_kernel()
        assert k.from_deferred and k.deferred_live
        w.call("load_world")
        assert not w.d.last_kernel().deferred_live
        w.call("advance_world", [0, 0])
    # one extra launch wrote image 0; bgr_save_world instead started from the base slot inside its own launch
    assert (w.d.launch_count() - l0) - (w.e.launch_count() - le0) == (0 if entry == "stepwise" else 1)
    for info, reqs in vectors[6:]:
        k, launches = w.tick(info, reqs)
        assert launches == 1
    assert w.d.last_kernel().deferred_live
    w.check()
    w.close()


@pytest.mark.parametrize("session", ["synctest", "p2p"])
@pytest.mark.parametrize("variant", SOME)
def test_pipelined_submits_four_in_flight(monkeypatch, variant, session):
    """bgr_submit_requests with four vectors in flight: consecutive launches overlap through per-tile dependencies
    (BGR_TUNE_JIT_TILEDEP=1 for the generated kernel), and a program that starts from a base slot depends on the
    previous launch's tiles exactly as one that reads the live image."""
    monkeypatch.setenv("BGR_TUNE_JIT_TILEDEP", "1")
    w = Worlds(monkeypatch, variant, 120_000)
    vectors = _synctest(3, 24) if session == "synctest" else [(i, r) for i, r, _ in _p2p(40)]
    got, want = {0: [], 1: []}, []
    for k, eng in enumerate(w.engines):
        inflight = 0
        for info, reqs in vectors:
            eng.submit_requests(info, reqs)
            inflight += 1
            if inflight == 4:
                got[k] += eng.collect()
                inflight -= 1
        while inflight:
            got[k] += eng.collect()
            inflight -= 1
    for info, reqs in vectors:
        want += w.orc.handle_requests(info, reqs)
    assert got[0] == got[1] == want and len(want) >= len(vectors)
    assert w.d.last_kernel().deferred_live
    w.check()
    w.close()


@pytest.mark.parametrize("variant", ["bundle_mode1", "interpreter"])
def test_depth_one_ring_writes_the_live_image_before_reusing_the_base_slot(monkeypatch, variant):
    """max_prediction 1: every Save evicts the previous frame and reuses its slot, which is the deferred image's base.
    The live image is written first (a second launch), then the vector runs and defers again."""
    w = Worlds(monkeypatch, variant, 4097, depth=1)
    for f in range(8):
        k, launches = w.tick((capi.BGR_SESSION_P2P, 1, 0, f - 1), [Request(SAVE, f), Request(ADVANCE, 0, [0, 0])])
        assert k.deferred_live == (f > 0) and not k.from_deferred
        assert launches == (1 if f < 2 else 2)
    w.check()
    w.close()


def test_spawn_after_the_last_save_stays_eager(monkeypatch):
    """An Advance that spawns particles after the last Save: the new rows are not in the base slot, so that vector
    writes the live image itself; the next one defers again."""
    w = Worlds(monkeypatch, "bundle_mode1", 3000, extra_rows=16 * 12, spawn_rate=16)
    spawn = [False, False, True, False, True, True, False, False]
    prev = False
    for f, s in enumerate(spawn):
        k, launches = w.tick((capi.BGR_SESSION_P2P, 8, 0, f - 8),
                             [Request(SAVE, f), Request(ADVANCE, 0, [(1 << 4) if s else 0, 0])])
        assert launches == 1
        assert k.deferred_live == (f > 0 and not s)
        assert k.from_deferred == prev
        prev = k.deferred_live
    assert w.d.row_count() == 3000 + 16 * sum(spawn)
    w.check()
    w.close()


@pytest.mark.parametrize("variant", ["bundle_mode1", "interpreter"])
def test_reading_live_every_tick_goes_eager(monkeypatch, variant):
    """A caller that reads the live world after every tick: one materialisation after the first deferred tick, then
    every vector writes image 0 itself — one launch per tick, nothing rebuilt."""
    w = Worlds(monkeypatch, variant, 4097, oracle=False)
    vectors = _synctest(4, 14)
    for info, reqs in vectors[:2]:
        w.tick(info, reqs)
    assert w.d.last_kernel().deferred_live
    for t, (info, reqs) in enumerate(vectors[2:]):
        l0 = w.d.launch_count()
        w.call("read_alive", 0, 4097)
        assert w.d.launch_count() - l0 == (2 if t == 0 else 1)   # k_gather_alive (+ the materialisation once)
        k, launches = w.tick(info, reqs)
        assert launches == 1 and not k.deferred_live and not k.from_deferred
    w.check()
    w.close()


@pytest.mark.parametrize("session", ["synctest", "p2p"])
@pytest.mark.parametrize("flag", [capi.BGR_CFG_SKIP_UNCHANGED_PLANES, capi.BGR_CFG_DESYNC_CAPTURE])
@pytest.mark.parametrize("variant", SOME)
def test_skip_unchanged_planes_and_desync_capture_engines(monkeypatch, variant, flag, session):
    """The opt-in flags that change which bytes a Save moves (content versions of the passive planes) or which slots
    the ring hands out (first-snapshot witnesses): snapshots, the live world and the desync reports stay identical."""
    w = Worlds(monkeypatch, variant, 4097, flags=flag)
    vectors = _synctest(3, 14) if session == "synctest" else [(i, r) for i, r, _ in _p2p(60)]
    for t, (info, reqs) in enumerate(vectors):
        k, _ = w.tick(info, reqs)
        assert k.deferred_live == (t not in (0, 11))
        if t == 10:
            w.check()
    w.check()
    if flag == capi.BGR_CFG_DESYNC_CAPTURE:
        for f in w.call("desync_frames"):
            a, b = (eng.desync_diff(f) for eng in w.engines)
            assert np.array_equal(a.records, b.records)
            assert dataclasses.replace(a, records=None) == dataclasses.replace(b, records=None)
    w.close()
