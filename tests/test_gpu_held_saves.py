"""-m gpu: held Saves of the bundle kernel (content ids, engine.cu HostState).

A Save whose target slot already holds the content the registers have (same derivation, same row count) stores nothing
and only checksums.  Each case runs the same calls on the default engine, on an engine with BGR_TUNE_HELD_SAVES=0
(every Save stores), on one with BGR_TUNE_HELD_SAVES=2 (a held Save compares its target with the registers and counts the
words that differ), on the whole-image engine (BGR_TUNE_BUNDLE=0) and on the oracle.  Checksums are equal on every tick;
the live world and every queued frame hold the same columns and alive bytes; the verifying engine counts no mismatch.

Worlds with other systems (box_game's move_cube_system, the call-count test system) do not run the bundle kernel
(engine.cu detect_bundles): their Saves are never held, so they have no case here.  The friction factor and the call
count are still part of the advance key (tests/cpp/test_content_ids.cpp)."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import EDIT_DTYPE, Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, P2PTraceSession, Request, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld
from test_gpu_stable_planes import _build

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
SPAWN, NOOP = 1 << 4, 1 << 5
SEG_ROWS, TILE_ROWS = 64, 512


class Worlds:
    """Default `g`, never-held `h`, verifying `v`, whole-image `s` and the oracle `o` (None where a case cannot
    restate its calls on it), built identically."""

    def __init__(self, monkeypatch, n, spawn_rate=0, optional=False, flags=0, retain=None, extra_rows=0, nan=False,
                 multi_wave=True, oracle=True, env=()):
        def engine(**tune):
            with monkeypatch.context() as m:
                for k, v in dict(env).items():
                    m.setenv(k, v)
                if multi_wave:
                    m.setenv("BGR_TUNE_PASSIVE_EARLY", "0")
                for k, v in tune.items():
                    m.setenv(k, v)
                return Engine(max_entities=n + extra_rows, max_depth=9, flags=flags)

        self.g = engine()
        self.h = engine(BGR_TUNE_HELD_SAVES="0")
        self.v = engine(BGR_TUNE_HELD_SAVES="2")
        self.s = engine(BGR_TUNE_BUNDLE="0")
        self.o = OracleWorld() if oracle else None
        for w in self.all():
            self.cols = _build(w, n, spawn_rate, optional, retain if w is not self.o else None, True, nan)

    def engines(self):
        return (self.g, self.h, self.v, self.s)

    def all(self):
        return self.engines() + ((self.o,) if self.o is not None else ())

    def tick(self, info, reqs):
        out = [w.handle_requests(info, reqs) for w in self.all()]
        assert all(x == out[0] for x in out), reqs
        kg, kh, kv = self.g.last_kernel(), self.h.last_kernel(), self.v.last_kernel()
        assert kg.kind == kh.kind == kv.kind == "bundle" and self.s.last_kernel().kind != "bundle"
        assert not kh.held_saves and kg.held_saves == kv.held_saves
        assert self.g.held_saves()["last"] == self.v.held_saves()["last"]
        return self.g.held_saves()["last"]

    def check(self):
        g = self.g
        n = g.row_count()
        frames = g.snapshot_frames()
        for e in self.all():
            assert e.row_count() == n and e.snapshot_frames() == frames
        ref = self.o if self.o is not None else self.s
        alive = ref.read_alive(0, n).astype(bool)
        for e in self.engines():
            assert np.array_equal(e.read_alive(0, n).astype(bool), alive)
        for c in self.cols:
            want = ref.read_component_alive(c, 0, n) if self.o is not None else (ref.read_component(c, 0, n), ref.has_component(c, 0, n))
            for e in self.engines():
                self._same((e.read_component(c, 0, n), e.has_component(c, 0, n)), want, c)
        for f in frames:
            rows = g.frame_digest(f)[0].rows
            for c in self.cols:
                want = ref.peek(f, c, 0, rows)
                for e in self.engines():
                    self._same(e.peek(f, c, 0, rows), want, c)
            # the held engine's frame digest covers every column and the mask byte of every row below the row count
            hd = g.frame_digest(f)
            for e in (self.h, self.v):
                d = e.frame_digest(f)
                assert d[0].root == hd[0].root and np.array_equal(d[1], hd[1]), f
        assert self.v.held_saves()["mismatched_words"] == 0

    @staticmethod
    def _same(got, want, c):
        (vg, hg), (vo, ho) = got, want
        m = np.asarray(ho).astype(bool)
        assert np.array_equal(np.asarray(hg).astype(bool), m), c
        assert np.array_equal(vg[m], np.asarray(vo)[m]), c

    def held_total(self):
        assert self.h.held_saves()["total"] == 0
        return self.g.held_saves()["total"]

    def close(self):
        for w in self.all():
            w.close()


def _vectors(session, ticks, spawn=False, seed=0xB200, d=8, inputs=None):
    sess = SyncTestSession(2, d, 9, input_delay=2) if session == "synctest" else P2PTraceSession(2, 8, 2, seed=seed)
    out = []
    for t in range(ticks):
        a, b = inputs(t) if inputs else (SPAWN if spawn and t % 7 in (2, 3) else 0, NOOP if t % 3 == 0 else 0)
        sess.add_local_input(0, a)
        sess.add_local_input(1, b)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        out.append((sess.info(), reqs))
    return out


@pytest.mark.parametrize("d", range(1, 9))
def test_synctest_every_check_distance(monkeypatch, d):
    """SyncTest at d: once the ring is full every tick re-saves d - 1 frames it already holds and holds them."""
    w = Worlds(monkeypatch, 70_001)
    held = [w.tick(info, reqs) for info, reqs in _vectors("synctest", 24, d=d)]
    assert held[-8:] == [d - 1] * 8
    w.check()
    w.close()


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_bundle_modes(monkeypatch, mode):
    """MODE 0 (checksums without the finite assertion, NaN payloads), 1 (the stress registration) and 2 (per-entity
    presence), SyncTest d=8 over ttl values that reach 0 inside the window.  The GPU's f32 arithmetic does not keep NaN
    payloads as the CPU oracle does, so MODE 0 holds the engines to each other."""
    w = Worlds(monkeypatch, 9_001, optional=mode == 2, nan=mode == 0, oracle=mode != 0)
    held = []
    for t, (info, reqs) in enumerate(_vectors("synctest", 30)):
        held.append(w.tick(info, reqs))
        if t == 15:
            w.check()
    assert held[-5:] == [7] * 5
    w.check()
    w.close()


def test_p2p_corrected_inputs_store_again(monkeypatch):
    """Every third rollback of the P2P trace gets corrected inputs on all its Advances, as GGRS gives them when a remote
    input arrives: a new key, so a new id, and every re-save of that vector stores.  (The trace's other rollbacks keep
    their inputs, but its confirmed frame moves every tick: the confirmation frees an older slot after the Load has
    freed the re-saved frame's, and the ring hands that one out first, so those re-saves land in another slot.)"""
    w = Worlds(monkeypatch, 20_011)
    corrected = 0
    for t, (info, reqs) in enumerate(_vectors("p2p", 60)):
        fix = reqs[0].kind == LOAD and t % 3 == 0
        if fix:
            reqs = [Request(ADVANCE, 0, [r.inputs[0], r.inputs[1] ^ 1], r.status) if r.kind == ADVANCE else r for r in reqs]
        held = w.tick(info, reqs)
        if fix:
            corrected += 1
            assert held == 0, reqs
        if t == 30:
            w.check()
    assert corrected >= 3
    w.held_total()
    w.check()
    w.close()


class _Depth:
    """Stands in for the P2P trace's generator for one tick: a rollback of `depth` frames."""

    def __init__(self, depth):
        self.depth = depth

    def next_f64(self):
        return 0.0

    def next_u64(self):
        return self.depth - 1


def test_p2p_host_write_before_the_rollback_frame_stores(monkeypatch):
    """Clean P2P ticks, then a rollback of two frames with unchanged inputs: its re-save holds.  Then a host write of
    the live world, two clean ticks that save the written world, and a rollback to a frame from before the write: the
    re-simulated frames differ from what their slots hold, and none of its Saves is held.  The confirmed frame stays
    put, so the ring gives each re-save the slot its frame had (a confirmation between the Load and the re-save would
    free an older slot and hand that out first)."""
    w = Worlds(monkeypatch, 20_011)
    sess = P2PTraceSession(2, 8, 2, seed=5, p_clean=1.0)

    def tick(depth=0):
        sess.add_local_input(0, 0)
        sess.add_local_input(1, 0)
        if depth:
            rng, sess._rng, sess._p_clean = sess._rng, _Depth(depth), 0.0
        reqs = sess.advance_frame()
        if depth:
            sess._rng, sess._p_clean = rng, 1.0
            assert reqs[0].kind == LOAD
        return w.tick((sess.info()[0], 8, 0, -1), reqs)

    assert [tick() for _ in range(16)] == [0] * 16
    assert tick(2) == 1
    assert [tick() for _ in range(3)] == [0] * 3
    vals = w.g.read_component(w.cols[1], 0, 500).view(np.float32).copy()
    vals[:, 0] += np.float32(0.5)
    for x in w.all():
        x.write_component(w.cols[1], 0, vals)
    assert [tick() for _ in range(2)] == [0] * 2
    assert tick(3) == 0
    w.check()
    w.close()


@pytest.mark.parametrize("session", ["synctest", "p2p"])
def test_host_writers_between_ticks(monkeypatch, session):
    """A host write, a despawn, a spawn, the startup system and an edit batch between ticks.  Each gives the live image
    a fresh id: P2P ticks save the written world, and rollbacks to frames from before a write re-simulate content the
    later slots do not hold.  A SyncTest tick starts with Load(f-d), which rolls the write back: it still holds."""
    n, rate = 9_001, 16
    w = Worlds(monkeypatch, n, spawn_rate=rate, extra_rows=4096)
    t_col, v_col, _ = w.cols
    rng = np.random.default_rng(3)
    held = []
    for t, (info, reqs) in enumerate(_vectors(session, 48)):
        if t == 12:
            vals = w.g.read_component(t_col, 100, 3000).view(np.float32).copy()
            vals[:, 0] = rng.uniform(-9.0, 9.0, 3000)
            for x in w.all():
                x.write_component(t_col, 100, vals)
        if t == 18:
            for r in (0, 63, 64, 4097, n - 1):
                for x in w.all():
                    x.despawn(r)
        if t == 24:
            for x in w.all():
                x.spawn(37)
        if t == 30:
            for x in w.all():
                x.run_startup_system(capi.BGR_SYS_PARTICLES_SPAWN)
        if t == 36:   # one edit batch on the engines, the same records as single calls on the oracle
            row = 777
            val = np.array([1.25, -3.5, 0.0], np.float32)
            recs = np.array([(capi.BGR_EDIT_WRITE, t_col, row, 1, 0, 12, 0, 0), (capi.BGR_EDIT_DESPAWN, 0, 901, 1, 0, 0, 0, 0)],
                            EDIT_DTYPE)
            for x in w.engines():
                x.apply_edits(recs, val.tobytes())
            cur = w.o.read_component(t_col, row, 1).view(np.float32).copy()
            cur[0, :3] = val
            w.o.write_component(t_col, row, cur)
            w.o.despawn(901)
        held.append(w.tick(info, reqs))
        if t in (13, 19, 25, 31, 37):
            w.check()
    if session == "synctest":
        assert held[-8:] == [7] * 8
    w.check()
    w.close()


def test_checkpoint_restore_between_ticks(monkeypatch):
    """Every engine restores the same checkpoint mid-run (image 0 and the one slot the ring then queues get one fresh
    id).  Clean P2P ticks refill the ring from its frame, holding nothing; SyncTest ticks from there hold again."""
    w = Worlds(monkeypatch, 30_001, oracle=False)
    for info, reqs in _vectors("synctest", 20):
        w.tick(info, reqs)
    blob = w.g.checkpoint(w.g.snapshot_frames()[-1])
    assert blob is not None
    for e in w.engines():
        e.restore(blob)
    w.check()
    p2p = P2PTraceSession(2, 8, 2, seed=0xC4, p_clean=1.0)   # the ring holds the checkpoint's frame alone
    p2p.current_frame = w.g.rollback_frame_count()
    clean = []
    for _ in range(10):
        p2p.add_local_input(0, 0)
        p2p.add_local_input(1, 0)
        clean.append(w.tick(p2p.info(), p2p.advance_frame()))
    assert clean == [1] + [0] * 9   # the first re-saves the restored frame into its own slot, which holds it
    sess = SyncTestSession(2, 8, 9, input_delay=2)
    sess.current_frame = p2p.current_frame
    held = []
    for _ in range(16):
        sess.add_local_input(0, 0)
        sess.add_local_input(1, 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        held.append(w.tick(sess.info(), reqs))
    assert held[-5:] == [7] * 5
    w.check()
    w.close()


def test_spawning_world_and_the_one_wave_size(monkeypatch):
    """A spawning P2P world around the one-wave size: stamped and unstamped launches, both instances holding Saves."""
    import torch
    edge = 3 * torch.cuda.get_device_properties(0).multi_processor_count * TILE_ROWS
    rate, ticks, n = 512, 40, edge - 700
    w = Worlds(monkeypatch, n, spawn_rate=rate, extra_rows=rate * ticks, multi_wave=False)
    sides = set()
    for t, (info, reqs) in enumerate(_vectors("p2p", ticks, spawn=True)):
        w.tick(info, reqs)
        sides.add(w.g.last_kernel().stable_planes)
        if t in (12, 25):
            w.check()
    assert sides == {True, False}
    w.check()
    w.close()


@pytest.mark.parametrize("kind", ["capture", "retain"])
def test_capture_and_retention(monkeypatch, kind):
    """Desync capture hands witness slots out again and retention keeps confirmed frames: ids stay with slot indices."""
    ticks = 40
    flags, retain = (capi.BGR_CFG_DESYNC_CAPTURE, None) if kind == "capture" else (0, (10, 4))
    w = Worlds(monkeypatch, 5_001, flags=flags, retain=retain)
    held = [w.tick(info, reqs) for info, reqs in _vectors("synctest", ticks)]
    # with capture, a frame's first snapshot stays in its slot as the witness and re-saves take other slots
    assert w.held_total() > 0 and (kind == "capture" or held[-5:] == [7] * 5), held
    w.check()
    if kind == "capture":
        frames = w.g.desync_frames()
        assert frames == w.h.desync_frames() == w.s.desync_frames()
        for f in frames:
            assert w.g.desync_diff(f).summary_tuple() == w.h.desync_diff(f).summary_tuple()
    else:
        frames = w.g.retained_frames()
        assert frames and frames == w.h.retained_frames()
        for f in frames:
            (hg, dg), (hh, dh) = w.g.frame_digest(f), w.h.frame_digest(f)
            assert hg.rows == hh.rows and hg.root == hh.root and np.array_equal(dg, dh)
    w.close()


def test_single_wave_grids_hold(monkeypatch):
    """A one-wave world runs the kernel instance without stamps: it holds the same re-saves."""
    w = Worlds(monkeypatch, 20_011, multi_wave=False)
    held = []
    for info, reqs in _vectors("synctest", 24):
        held.append(w.tick(info, reqs))
        assert not w.g.last_kernel().stable_planes
    assert held[-8:] == [7] * 8
    w.check()
    w.close()


def test_stamp_rollover_stores_everything(monkeypatch):
    """The vector at which the stamp range rolls over forgets every content id: it holds nothing, and later ticks
    hold again."""
    w = Worlds(monkeypatch, 30_001, env={"BGR_TEST_STAMP_FIRST": str(0xFFFFFFFF - 81 - 10 * 20)})
    held = [w.tick(info, reqs) for info, reqs in _vectors("synctest", 40)]
    # a SyncTest tick of d = 8 takes 19 stamps: the range runs out after about ten ticks
    zero_after_full = [i for i in range(12, 40) if held[i] == 0]
    assert zero_after_full and held[-5:] == [7] * 5
    w.check()
    w.close()


def test_four_vectors_in_flight_then_synchronous(monkeypatch):
    n, ticks = 120_001, 40
    w = Worlds(monkeypatch, n)
    vectors = _vectors("synctest", ticks)
    got_by = {}
    for e in (w.g, w.v):
        got, inflight = [], 0
        for info, reqs in vectors[:30]:
            e.submit_requests(info, reqs)
            inflight += 1
            if inflight == 4:
                got += e.collect()
                inflight -= 1
        while inflight:
            got += e.collect()
            inflight -= 1
        got_by[id(e)] = got
    want = [w.o.handle_requests(info, reqs) for info, reqs in vectors[:30]]
    for e in (w.h, w.s):
        assert [e.handle_requests(info, reqs) for info, reqs in vectors[:30]] == want
    flat = [c for out in want for c in out]
    assert got_by[id(w.g)] == flat and got_by[id(w.v)] == flat
    for info, reqs in vectors[30:]:
        w.tick(info, reqs)
    w.check()
    w.close()


def test_steady_state_tick_holds_seven_of_eight(monkeypatch):
    """1M entities, SyncTest d=8 (the headline workload): a steady-state tick holds 7 of its 8 Saves and its launch
    trace counts one Save's stored units."""
    n = 1_000_000
    w = Engine(max_entities=n, max_depth=9)
    cols = register_particles(w)
    w.build()
    populate(w, cols, *synth_particles(n, 5, 100_000, 200_000))
    vectors = _vectors("synctest", 40)
    for info, reqs in vectors[:20]:
        w.handle_requests(info, reqs)
    w.trace_enable(4)
    held, kinds = [], []
    for info, reqs in vectors[20:24]:
        w.handle_requests(info, reqs)
        held.append(w.held_saves()["last"])
        kinds.append(w.last_kernel())
    units = [int(r[3]) for r in w.trace_read(4)]
    w.trace_enable(0)
    assert held == [7] * 4 and all(k.held_saves and k.stable_planes for k in kinds)
    # Save(f) stores the four planes a frame changes, 4 units each per 64-row segment; the live image is deferred
    segs = -(-n // SEG_ROWS)
    # (and the few segments whose alive byte or ttl.hi a frame changes)
    assert all(k.deferred_live for k in kinds) and all(16 * segs <= u < 17 * segs for u in units), units
    # a host write between ticks gives the live image a fresh id, but the next tick's Load(f-8) rolls it back: the
    # re-simulation is the one the slots hold, and it still holds 7
    vals = w.read_component(cols[1], 0, 10).view(np.float32).copy()
    vals[:, 0] += 1.0
    w.write_component(cols[1], 0, vals)
    w.handle_requests(*vectors[24])
    assert w.held_saves()["last"] == 7
    w.close()


@pytest.mark.parametrize("name", ["bundle_mode1_stamped", "bundle_mode1_one_wave", "bundle_mode2_stamped",
                                  "bundle_multi_wave", "bundle_crossing_sides"])
def test_random_interleavings_verify_every_held_save(name):
    """The random interleavings of every entry point (tests/interleave_driver.py) with BGR_TUNE_HELD_SAVES=2 on the
    engine: each held Save compares its target with the registers, and no word differs.  Saves are held, except in
    bundle_crossing_sides, whose vectors spawn on nearly every tick (a spawn gives a fresh id)."""
    from interleave_driver import Config, Interleaving
    from test_gpu_interleavings import FLAG_SETS, configs, new_engine

    cfg0 = {c.name: c for c in configs()}[name]
    held = 0
    for seed, (flags, retain) in enumerate(FLAG_SETS[:5]):
        cfg = Config(**{**cfg0.__dict__, "flags": flags, "retain": retain, "env": {**cfg0.env, "BGR_TUNE_HELD_SAVES": "2"}})
        drv = Interleaving(cfg, seed, new_engine(name))
        try:
            drv.run()
            h = drv.eng.held_saves()
        finally:
            drv.close()
        assert h["mismatched_words"] == 0, f"{name} seed {seed}: {h}"
        held += h["total"]
    assert held > 0 or name == "bundle_crossing_sides", name
