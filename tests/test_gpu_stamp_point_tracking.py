"""-m gpu: the bundle kernel's stamped instances find a stored Save's changed active planes by comparing the registers
once with the content of the last stamp point (a shared-memory snapshot taken at every Load, read of the live image,
stored Save and live write), instead of OR-ing the changes of every Advance in between.

Each case runs the same calls on the default engine (several waves: stamps), on a whole-image engine
(BGR_CFG_FORCE_STEPWISE) and on the oracle, with checksums equal on every tick and state compared with
test_gpu_stable_planes' checks.  The launch trace's stored units are held to a per-Advance model of the same ticks: never
more than storing every plane a stored Save or live write could claim, and in the steady state of a 2-D world with long
ttl exactly what the per-Advance rule stores (translation.x/y, velocity.y and ttl.lo of every segment touched since the
last stamp point)."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld
from test_gpu_stable_planes import SEG_ROWS, TILE_ROWS, Worlds, _build, _vectors

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
STAMP_LIMIT = 0xFFFFFFFF - 81       # run_fused clears the stamp table when the next stamp is past this
ALL_UNITS = 4 * 8 + 1               # eight word planes of a segment (4 units of 64 B each) and its alive plane
STEADY_UNITS = 4 * 4                # translation.x/y, velocity.y, ttl.lo: what every Advance of a 2-D world changes


class Trio(Worlds):
    """Worlds with a chosen ring depth, extra engine settings and the whole-image engine forced to the stepwise path."""

    def __init__(self, monkeypatch, n, depth=9, env=None, spawn_rate=0, optional=False, extra_rows=0, edges=True):
        with monkeypatch.context() as m:
            m.setenv("BGR_TUNE_PASSIVE_EARLY", "0")
            for k, v in (env or {}).items():
                m.setenv(k, v)
            self.g = Engine(max_entities=n + extra_rows, max_depth=depth)
        self.s = Engine(max_entities=n + extra_rows, max_depth=depth, flags=capi.BGR_CFG_FORCE_STEPWISE)
        self.o = OracleWorld(max_depth=depth)
        for w in self.all():
            self.cols = _build(w, n, spawn_rate, optional, None, edges, False)
        self.rng = np.random.default_rng(11)

    def segs(self):
        return -(-self.g.row_count() // TILE_ROWS) * (TILE_ROWS // SEG_ROWS)

    def run(self, vectors, between=None, check_at=()):
        """Ticks with the launch trace on; every tick's stored units within what its stored Saves and live write
        could claim."""
        self.g.trace_enable(len(vectors))
        bounds = []
        for t, (info, reqs) in enumerate(vectors):
            if between:
                between(t)
            k = self.tick(info, reqs)
            stored = sum(r.kind == SAVE for r in reqs) - self.g.held_saves()["last"]
            bounds.append((stored + (0 if k.deferred_live else 1)) * ALL_UNITS * self.segs())
            if t in check_at:
                self.check()
        units = [int(r[3]) for r in self.g.trace_read(len(vectors))]
        self.g.trace_enable(0)
        assert all(u <= b for u, b in zip(units, bounds)), (units, bounds)
        self.check()
        return units


def _synctest(d, ticks):
    sess = SyncTestSession(2, d, d + 1, input_delay=2)
    out = []
    for t in range(ticks):
        sess.add_local_input(0, 0)
        sess.add_local_input(1, (1 << 5) if t % 3 == 0 else 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        out.append((sess.info(), reqs))
    return out


def _per_advance_units(reqs, n_stored, segs):
    """Units the per-Advance rule stores for one vector of a long-ttl 2-D world whose stable planes every slot holds
    already: the last n_stored Saves are the stored ones (the others re-save frames their slots hold), and a stored Save
    stores the four moving planes when an Advance ran since the last stamp point (the Load or the previous stored
    Save).  The live image is deferred."""
    saves = [i for i, r in enumerate(reqs) if r.kind == SAVE]
    stored = set(saves[len(saves) - n_stored:])
    units, moved = 0, False
    for i, r in enumerate(reqs):
        if r.kind == LOAD:
            moved = False
        elif r.kind == ADVANCE:
            moved = True
        elif i in stored:
            units += STEADY_UNITS * segs if moved else 0
            moved = False
    return units


@pytest.mark.parametrize("d", [1, 2, 3, 4, 5, 6, 7, 8, 16])
def test_synctest_depths(monkeypatch, d):
    w = Trio(monkeypatch, 9_001, depth=d + 1)
    w.run(_synctest(d, 2 * d + 14), check_at=(d + 3,))
    w.close()


@pytest.mark.parametrize("d", [1, 4, 8, 16])
def test_steady_state_equals_per_advance_rule(monkeypatch, d):
    """A 2-D world with long ttl, whole tiles: after the ring has filled, every tick stores exactly what the per-Advance
    rule stores, and the checksums equal the whole-image engine's."""
    n = 48 * TILE_ROWS
    segs = n // SEG_ROWS
    monkeypatch.setenv("BGR_TUNE_PASSIVE_EARLY", "0")
    g = Engine(max_entities=n, max_depth=d + 1)
    s = Engine(max_entities=n, max_depth=d + 1, flags=capi.BGR_CFG_FORCE_STEPWISE)
    for w in (g, s):
        cols = register_particles(w)
        w.build()
        populate(w, cols, *synth_particles(n, 5, 100_000, 200_000))
    vectors = _synctest(d, 3 * d + 30)
    warm = 2 * d + 12
    for info, reqs in vectors[:warm]:
        assert g.handle_requests(info, reqs) == s.handle_requests(info, reqs)
    g.trace_enable(len(vectors) - warm)
    model = []
    for info, reqs in vectors[warm:]:
        assert g.handle_requests(info, reqs) == s.handle_requests(info, reqs)
        k = g.last_kernel()
        assert k.kind == "bundle" and k.stable_planes and k.deferred_live
        n_saves = sum(r.kind == SAVE for r in reqs)
        model.append(_per_advance_units(reqs, n_saves - g.held_saves()["last"], segs))
    units = [int(r[3]) for r in g.trace_read(len(vectors) - warm)]
    assert units == model and all(u == STEADY_UNITS * segs for u in units)
    g.close()
    s.close()


def test_p2p_with_corrected_inputs(monkeypatch):
    """The C4 trace: rollbacks re-simulate with corrected inputs, so a vector stores several Saves."""
    w = Trio(monkeypatch, 20_011)
    w.run(_vectors("p2p", 40), check_at=(15,))
    assert w.g.held_saves()["total"] > 0
    w.close()


def test_spawns_inside_the_rollback_window(monkeypatch):
    rate, ticks = 24, 40
    w = Trio(monkeypatch, 6_001, spawn_rate=rate, extra_rows=rate * ticks)
    w.run(_vectors("p2p", ticks, spawn=True), check_at=(20,))
    assert w.g.row_count() > 6_001 + rate
    w.close()


def test_host_writes_between_ticks(monkeypatch):
    n = 9_001
    w = Trio(monkeypatch, n, spawn_rate=16, extra_rows=4096)
    t_col, v_col, _ = w.cols

    def between(t):
        if t == 12:   # translation.z of a band of rows
            vals = w.g.read_component(t_col, 100, 3000).view(np.float32).copy()
            vals[:, 2] = w.rng.uniform(-9.0, 9.0, 3000)
            for x in w.all():
                x.write_component(t_col, 100, vals)
        if t == 15:   # a write that puts back the bits the rows hold: nothing changes
            vals = w.g.read_component(v_col, 2000, 500)
            for x in w.all():
                x.write_component(v_col, 2000, vals)
        if t == 18:
            for r in (0, 63, 64, 4097, n - 1):
                for x in w.all():
                    x.despawn(r)
        if t == 21:
            for x in w.all():
                x.spawn(37)

    w.run(_vectors("synctest", 32), between=between, check_at=(13, 19, 22))
    w.close()


def test_mode2_remove_and_insert(monkeypatch):
    n = 6_007
    w = Trio(monkeypatch, n, optional=True)
    _, v, l = w.cols

    def between(t):
        if t in (10, 11, 14):
            alive = w.o.read_alive(0, n).astype(bool)
            for r in [r for r in range(t * 7, n, 331) if alive[r]]:
                col = v if r % 2 else l
                if t == 14:
                    value = w.g.read_component(col, r - 1, 1)[0]
                    for x in w.all():
                        x.insert_component(col, r, value)
                else:
                    for x in w.all():
                        x.remove_component(col, r)

    w.run(_vectors("synctest", 26), between=between, check_at=(12, 16))
    w.close()


@pytest.mark.parametrize("env", [{"BGR_TUNE_DEFER_LIVE": "0"}, {"BGR_TUNE_HELD_SAVES": "0"}, {"BGR_TUNE_HELD_SAVES": "2"}],
                         ids=["live_every_tick", "no_held_saves", "verify_held_saves"])
def test_engine_settings(monkeypatch, env):
    w = Trio(monkeypatch, 20_011, env=env)
    w.run(_vectors("synctest", 30), check_at=(12,))
    if env.get("BGR_TUNE_HELD_SAVES") == "2":
        held = w.g.held_saves()
        assert held["total"] > 0 and held["mismatched_words"] == 0
    if env.get("BGR_TUNE_HELD_SAVES") == "0":
        assert w.g.held_saves()["total"] == 0
    w.close()


def test_stamp_table_rollover(monkeypatch):
    """The stamp range runs out a few launches in: the table is cleared and the snapshots start from unknown stamps."""
    w = Trio(monkeypatch, 9_001, env={"BGR_TEST_STAMP_FIRST": str(STAMP_LIMIT - 60)})
    w.run(_vectors("p2p", 24), check_at=(2, 6))
    w.close()


def test_four_vectors_in_flight(monkeypatch):
    n, ticks = 120_001, 36
    w = Trio(monkeypatch, n)
    vectors = _vectors("synctest", ticks)
    got, inflight = [], 0
    for info, reqs in vectors[:28]:
        w.g.submit_requests(info, reqs)
        inflight += 1
        if inflight == 4:
            got += w.g.collect()
            inflight -= 1
    while inflight:
        got += w.g.collect()
        inflight -= 1
    want = [w.o.handle_requests(info, reqs) for info, reqs in vectors[:28]]
    assert [w.s.handle_requests(info, reqs) for info, reqs in vectors[:28]] == want
    assert got == [c for out in want for c in out]
    w.run(vectors[28:])
    w.close()


@pytest.mark.parametrize("extra,stamped", [(16, True), (8, False)])
def test_wide_registration(monkeypatch, extra, stamped):
    """The particles schema with `extra` non-checksummed word planes (passive).  With 16 the passive double buffer
    already limits the SM to two blocks and the snapshot fits beside it; with 8 it would cost a third block, so the
    registration runs the instance without stamps."""
    n = 40 * TILE_ROWS + 77
    monkeypatch.setenv("BGR_TUNE_PASSIVE_EARLY", "0")
    g = Engine(max_entities=n, max_depth=9)
    monkeypatch.delenv("BGR_TUNE_PASSIVE_EARLY")
    s = Engine(max_entities=n, max_depth=9, flags=capi.BGR_CFG_FORCE_STEPWISE)
    vals = np.random.default_rng(extra).integers(0, 2**32, (n, extra), dtype=np.uint32)
    for w in (g, s):
        cols = register_particles(w)
        x = w.rollback_component("Extra", 4 * extra, capi.BGR_STRATEGY_CLONE)
        w.build()
        populate(w, cols, *synth_particles(n, 9, 30, 400, z_fraction=0.2))
        w.write_component(x, 0, vals)
    for info, reqs in _vectors("synctest", 30):
        assert g.handle_requests(info, reqs) == s.handle_requests(info, reqs)
        k = g.last_kernel()
        assert k.kind == "bundle" and k.stable_planes == stamped
    rows = g.row_count()
    assert s.row_count() == rows and g.snapshot_frames() == s.snapshot_frames()
    for f in g.snapshot_frames():
        for c in list(cols) + [x]:
            (vg, hg), (vs, hs) = g.peek(f, c, 0, rows), s.peek(f, c, 0, rows)
            m = hs.astype(bool)
            assert np.array_equal(hg, hs) and np.array_equal(vg[m], vs[m])
    g.close()
    s.close()
