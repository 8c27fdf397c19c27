"""-m gpu: the CUDA path through the C ABI vs the oracle, bit-exact (checksums, f32 bit patterns of
Transform/Velocity, Ttl, alive mask, frame counters, ring contents)."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from parity_util import compare_state, run_particles_synctest_pair

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,d,ticks", [(1, 2, 12), (33, 2, 12), (1000, 7, 24), (4097, 4, 16), (50_000, 8, 14)])
def test_synctest_fused_matches_oracle(n, d, ticks):
    r = run_particles_synctest_pair(n, d, ticks, seed=1234 + n)
    assert r["fused"]
    assert r["n_checksums"] > 0
    assert r["checksums_equal"]
    assert r["state_equal"]
    assert r["mismatch_events"] == (0, 0)
    assert r["frames"][0] == r["frames"][1] == ticks
    assert r["ring"][0] == r["ring"][1]
    assert r["confirmed"][0] == r["confirmed"][1]


@pytest.mark.parametrize("n,d,ticks", [(257, 3, 14), (10_000, 8, 12)])
def test_synctest_stepwise_matches_oracle(n, d, ticks):
    r = run_particles_synctest_pair(n, d, ticks, seed=99, flags=capi.BGR_CFG_FORCE_STEPWISE)
    assert not r["fused"]
    assert r["checksums_equal"] and r["state_equal"]
    assert r["ring"][0] == r["ring"][1]


@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
def test_despawn_inside_the_rollback_window(flags):
    """ttl ~ U(1, 2*window): particles die inside the window, are resurrected by Load and die again
    (entity.rs:55-99 reconcile + despawn_particles).  active count, entity checksum part and the
    alive mask must track the oracle exactly."""
    r = run_particles_synctest_pair(5000, 6, 30, seed=5, ttl_lo=1, ttl_hi=12, flags=flags)
    assert r["checksums_equal"] and r["state_equal"]
    assert r["active"][0] == r["active"][1]
    assert r["active"][0] == 0  # everything is dead after 30 frames


def test_fused_and_stepwise_agree_checksum_for_checksum():
    a = run_particles_synctest_pair(20_000, 8, 12, seed=42)
    b = run_particles_synctest_pair(20_000, 8, 12, seed=42, flags=capi.BGR_CFG_FORCE_STEPWISE)
    assert a["checksums"] == b["checksums"]
    # one launch per tick on the fused path (+0 for setup): stepwise needs dozens
    assert a["launches"] == 12
    assert b["launches"] > 10 * a["launches"]


@pytest.mark.parametrize("ticks", [4, 5, 6])
def test_spawn_in_plain_save_advance_ticks_writes_whole_rows(ticks):
    """Before the first rollback (check_distance 6) the ticks are [Save, Advance]; with input_delay 2 the spawn
    key pressed on ticks 1-2 fires on frames 3-4.  Rows spawned there must be complete in the live image
    (Transform::default() rotation / scale are passive planes)."""
    r = run_particles_synctest_pair(100, 6, ticks, seed=3, ttl_lo=50, ttl_hi=60, spawn_rate=30, spawn_ttl=50)
    assert r["fused"] and r["rows"][0] == r["rows"][1] > 100
    assert r["checksums_equal"] and r["state_equal"]


@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_SKIP_UNCHANGED_PLANES])
def test_skip_unchanged_planes_is_observably_identical(flags):
    """BGR_CFG_SKIP_UNCHANGED_PLANES only elides redundant stores: checksums, live state, and the bytes peeked
    out of every snapshot (including passive rotation/scale) equal the oracle's, with spawns bumping the
    content version mid-run."""
    r = run_particles_synctest_pair(2000, 5, 30, seed=8, ttl_lo=4, ttl_hi=60, flags=flags, spawn_rate=20, spawn_ttl=12,
                                    peek_check=True)
    assert r["fused"] and r["checksums_equal"] and r["state_equal"] and r["peek_equal"]


@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
def test_spawn_particles_inside_the_rollback_window(flags):
    """SURVEY §8f rank 1: spawn_particles.run_if(spawn_pressed) with the rolled-back ParticleRng — rows are born
    (and, with ttl 9, die) inside the rollback window; Load shrinks RollbackOrdered and the resimulation must
    re-spawn the same particles.  Row count, alive mask, columns and every checksum track the oracle."""
    r = run_particles_synctest_pair(300, 6, 36, seed=11, ttl_lo=3, ttl_hi=40, flags=flags, spawn_rate=40,
                                    spawn_ttl=9, startup_burst=True)
    assert r["fused"] == (flags == 0)
    assert r["rows"][0] == r["rows"][1] > 300 + 40 * 10
    assert r["checksums_equal"] and r["state_equal"]
    assert r["active"][0] == r["active"][1]
    assert r["mismatch_events"] == (0, 0)
    assert r["ring"][0] == r["ring"][1]


def test_extra_passive_columns_of_odd_sizes_ride_along():
    """SURVEY §8f rank 3: the example also registers render-side PODs (GlobalTransform 48 B, Visibility /
    InheritedVisibility / ViewVisibility 1 B each).  No compiled system touches them: they are passive planes
    (several TMA runs, sub-word elements) and must survive save / load / resimulation byte for byte."""
    import numpy as np
    from bevy_ggrs_b200.engine import Engine
    from bevy_ggrs_b200.plugin import App, GgrsPlugin, LocalInputs, ReadInputs, Session
    from bevy_ggrs_b200.session import SyncTestSession
    from bevy_ggrs_b200.stress import synth_particles
    from oracle_backend import OracleWorld

    n, d, ticks = 3000, 5, 20
    rng = np.random.default_rng(3)
    gt = rng.integers(0, 256, size=(n, 48), dtype=np.uint8)
    vis = rng.integers(0, 3, size=(n, 1), dtype=np.uint8)
    odd = rng.integers(0, 256, size=(n, 6), dtype=np.uint8)      # a 6-byte POD: 1.5 words
    worlds, apps, colsets = [], [], []
    for backend in (Engine(max_entities=n, max_depth=8), OracleWorld()):
        app = App(backend)
        app.add_plugins(GgrsPlugin())
        app.add_systems(ReadInputs, lambda a: a.insert_resource(LocalInputs({h: 0 for h in a.local_players.handles})))
        c_gt = app.rollback_component_with_clone("GlobalTransform", 48)
        c_t = app.rollback_component_with_clone("Transform", 40)
        c_vis = app.rollback_component_with_clone("Visibility", 1)
        c_v = app.rollback_component_with_copy("Velocity", 12)
        c_odd = app.rollback_component_with_copy("Odd6", 6)
        c_l = app.rollback_component_with_copy("Ttl", 8)
        app.checksum_component(c_v, 0, 12, assert_finite=True).checksum_component(c_t, 0, 12, assert_finite=True)
        backend.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [c_t, c_v])
        backend.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [c_l])
        app.insert_resource(Session.SyncTest(SyncTestSession(1, d, 8)))
        app._finish()
        tf, vel, ttl = synth_particles(n, 21, 4, 30)
        first = backend.spawn(n)
        for c, a in ((c_gt, gt), (c_t, tf), (c_vis, vis), (c_v, vel), (c_odd, odd), (c_l, ttl)):
            backend.write_component(c, first, a)
        worlds.append(backend); apps.append(app); colsets.append((c_gt, c_t, c_vis, c_v, c_odd, c_l))
    cs = [[], []]
    for _ in range(ticks):
        for i, app in enumerate(apps):
            app.step()
            cs[i] += app.last_checksums
    eng, orc = worlds
    assert eng.last_path_fused()
    assert cs[0] == cs[1] and len(cs[0]) > ticks
    alive = orc.read_alive(0, n).astype(bool)
    assert np.array_equal(eng.read_alive(0, n).astype(bool), alive) and alive.any() and not alive.all()
    for c in colsets[0]:
        assert np.array_equal(eng.read_component(c, 0, n)[alive], orc.read_component(c, 0, n)[alive])
    # passive columns are untouched by 20 frames of rollback
    assert np.array_equal(eng.read_component(colsets[0][0], 0, n)[alive], gt[alive])
    assert np.array_equal(eng.read_component(colsets[0][4], 0, n)[alive], odd[alive])
    # peek a snapshot: same bytes as the oracle's snapshot of that frame
    f = eng.snapshot_frames()[-1]
    pe, po = eng.peek(f, colsets[0][0], 0, n), orc.peek(f, colsets[0][0], 0, n)
    m = po[1].astype(bool)
    assert np.array_equal(pe[1].astype(bool), m) and np.array_equal(pe[0][m], po[0][m])


@pytest.mark.parametrize("z_fraction", [1.0, 0.02, 0.5])
@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
def test_non_zero_z_takes_the_general_hash_path(z_fraction, flags):
    """The fused kernel skips one diffusion when a whole warp has z == +0.0 (the example is 2-D); rows with a
    non-zero z — all of them, a few (mixed warps), half — must hash exactly like the oracle."""
    r = run_particles_synctest_pair(6000, 4, 14, seed=31, ttl_lo=3, ttl_hi=40, flags=flags, z_fraction=z_fraction)
    assert r["checksums_equal"] and r["state_equal"]


@pytest.mark.parametrize("bps,dynamic", [("1", "1"), ("1", "0"), ("2", "1")])
def test_many_tiles_per_block(monkeypatch, bps, dynamic):
    """Blocks that run many tile iterations (one resident block per SM, 780 tiles): exercises the dynamic tile
    ring (claims two ahead, slot reuse, empty/full mbarrier phases) and the static stride far past the first
    wave.  A protocol error here hangs, so the run is bounded by pytest-timeout."""
    monkeypatch.setenv("BGR_TUNE_BPS", bps)
    monkeypatch.setenv("BGR_TUNE_DYNAMIC", dynamic)
    r = run_particles_synctest_pair(400_000, 2, 6, seed=17, ttl_lo=2, ttl_hi=30)
    assert r["fused"] and r["checksums_equal"] and r["state_equal"]


test_many_tiles_per_block = pytest.mark.timeout(120)(test_many_tiles_per_block)


@pytest.mark.parametrize("group,flags", [(3, 0), (4, 0), (2, capi.BGR_CFG_FORCE_STEPWISE)])
def test_catch_up_ticks_in_one_request_vector_match_tick_by_tick(group, flags):
    """run_ggrs_schedules runs several GGRS ticks back to back when a frame was long (schedule_systems.rs:60-82).
    Handing their request vectors to bgr_handle_requests as ONE vector (several LoadGameState inside) is one fused
    launch and is observably identical to the oracle executing them one tick at a time: checksums, live state,
    snapshot contents; particles die and are spawned inside the window."""
    from bevy_ggrs_b200.session import SAVE, SyncTestSession
    from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
    from oracle_backend import OracleWorld
    n, d, maxp, n_ticks = 2500, 4, 8, 24
    eng, orc = Engine(max_entities=n + 60 * n_ticks, max_depth=maxp, flags=flags), OracleWorld()
    cols = None
    for w in (eng, orc):
        cols = register_particles(w, spawn_rate=40, spawn_ttl=7)
        w.build()
        populate(w, cols, *synth_particles(n, 21, 3, 40))
    sess = SyncTestSession(2, d, maxp, input_delay=2)
    vectors = []
    for t in range(n_ticks):
        sess.add_local_input(0, (1 << 4) if t % 5 in (1, 2) else 0)   # INPUT_SPAWN
        sess.add_local_input(1, (1 << 5) if t % 3 == 0 else 0)        # INPUT_NOOP
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)   # checksums are compared below, not by the stand-in session
        vectors.append(reqs)
    got, want = [], []
    launches0 = eng.launch_count()
    for g in range(0, n_ticks, group):
        merged = [r for v in vectors[g:g + group] for r in v]
        got += eng.handle_requests(sess.info(), merged)
        for v in vectors[g:g + group]:
            want += orc.handle_requests(sess.info(), v)
    assert got == want and len(got) > n_ticks
    if not flags:
        assert eng.last_path_fused() and eng.launch_count() - launches0 == n_ticks // group
    rows = eng.row_count()
    assert rows == orc.row_count() > n
    assert compare_state(eng, orc, cols, rows)
    assert eng.snapshot_frames() == orc.snapshot_frames()
    for f in eng.snapshot_frames():
        for c in cols:
            pe, po = eng.peek(f, c, 0, rows), orc.peek(f, c, 0, rows)
            m = po[1].astype(bool)
            assert np.array_equal(pe[1].astype(bool), m) and np.array_equal(pe[0][m], po[0][m])


@pytest.mark.timeout(180)
@pytest.mark.parametrize("tiledep", ["0", "1", "2"])
@pytest.mark.parametrize("n,spawn", [(3000, 40), (300_000, 0)])
def test_pipelined_submits_overlap_without_observable_change(monkeypatch, tiledep, n, spawn):
    """Four request vectors in flight (bgr_submit_requests / bgr_collect).  With BGR_TUNE_TILEDEP=1 consecutive fused
    launches overlap on the GPU: tile i of tick k+1 starts as soon as tile i of tick k has signalled, not when the
    whole grid of tick k is done.  Checksums of every tick, the final world and every snapshot equal the oracle's.
    A dependency bug hangs or corrupts: bounded by pytest-timeout."""
    from bevy_ggrs_b200.session import SAVE, SyncTestSession
    from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
    from oracle_backend import OracleWorld
    monkeypatch.setenv("BGR_TUNE_TILEDEP", tiledep)
    d, maxp, n_ticks = 3, 8, 30 if n < 100_000 else 12
    eng, orc = Engine(max_entities=n + (spawn + 1) * n_ticks, max_depth=maxp), OracleWorld()
    cols = None
    for w in (eng, orc):
        cols = register_particles(w, spawn_rate=spawn, spawn_ttl=7) if spawn else register_particles(w)
        w.build()
        populate(w, cols, *synth_particles(n, 33, 3, 40))
    sess = SyncTestSession(2, d, maxp, input_delay=2)
    vectors = []
    for t in range(n_ticks):
        sess.add_local_input(0, (1 << 4) if (spawn and t % 5 in (1, 2)) else 0)
        sess.add_local_input(1, (1 << 5) if t % 3 == 0 else 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        vectors.append(reqs)
    got, want, inflight = [], [], 0
    for v in vectors:
        eng.submit_requests(sess.info(), v)
        inflight += 1
        if inflight == 4:
            got += eng.collect()
            inflight -= 1
        want += orc.handle_requests(sess.info(), v)
    while inflight:
        got += eng.collect()
        inflight -= 1
    assert got == want and len(got) >= n_ticks
    assert eng.last_path_fused()
    rows = eng.row_count()
    assert rows == orc.row_count()
    assert compare_state(eng, orc, cols, rows)
    assert eng.snapshot_frames() == orc.snapshot_frames()
    for f in eng.snapshot_frames()[:3]:
        for c in cols:
            pe, po = eng.peek(f, c, 0, rows), orc.peek(f, c, 0, rows)
            m = po[1].astype(bool)
            assert np.array_equal(pe[1].astype(bool), m) and np.array_equal(pe[0][m], po[0][m])


@pytest.mark.parametrize("jit_rows", ["4", "2", "1"])
@pytest.mark.parametrize("n,d,ticks", [(257, 3, 14), (10_000, 8, 12)])
def test_particles_world_on_the_generic_program_matches_oracle(monkeypatch, generic_kernel, n, d, ticks, jit_rows):
    """BGR_TUNE_BUNDLE=0 takes the specialised particles kernel out: the same world runs on the generic one-launch
    program (shared-memory tile, systems and hashes driven by the registration) and must match the oracle bit for bit,
    including despawns inside the window and the passive Transform planes of every snapshot."""
    monkeypatch.setenv("BGR_TUNE_BUNDLE", "0")
    monkeypatch.setenv("BGR_TUNE_JIT_ROWS", jit_rows)  # specialised whole-tile kernel: 4 / 2 / 1 rows per thread
    r = run_particles_synctest_pair(n, d, ticks, seed=5, ttl_lo=3, ttl_hi=40, peek_check=True, z_fraction=0.3)
    assert r["fused"] and r["launches"] == ticks
    assert r["checksums_equal"] and r["state_equal"] and r["peek_equal"]
    assert r["ring"][0] == r["ring"][1] and r["active"][0] == r["active"][1] < n


@pytest.mark.timeout(180)
@pytest.mark.parametrize("grid,jit_rows", [("3", "4"), ("7", "2"), ("40", "4")])
def test_generic_program_blocks_that_run_many_tiles(monkeypatch, generic_kernel, grid, jit_rows):
    """The generic one-launch program with far fewer blocks than tiles (BGR_TUNE_GRID): every block claims tile after
    tile from the global counter, reloads its shared-memory tile, and must wait for its own bulk stores before the
    buffer is overwritten.  (Without the cap a world needs > 1.2M entities before a block sees a second tile.)"""
    monkeypatch.setenv("BGR_TUNE_BUNDLE", "0")
    monkeypatch.setenv("BGR_TUNE_GRID", grid)
    monkeypatch.setenv("BGR_TUNE_JIT_ROWS", jit_rows)
    r = run_particles_synctest_pair(60_000, 4, 10, seed=23, ttl_lo=3, ttl_hi=40, peek_check=True, z_fraction=0.2)
    assert r["fused"] and r["launches"] == 10
    assert r["checksums_equal"] and r["state_equal"] and r["peek_equal"]
    assert r["active"][0] == r["active"][1] < 60_000


@pytest.mark.parametrize("n,d,spawn", [(700, 3, 0), (20_000, 8, 0), (3000, 6, 40)])
def test_small_worlds_match_the_oracle(n, d, spawn):
    """Single-wave worlds (2 to 40 tiles) on the fused kernel match the oracle — despawns, spawns inside the window,
    snapshots of every frame."""
    r = run_particles_synctest_pair(n, d, 16, seed=31, ttl_lo=3, ttl_hi=30, peek_check=True, z_fraction=0.25,
                                    spawn_rate=spawn, spawn_ttl=9, startup_burst=bool(spawn))
    assert r["fused"] and r["launches"] == 16
    assert r["checksums_equal"] and r["state_equal"] and r["peek_equal"]
    assert r["ring"][0] == r["ring"][1] and r["active"][0] == r["active"][1]


def test_pipelined_overlap_on_a_single_wave_world(monkeypatch):
    """Tile dependencies on synchronous and queued calls alike (BGR_TUNE_TILEDEP=2) on a world of 118 tiles."""
    from bevy_ggrs_b200.session import SAVE, SyncTestSession
    from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
    from oracle_backend import OracleWorld
    monkeypatch.setenv("BGR_TUNE_TILEDEP", "2")
    n, d, maxp, n_ticks = 60_000, 3, 8, 24
    eng, orc = Engine(max_entities=n, max_depth=maxp), OracleWorld()
    for w in (eng, orc):
        cols = register_particles(w)
        w.build()
        populate(w, cols, *synth_particles(n, 77, 3, 40))
    sess = SyncTestSession(2, d, maxp, input_delay=2)
    got, want, inflight = [], [], 0
    for t in range(n_ticks):
        sess.add_local_input(0, 0); sess.add_local_input(1, (1 << 5) if t % 3 == 0 else 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        eng.submit_requests(sess.info(), reqs)
        inflight += 1
        if inflight == 4:
            got += eng.collect(); inflight -= 1
        want += orc.handle_requests(sess.info(), reqs)
    while inflight:
        got += eng.collect(); inflight -= 1
    assert got == want
    assert compare_state(eng, orc, cols, n)
    eng.close(); orc.close()
