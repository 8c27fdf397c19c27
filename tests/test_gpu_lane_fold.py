"""-m gpu: the bundle kernel's checksum fold against the oracle.

Every lane adds the partials of each Save to its own shared-memory slot, and each block reduces the slots once, after
its tiles (the lane fold).  A launch whose slots would cost a resident block reduces over the warp at every Save
instead (the warp fold, Engine.last_kernel().warp_fold).  The cases cover vectors of 1 to 40 Saves on every MODE, grids
whose blocks run several tiles, single-wave and multi-wave grids, row counts that are not a multiple of 64, despawns
and dead rows inside the vector, a non-finite value in the last tile, absent components, the warp-fold fallback of a
wide registration and four vectors in flight."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request
from bevy_ggrs_b200.stress import synth_particles
from oracle_backend import OracleError, OracleWorld
from parity_util import compare_state

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
CLONE, COPY = capi.BGR_STRATEGY_CLONE, capi.BGR_STRATEGY_COPY
# SyncTest of check distance 2: frames older than two behind the current one leave the snapshot ring
SESS = (capi.BGR_SESSION_SYNCTEST, 8, 2, 0)
# the render-side components of the example next to the bundle: with the Transform's 7, 22 passive planes, a passive
# double buffer of 2 x 44 KB and two resident blocks per SM, which 40 Saves' lane slots (25 KB) would cut to one
RENDER_SIDE = (("GlobalTransform", 48, CLONE), ("Visibility", 1, CLONE), ("Odd6", 6, COPY))
# 20 tiles, BGR_TUNE_GRID=3: every block runs six or seven tiles; 6 tiles on 132 SMs: one wave, one tile per block
GRIDS = {"tiles_per_block": (10_037, "3"), "single_wave": (3_029, None)}


def _pair(mode, n, extra=(), ck=None, seed=5):
    """Engine + oracle with the particles bundle after `extra` columns.  mode 0: both columns checksummed without the
    finite assertion; 1: both with it; 2: Velocity and Ttl optional, some rows without one of them.  Some rows are
    despawned and the Ttl of the others runs out from frame 1 on.  ck = (t flags, v flags) overrides the checksums."""
    eng, orc = Engine(max_entities=n, max_depth=8), OracleWorld()
    rng = np.random.default_rng(seed)
    tf, vel, ttl = synth_particles(n, seed, 1, 120, z_fraction=0.2)
    data = [rng.integers(0, 256, (n, size), dtype=np.uint8) for _, size, _ in extra]
    rows = rng.permutation(n)
    gone, absent = rows[:n // 50], rows[n // 50:n // 50 + n // 20]
    cols = None
    for w in (eng, orc):
        xs = [w.rollback_component(name, size, strat) for name, size, strat in extra]
        t = w.rollback_component("Transform", 40, CLONE)
        v = w.rollback_component("Velocity", 12, COPY | (OPT if mode == 2 else 0))
        l = w.rollback_component("Ttl", 8, COPY | (OPT if mode == 2 else 0))
        ft, fv = ck if ck is not None else ((0, 0) if mode == 0 else (FIN, FIN))
        w.checksum_component(v, 0, 12, fv)
        w.checksum_component(t, 0, 12, ft)
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        w.build()
        w.spawn(n)
        w.write_component(t, 0, tf); w.write_component(v, 0, vel); w.write_component(l, 0, ttl)
        for c, a in zip(xs, data):
            w.write_component(c, 0, a)
        for r in gone:
            w.despawn(int(r))
        if mode == 2:
            for i, r in enumerate(absent):
                w.remove_component((v, l)[i % 2], int(r))
        cols = xs + [t, v, l]
    return eng, orc, cols


def _saves(frame, count, load=None):
    """[Load(load)] + (Save, Advance) x count from `frame`, the current frame (`load` after a Load); returns the vector
    and the frame after it"""
    reqs = [Request(LOAD, load)] if load is not None else []
    frame = load if load is not None else frame
    for k in range(count):
        reqs += [Request(SAVE, frame + k), Request(ADVANCE, 0, [0])]
    return reqs, frame + count


def _outcome(w, reqs):
    try:
        return ("ok", w.handle_requests(SESS, reqs))
    except (BgrError, OracleError) as ex:
        return ("raised", ex.status, str(ex))


def _same_worlds(eng, orc, cols, mode=1):
    rows = eng.row_count()
    assert rows == orc.row_count()
    if mode == 2:  # per-column presence, and the values where present
        assert np.array_equal(eng.read_alive(0, rows).astype(bool), orc.read_alive(0, rows).astype(bool))
        for c in cols:
            vo, ho = orc.read_component_alive(c, 0, rows)
            he = eng.has_component(c, 0, rows).astype(bool)
            assert np.array_equal(he, ho.astype(bool)), c
            assert np.array_equal(eng.read_component(c, 0, rows)[he], vo[he]), c
    else:
        assert compare_state(eng, orc, cols, rows)
    assert eng.snapshot_frames() == orc.snapshot_frames()


@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("saves", [1, 8, 16, 40])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_lane_fold_matches_the_oracle(monkeypatch, mode, saves, grid):
    """A vector of `saves` Saves from the live image, then one that Loads its last frame and saves again."""
    n, tune_grid = GRIDS[grid]
    if tune_grid:
        monkeypatch.setenv("BGR_TUNE_GRID", tune_grid)
    eng, orc, cols = _pair(mode, n, seed=saves + mode)
    second = min(saves, 39)  # a Load and 39 (Save, Advance) pairs fill the 80 requests of a vector
    for reqs, _ in (_saves(0, saves), _saves(saves, second, load=saves - 1)):
        assert eng.handle_requests(SESS, reqs) == orc.handle_requests(SESS, reqs)
        k = eng.last_kernel()
        assert (k.kind, k.mode) == ("bundle", mode) and not k.warp_fold
    assert 0 < orc.read_alive(0, n).sum() < n
    _same_worlds(eng, orc, cols, mode)
    eng.close(); orc.close()


def test_lane_fold_on_a_multi_wave_grid_with_stamps():
    """489 tiles: the stamped instance on a grid of several waves, three vectors of 16 Saves."""
    n = 250_013
    eng, orc, cols = _pair(1, n, seed=11)
    frame = 0
    for i in range(3):
        reqs, frame = _saves(frame, 16, load=frame - 1 if i else None)
        assert eng.handle_requests(SESS, reqs) == orc.handle_requests(SESS, reqs)
        k = eng.last_kernel()
        assert k.kind == "bundle" and k.stable_planes and not k.warp_fold
    _same_worlds(eng, orc, cols)
    eng.close(); orc.close()


@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("setup", ["mode1", "t_fin_v_plain"])
def test_non_finite_in_the_last_tile_raises_where_the_oracle_panics(monkeypatch, setup, grid):
    """+inf in the y of one live row's Velocity, in the last tile.  With both columns asserted the first Save raises;
    with only the Transform asserted the Save after the first Advance does.  Either way the engine raises on the vector
    and with the text the oracle panics with, and returns the oracle's checksums on every vector before it."""
    n, tune_grid = GRIDS[grid]
    if tune_grid:
        monkeypatch.setenv("BGR_TUNE_GRID", tune_grid)
    eng, orc, cols = _pair(1, n, ck=None if setup == "mode1" else (FIN, 0), seed=3)
    row = n - 7
    alive = orc.read_alive(0, n)
    while not alive[row]:
        row -= 1
    assert row // 512 == (n - 1) // 512
    vel = orc.read_component(cols[1], row, 1).view(np.uint32).copy()
    vel[0, 1] = 0x7F800000
    for w in (eng, orc):
        w.write_component(cols[1], row, vel)
        w.write_component(cols[2], row, np.array([50], np.uint64))  # alive for the whole vector
    outcomes = []
    for f in range(3):
        reqs, _ = _saves(8 * f, 8)
        a, b = _outcome(eng, reqs), _outcome(orc, reqs)
        assert a == b, (f, a, b)
        outcomes.append(a[0])
        if a[0] == "raised":
            assert a[1] == capi.BGR_ERR_NON_FINITE
            break
    assert outcomes == ["raised"]
    k = eng.last_kernel()
    assert k.kind == "bundle" and k.mode == (1 if setup == "mode1" else 0) and not k.warp_fold
    eng.close(); orc.close()


def test_wide_registration_takes_the_warp_fold():
    """RENDER_SIDE: a vector of 8 Saves keeps the lane fold, one of 40 runs the warp fold, both in the passive-TMA
    configuration; both match the oracle, and so do the 8 Saves after it."""
    n = 3_029
    eng, orc, cols = _pair(1, n, extra=RENDER_SIDE, seed=13)
    for (reqs, _), warp in ((_saves(0, 8), False), (_saves(8, 40), True), (_saves(48, 8, load=47), False)):
        assert eng.handle_requests(SESS, reqs) == orc.handle_requests(SESS, reqs)
        k = eng.last_kernel()
        assert k.kind == "bundle" and k.mode == 1 and k.passive_tma and k.warp_fold == warp
    _same_worlds(eng, orc, cols)
    eng.close(); orc.close()


@pytest.mark.parametrize("mode", [1, 2])
def test_four_vectors_in_flight(mode):
    """Up to four vectors queued behind each other, 1 to 40 Saves each: overlapping launches rotate over the
    accumulator sets, which each launch's last block re-arms."""
    n = 20_011
    eng, orc, cols = _pair(mode, n, seed=17)
    counts = [8, 1, 40, 16, 8, 39, 2, 8, 16, 40, 8]
    got, want, inflight, frame = [], [], 0, 0
    for i, c in enumerate(counts):
        reqs, frame = _saves(frame, c, load=frame - 1 if i % 2 and c < 40 else None)
        eng.submit_requests(SESS, reqs)
        inflight += 1
        if inflight == 4:
            got += eng.collect()
            inflight -= 1
        want += orc.handle_requests(SESS, reqs)
    while inflight:
        got += eng.collect()
        inflight -= 1
    assert got == want and len(got) == sum(counts)
    assert eng.last_kernel().kind == "bundle"
    _same_worlds(eng, orc, cols, mode)
    eng.close(); orc.close()
