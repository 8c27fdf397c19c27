"""-m gpu: every variant of the compiled particles kernel the engine can select, against the oracle.

The bundle kernel (k_particles_program) is instantiated per checksum mode (MODE 0: the checksum / finite flags are
tested at run time; MODE 1: both columns checksummed with the finite assertion; MODE 2: optional columns), and a launch
moves the passive planes by TMA bulk copies or per thread.  Each case asserts through Engine.last_kernel() that the variant it names is the one that
ran, then compares checksums, live state, ring frames and snapshot bytes with the oracle."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleError, OracleWorld
from parity_util import compare_state, run_particles_synctest_pair

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
SINGLE_WAVE, MULTI_WAVE = 3000, 250_000   # 6 tiles; 489 tiles (> 3 x 132 SMs: the grid runs several waves)


def _ck(v=None, t=None):
    """A checksum registration for register_particles: None = column not checksummed, else its flags."""
    def reg(w, tc, vc):
        if v is not None:
            w.checksum_component(vc, 0, 12, v)
        if t is not None:
            w.checksum_component(tc, 0, 12, t)
    return reg


# the six checksum setups that run MODE 0 (MODE 1 needs both columns with the finite assertion)
MODE0_SETUPS = {"none": _ck(), "v_only": _ck(v=FIN), "t_only": _ck(t=FIN), "both_plain": _ck(v=0, t=0),
                "t_fin_v_plain": _ck(v=0, t=FIN), "v_fin_t_plain": _ck(v=FIN, t=0)}
MODE1 = _ck(v=FIN, t=FIN)


def _assert_parity(r, peek=True):
    assert r["checksums_equal"] and r["state_equal"], r["kernel"]
    assert r["ring"][0] == r["ring"][1] and r["active"][0] == r["active"][1]
    assert r["mismatch_events"] == (0, 0)
    if peek:
        assert r["peek_equal"]


# ---------------------------------------------------------------------------------------------------------------------
# MODE 0: checksum flags tested at run time
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 33, 4097])
@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
@pytest.mark.parametrize("setup", list(MODE0_SETUPS))
def test_mode0_checksum_setups_match_the_oracle(setup, flags, n):
    """Deaths (ttl from 1) and spawns (rate 20, ttl 6) inside the rollback window, every snapshot peeked."""
    r = run_particles_synctest_pair(n, 4, 14, seed=40 + n, ttl_lo=1, ttl_hi=16, spawn_rate=20, spawn_ttl=6,
                                    peek_check=True, z_fraction=0.3, flags=flags, checksums=MODE0_SETUPS[setup])
    k = r["kernel"]
    if flags:
        assert not r["fused"] and k.kind == "stepwise_tma"
    else:
        assert r["fused"] and k.kind == "bundle" and k.mode == 0 and k.vec == 2
    assert r["rows"][0] == r["rows"][1] > n
    _assert_parity(r)


def _outcome(w, reqs):
    try:
        return ("ok", w.handle_requests(NOSESS, reqs))
    except (BgrError, OracleError) as ex:
        return ("raised", ex.status, str(ex))


# +inf, -inf, quiet NaNs of both signs, signalling NaNs (one with a payload): every encoding the hasher refuses
NON_FINITE = [0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFC01234]


@pytest.mark.parametrize("pattern", NON_FINITE, ids=hex)
@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
@pytest.mark.parametrize("column", ["velocity", "transform"])
@pytest.mark.parametrize("setup", list(MODE0_SETUPS) + ["mode1"])
def test_non_finite_raises_exactly_when_the_oracle_panics(setup, column, flags, pattern):
    """A non-finite bit pattern in the y of one live row's Velocity or Transform.translation.  The hasher's assertion
    fires only where the column is checksummed with the finite flag (a non-finite velocity reaches the translation on
    the next Advance): the engine raises BGR_ERR_NON_FINITE with the reference's text on exactly the vector where the
    oracle panics, and returns the oracle's checksums on every vector before it."""
    reg = MODE1 if setup == "mode1" else MODE0_SETUPS[setup]
    n = 700
    eng, orc = Engine(max_entities=n, max_depth=8, flags=flags), OracleWorld()
    for w in (eng, orc):
        cols = register_particles(w, checksums=reg)
        w.build()
        tf, vel, ttl = synth_particles(n, 12, 50, 60)
        (vel if column == "velocity" else tf).view(np.uint32)[517, 1] = pattern
        populate(w, cols, tf, vel, ttl)
    outcomes = []
    nan = (pattern & 0x7FFFFF) != 0
    for f in range(3):
        reqs = [Request(SAVE, f), Request(ADVANCE, 0, [0])]
        a, b = _outcome(eng, reqs), _outcome(orc, reqs)
        if nan and f > 0 and a[0] == "ok":
            # a NaN that went through an Advance: its payload is not specified, so neither is a checksum without the assertion
            assert b[0] == "ok" and len(a[1]) == len(b[1]), (f, a, b)
        else:
            assert a == b, (f, a, b)
        k = eng.last_kernel()
        assert k.kind == ("stepwise_tma" if flags else "bundle") and (flags or k.mode == (1 if setup == "mode1" else 0))
        outcomes.append(a[0])
        if a[0] == "raised":
            assert a[1] == capi.BGR_ERR_NON_FINITE and a[2] == "Hashing is not stable for NaN f32 values."
            break
    fin_v = setup in ("v_only", "v_fin_t_plain", "mode1")
    fin_t = setup in ("t_only", "t_fin_v_plain", "mode1")
    # velocity inf: V's own hash at the first Save; it reaches the translation after one Advance
    expect = ["raised"] if (fin_v and column == "velocity") or (fin_t and column == "transform") else \
        (["ok", "raised"] if fin_t and column == "velocity" else ["ok"] * 3)
    assert outcomes == expect
    eng.close(); orc.close()


# ---------------------------------------------------------------------------------------------------------------------
# the instantiation matrix: MODE 0 and 1, single-wave and multi-wave grids
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [SINGLE_WAVE, MULTI_WAVE])
@pytest.mark.parametrize("mode", [0, 1])
def test_every_vec_tier_mode_instantiation_matches_the_oracle(mode, n):
    big = n == MULTI_WAVE
    r = run_particles_synctest_pair(n, 2 if big else 4, 6 if big else 12, seed=22, ttl_lo=2,
                                    ttl_hi=20, z_fraction=0.2, peek_check=not big,
                                    checksums=MODE1 if mode else MODE0_SETUPS["both_plain"])
    k = r["kernel"]
    assert r["fused"] and k.kind == "bundle"
    assert (k.vec, k.mode, k.tier, k.item_rows) == (2, mode, 1, 512)
    assert k.passive_tma   # the example's layout: the Transform's 7 passive planes are one TMA run
    _assert_parity(r, peek=not big)


# ---------------------------------------------------------------------------------------------------------------------
# worlds with extra passive columns (registration order decides the plane layout)
# ---------------------------------------------------------------------------------------------------------------------
def _extra_pair(layout, n, max_depth=8, spawn_rate=0, spawn_ttl=7, seed=3):
    """Engine + oracle with the particles bundle plus extra columns.  layout: registration order, "T" / "V" / "L" for
    Transform / Velocity / Ttl, else (name, elem_bytes, strategy).  Returns (eng, orc, columns in layout order)."""
    extra_cap = spawn_rate * 64
    eng, orc = Engine(max_entities=n + extra_cap, max_depth=max_depth), OracleWorld()
    rng = np.random.default_rng(seed)
    tf, vel, ttl = synth_particles(n, seed, 3, 40, z_fraction=0.2)
    data = {i: rng.integers(0, 256, (n, it[1]), dtype=np.uint8) for i, it in enumerate(layout) if isinstance(it, tuple)}
    cols = None
    for w in (eng, orc):
        cols, named = [], {}
        for it in layout:
            if it == "T":
                c = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
            elif it == "V":
                c = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
            elif it == "L":
                c = w.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY)
            else:
                c = w.rollback_component(it[0], it[1], it[2])
            cols.append(c)
            if isinstance(it, str):
                named[it] = c
        t, v, l = named["T"], named["V"], named["L"]
        w.checksum_component(v, 0, 12, FIN)
        w.checksum_component(t, 0, 12, FIN)
        if spawn_rate:
            w.add_system(capi.BGR_SYS_PARTICLES_SPAWN, [t, v, l], [spawn_rate, spawn_ttl, 77, 0])
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        w.build()
        first = w.spawn(n)
        w.write_component(t, first, tf); w.write_component(v, first, vel); w.write_component(l, first, ttl)
        for i, a in data.items():
            w.write_component(cols[i], first, a)
    return eng, orc, cols


def _synctest_vectors(n_ticks, d, maxp, spawn_ticks=(), input_delay=0):
    sess = SyncTestSession(2, d, maxp, input_delay=input_delay)
    vectors = []
    for t in range(n_ticks):
        sess.add_local_input(0, (1 << 4) if t in spawn_ticks else 0)   # INPUT_SPAWN
        sess.add_local_input(1, (1 << 5) if t % 3 == 0 else 0)        # INPUT_NOOP
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)   # checksums are compared against the oracle, not by the stand-in session
        vectors.append(reqs)
    return sess.info(), vectors


def _run_vectors(eng, orc, cols, info, vectors, merge_first=1):
    """The first `merge_first` tick vectors as ONE request vector on the engine (tick by tick on the oracle), then one
    vector per tick.  Compares checksums after every vector; returns the kernel of each engine vector."""
    kernels = []
    groups = [vectors[:merge_first]] + [[v] for v in vectors[merge_first:]]
    for g in groups:
        got = eng.handle_requests(info, [r for v in g for r in v])
        want = [c for v in g for c in orc.handle_requests(info, v)]
        assert got == want
        kernels.append(eng.last_kernel())
    rows = eng.row_count()
    assert rows == orc.row_count()
    assert compare_state(eng, orc, cols, rows)
    assert eng.snapshot_frames() == orc.snapshot_frames()
    for f in eng.snapshot_frames():
        for c in cols:
            pe, po = eng.peek(f, c, 0, rows), orc.peek(f, c, 0, rows)
            m = po[1].astype(bool)
            assert np.array_equal(pe[1].astype(bool), m) and np.array_equal(pe[0][m], po[0][m])
    return kernels


CLONE, COPY = capi.BGR_STRATEGY_CLONE, capi.BGR_STRATEGY_COPY
# the render-side components of the example next to the bundle: 22 passive planes, 2 x 44 KB of shared memory
RENDER_SIDE = [("GlobalTransform", 48, CLONE), "T", ("Visibility", 1, CLONE), "V", ("Odd6", 6, COPY), "L"]


def test_first_vector_with_a_spawn_then_plain_ticks_with_a_large_passive_buffer():
    """The first launch of the kernel variant moves passive planes per thread (a spawn), every later plain tick uses the
    88 KB passive double buffer: that launch needs its own shared-memory opt-in and occupancy."""
    eng, orc, cols = _extra_pair(RENDER_SIDE, 3000, spawn_rate=25, spawn_ttl=9)
    info, vectors = _synctest_vectors(16, 3, 8, spawn_ticks=(0, 7))
    kernels = _run_vectors(eng, orc, cols, info, vectors)
    assert all(k.kind == "bundle" and k.mode == 1 for k in kernels)
    assert not kernels[0].passive_tma and not kernels[7].passive_tma   # the spawning vectors
    assert kernels[1].passive_tma and kernels[-1].passive_tma
    assert eng.row_count() == 3000 + 2 * 25


def test_first_vector_with_two_loads_then_plain_ticks_with_a_large_passive_buffer():
    """The same with a catch-up vector first: five SyncTest ticks of check distance 1 in one request vector hold three
    Loads (no passive TMA), the single-tick vectors after it one leading Load each (passive TMA)."""
    eng, orc, cols = _extra_pair(RENDER_SIDE, 3000)
    info, vectors = _synctest_vectors(14, 1, 8)
    kernels = _run_vectors(eng, orc, cols, info, vectors, merge_first=5)
    assert all(k.kind == "bundle" for k in kernels)
    assert not kernels[0].passive_tma and all(k.passive_tma for k in kernels[1:])


def test_passive_runs_at_their_maximum():
    """Three active blocks (translation, velocity, ttl) split the passive planes into at most four runs: extra columns
    before, between and after them give exactly four TMA bulk copies per tile.  (kMaxRuns = 8 cannot be exceeded by
    this bundle, so the per-thread fallback for too many runs is unreachable.)"""
    layout = [("A", 8, COPY), "T", ("B", 4, CLONE), "V", ("C", 12, COPY), "L", ("D", 3, COPY)]
    eng, orc, cols = _extra_pair(layout, 2500, spawn_rate=0)
    info, vectors = _synctest_vectors(12, 3, 8)
    kernels = _run_vectors(eng, orc, cols, info, vectors)
    assert all(k.kind == "bundle" and k.passive_tma for k in kernels[1:])


@pytest.mark.parametrize("planes", [64, 65])
def test_passive_plane_limit(planes):
    """The Transform's 7 passive planes + one wide extra column.  64 passive planes (kMaxPassive) still run the bundle,
    with per-thread passive copies (2 x 128 KB does not fit shared memory); 65 are refused by the bundle.  That row is
    73 words wide: too wide for the generic one-launch program (tile > 100 KB; spawn_particles has no generic
    implementation either) and for two TMA stages, so it runs stepwise on k_checksum_column + k_copy_image."""
    layout = ["T", "V", "L", ("Wide", 4 * (planes - 7), COPY)]
    eng, orc, cols = _extra_pair(layout, 1500, spawn_rate=10, spawn_ttl=5)
    info, vectors = _synctest_vectors(10, 3, 8, spawn_ticks=(2,))
    kernels = _run_vectors(eng, orc, cols, info, vectors)
    if planes == 64:
        assert all(k.kind == "bundle" and k.mode == 1 and not k.passive_tma for k in kernels)
    else:
        assert all(k.kind == "stepwise_flat" for k in kernels)


def test_optional_column_runs_mode2():
    """An optional column selects the presence-aware variant (MODE 2, 2 rows per thread)."""
    eng, orc, cols = _extra_pair(["T", "V", "L", ("Tag", 4, COPY | capi.BGR_STRATEGY_OPTIONAL)], 2000)
    info, vectors = _synctest_vectors(10, 3, 8)
    kernels = _run_vectors(eng, orc, cols, info, vectors)
    assert all((k.kind, k.vec, k.mode) == ("bundle", 2, 2) for k in kernels)


# ---------------------------------------------------------------------------------------------------------------------
# knobs, one at a time
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [SINGLE_WAVE, MULTI_WAVE])
@pytest.mark.parametrize("knob,value", [("BGR_TUNE_PASSIVE_TMA", "0"), ("BGR_TUNE_PREFETCH", "0"),
                                        ("BGR_TUNE_PASSIVE_EARLY", "0"), ("BGR_TUNE_PASSIVE_EARLY", "1"),
                                        ("BGR_TUNE_STAGGER_NS", "0")])
def test_knob_matches_the_oracle(monkeypatch, knob, value, n):
    monkeypatch.setenv(knob, value)
    big = n == MULTI_WAVE
    r = run_particles_synctest_pair(n, 2 if big else 4, 6 if big else 12, seed=71, ttl_lo=2, ttl_hi=20,
                                    z_fraction=0.2, peek_check=not big)
    k = r["kernel"]
    assert k.kind == "bundle" and k.mode == 1
    assert k.passive_tma == (knob != "BGR_TUNE_PASSIVE_TMA")
    _assert_parity(r, peek=not big)


@pytest.mark.parametrize("knob,value", [("BGR_TUNE_POLL", "0")])
def test_knob_with_four_submits_in_flight(monkeypatch, knob, value):
    """collect() waiting on the event instead of polling the result block, with four request vectors queued and spawns
    changing the tile range."""
    monkeypatch.setenv(knob, value)
    eng, orc, cols = _extra_pair(["T", "V", "L"], 5000, spawn_rate=40, spawn_ttl=7, seed=9)
    info, vectors = _synctest_vectors(24, 3, 8, spawn_ticks=(1, 2, 11), input_delay=2)
    got, want, inflight = [], [], 0
    for v in vectors:
        eng.submit_requests(info, v)
        inflight += 1
        if inflight == 4:
            got += eng.collect()
            inflight -= 1
        want += orc.handle_requests(info, v)
    while inflight:
        got += eng.collect()
        inflight -= 1
    assert got == want and len(got) > 24
    k = eng.last_kernel()
    assert k.kind == "bundle" and k.mode == 1
    rows = eng.row_count()
    assert rows == orc.row_count() > 5000
    assert compare_state(eng, orc, cols, rows)
    assert eng.snapshot_frames() == orc.snapshot_frames()
    eng.close(); orc.close()
