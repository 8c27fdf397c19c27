"""-m gpu: the bundle kernel's TMA path for passive planes, on the ticks that take it.

Passive planes move only when their content changed (engine.cu HostState): a plain steady-state tick launches the
passive-TMA configuration but moves no passive plane, so test_gpu_bundle_variants no longer sees the bulk copies run.
A host write of Transform.rotation bumps the content version, and the next plain tick stages the passive planes through
TMA and stores them into the slots it saves.  Each case bumps the version before the ticks it checks, asserts through
Engine.last_kernel() that the variant it names ran and that it moved passive planes (BGR_KERNEL_PASSIVE_PLANES), and
compares checksums after every vector, the live state, ring frames and snapshot bytes with the oracle."""
import numpy as np
import pytest

from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld
from parity_util import compare_state
from test_gpu_bundle_variants import (CLONE, COPY, MODE0_SETUPS, MODE1, MULTI_WAVE, RENDER_SIDE, SINGLE_WAVE,
                                      _extra_pair, _synctest_vectors)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


def _write_rotation(eng, orc, t, rows, seed):
    """The host rewrites Transform.rotation of every row (translation and scale kept) on both worlds."""
    vals = eng.read_component(t, 0, rows).view(np.float32).copy()
    vals[:, 3:7] = np.random.default_rng(seed).uniform(-1.0, 1.0, (rows, 4))
    for w in (eng, orc):
        w.write_component(t, 0, vals)


def _run(eng, orc, cols, t, info, vectors, bump, merge_first=1):
    """Like test_gpu_bundle_variants' runner; the version is bumped before every engine vector whose index is in `bump`."""
    kernels = []
    groups = [vectors[:merge_first]] + [[v] for v in vectors[merge_first:]]
    for i, g in enumerate(groups):
        if i in bump:
            _write_rotation(eng, orc, t, eng.row_count(), i)
        got = eng.handle_requests(info, [r for v in g for r in v])
        want = [c for v in g for c in orc.handle_requests(info, v)]
        assert got == want, i
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
    eng.close(); orc.close()
    return kernels


def _particles_after_a_bump(n, checksums, seed):
    """The particles world (single- or multi-wave grid); the version is bumped before the last three ticks."""
    big = n == MULTI_WAVE
    d, ticks = (2, 8) if big else (4, 12)
    eng, orc = Engine(max_entities=n, max_depth=8), OracleWorld()
    for w in (eng, orc):
        cols = register_particles(w, checksums=checksums)
        w.build()
        populate(w, cols, *synth_particles(n, seed, 2, 20, z_fraction=0.2))
    info, vectors = _synctest_vectors(ticks, d, 8, input_delay=2)
    return _run(eng, orc, cols, cols[0], info, vectors, bump=(ticks - 3, ticks - 1))


@pytest.mark.parametrize("n", [SINGLE_WAVE, MULTI_WAVE])
@pytest.mark.parametrize("mode", [0, 1])
def test_every_vec_tier_mode_instantiation_after_a_host_write(mode, n):
    kernels = _particles_after_a_bump(n, MODE1 if mode else MODE0_SETUPS["both_plain"], 22)
    for k in (kernels[-3], kernels[-1]):
        assert k.kind == "bundle" and (k.vec, k.mode, k.tier, k.item_rows) == (2, mode, 1, 512)
        assert k.passive_tma and k.passive_planes   # the example's layout: the Transform's 7 passive planes are one TMA run


@pytest.mark.parametrize("n", [SINGLE_WAVE, MULTI_WAVE])
@pytest.mark.parametrize("knob,value", [("BGR_TUNE_PASSIVE_TMA", "0"), ("BGR_TUNE_PREFETCH", "0"),
                                        ("BGR_TUNE_PASSIVE_EARLY", "0"), ("BGR_TUNE_PASSIVE_EARLY", "1"),
                                        ("BGR_TUNE_STAGGER_NS", "0")])
def test_knob_after_a_host_write_matches_the_oracle(monkeypatch, knob, value, n):
    monkeypatch.setenv(knob, value)
    kernels = _particles_after_a_bump(n, None, 71)
    for k in (kernels[-3], kernels[-1]):
        assert k.kind == "bundle" and k.mode == 1
        assert k.passive_planes and k.passive_tma == (knob != "BGR_TUNE_PASSIVE_TMA")


def test_spawn_vectors_then_bumped_plain_ticks_with_a_large_passive_buffer():
    """The first launch of the kernel variant moves passive planes per thread (a spawn); plain ticks after a host write
    use the 88 KB passive double buffer: that launch needs its own shared-memory opt-in and occupancy."""
    eng, orc, cols = _extra_pair(RENDER_SIDE, 3000, spawn_rate=25, spawn_ttl=9)
    info, vectors = _synctest_vectors(16, 3, 8, spawn_ticks=(0, 7))
    kernels = _run(eng, orc, cols, cols[1], info, vectors, bump=(1, 15))
    assert all(k.kind == "bundle" and k.mode == 1 for k in kernels)
    assert not kernels[0].passive_tma and not kernels[7].passive_tma   # the spawning vectors: per thread
    assert all(kernels[i].passive_planes for i in (0, 1, 7, 15))
    assert kernels[1].passive_tma and kernels[15].passive_tma


def test_two_load_vector_then_bumped_plain_ticks_with_a_large_passive_buffer():
    """A catch-up vector first (five SyncTest ticks of check distance 1: three Loads, no passive TMA), then single-tick
    vectors with one leading Load each, which stage the passive planes by TMA after a host write."""
    eng, orc, cols = _extra_pair(RENDER_SIDE, 3000)
    info, vectors = _synctest_vectors(14, 1, 8)
    kernels = _run(eng, orc, cols, cols[1], info, vectors, bump=(1, 5, 9), merge_first=5)
    assert all(k.kind == "bundle" for k in kernels)
    assert not kernels[0].passive_tma and all(kernels[i].passive_tma and kernels[i].passive_planes for i in (1, 5, 9))


def test_passive_runs_at_their_maximum_after_a_host_write():
    """Three active blocks (translation, velocity, ttl) split the passive planes into four runs: extra columns before,
    between and after them give exactly four TMA bulk copies per tile on a tick that stages them."""
    layout = [("A", 8, COPY), "T", ("B", 4, CLONE), "V", ("C", 12, COPY), "L", ("D", 3, COPY)]
    eng, orc, cols = _extra_pair(layout, 2500, spawn_rate=0)
    info, vectors = _synctest_vectors(12, 3, 8)
    kernels = _run(eng, orc, cols, cols[1], info, vectors, bump=(1, 6, 11))
    assert all(k.kind == "bundle" for k in kernels)
    assert all(kernels[i].passive_tma and kernels[i].passive_planes for i in (1, 6, 11))
