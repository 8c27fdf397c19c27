"""-m gpu: growable worlds (BGR_CFG_GROWABLE).

Every case runs one script twice: on an engine created with BGR_CFG_GROWABLE for a small initial capacity, which the
script's spawns grow, and on its twin, the same registration and flags without BGR_CFG_GROWABLE, created with the
capacity the growable engine ended at.  Growth moves no byte, so every observation must be equal: checksums, the
kernel that ran, launch counts, row and active counts, the stored-unit counts of the launch trace (which show that the
content stamps survived), snapshots, change-feed reports and desync reports.  Worlds stay well under 2 GB."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import P2PTraceSession, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
GROW = capi.BGR_CFG_GROWABLE
ONE_WAVE_ROWS = 3 * 132 * 512  # the bundle runs its instance without stamps up to three tiles per SM


def _norm(x):
    """An observation as plain comparable values (arrays and C structs by their bytes)."""
    if isinstance(x, np.ndarray):
        return ("nd", x.dtype.str, x.shape, x.tobytes())
    if isinstance(x, C.Structure):
        return bytes(memoryview(x))
    if dataclasses.is_dataclass(x):
        return _norm(vars(x))
    if isinstance(x, dict):
        return tuple((k, _norm(v)) for k, v in sorted(x.items()))
    if isinstance(x, (list, tuple)):
        return tuple(_norm(v) for v in x)
    return x


def _twins(make, script, cap0=1024, flags=0, depth=9, min_growths=1):
    """script(engine, cols, caps) -> observations, on the growable engine and then on its twin.  `caps` collects the
    capacity after each step on the growable engine (not compared).  Returns the growable engine's capacities."""
    g = Engine(max_entities=cap0, max_depth=depth, flags=flags | GROW)
    cols = make(g)
    caps = [g.capacity()[0]]
    obs_g = _norm(script(g, cols, caps))
    final, ceiling = g.capacity()
    assert ceiling >= final
    g.close()
    f = Engine(max_entities=final, max_depth=depth, flags=flags)
    obs_f = _norm(script(f, make(f), []))
    assert f.capacity() == (final, final)
    f.close()
    growths = len(set(caps)) - 1
    assert growths >= min_growths, caps
    for i, (a, b) in enumerate(zip(obs_g, obs_f)):
        assert a == b, f"observation {i} differs"
    assert len(obs_g) == len(obs_f)
    return caps


# ---- worlds ----
def _particles(mode, n=1000, rate=4096):
    """The particles bundle with spawn_particles: MODE 1 (the example's registration) or MODE 2 (Velocity optional)."""
    def make(w):
        if mode == 2:
            t = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
            v = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY | OPT)
            l = w.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY)
            w.checksum_component(v, 0, 12, FIN)
            w.checksum_component(t, 0, 12, FIN)
            w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
            w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
            w.add_system(capi.BGR_SYS_PARTICLES_SPAWN, [t, v, l], [rate, 200, 123, 0])
            cols = (t, v, l)
        else:
            cols = register_particles(w, spawn_rate=rate, spawn_ttl=200)
        w.build()
        populate(w, cols, *synth_particles(n, 17, 4, 400, z_fraction=0.2))
        if mode == 2:
            for r in range(0, n, 13):
                w.remove_component(cols[1], r)
        return cols
    return make


def _scores(n=600):
    """A presence world the bundle does not cover: Score (optional, +1 per frame), Health (optional, despawns at 0),
    Tag (checksummed, untouched)."""
    def make(w):
        score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
        health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
        tag = w.rollback_component("Tag", 12, capi.BGR_STRATEGY_COPY)
        for c, ln in ((score, 4), (tag, 12), (health, 4)):
            w.checksum_component(c, 0, ln)
        w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
        w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
        w.build()
        _populate_scores(w, (score, health, tag), n, seed=5)
        return (score, health, tag)
    return make


def _populate_scores(w, cols, count, seed):
    score, health, tag = cols
    first = w.spawn(count)
    rng = np.random.default_rng(seed)
    w.write_component(score, first, rng.integers(0, 1000, count, dtype=np.uint32))
    w.write_component(health, first, rng.integers(3, 400, count, dtype=np.uint32))
    w.write_component(tag, first, rng.integers(0, 2**32, (count, 3), dtype=np.uint32))
    for r in range(first, first + min(count, 4000), 17):
        w.remove_component(score, r)


def _session(kind, seed=0xB200):
    return SyncTestSession(2, 7, 8, input_delay=2) if kind == "synctest" else P2PTraceSession(2, 8, 2, seed=seed)


def _tick(w, sess, inputs, kind):
    for h in range(2):
        sess.add_local_input(h, inputs[h])
    reqs = sess.advance_frame()
    out = w.handle_requests(sess.info(), reqs)
    for f, c in out:
        sess.save_cell(f, c if kind == "p2p" else 0)
    return out


def _snapshots(w, cols):
    n = w.row_count()
    return [(f, [w.peek(f, c, 0, n) for c in cols]) for f in w.snapshot_frames()]


def _live(w, cols):
    n = w.row_count()
    return [w.read_component(c, 0, n) for c in cols] + [w.read_alive(0, n)]


# ---- 1. the particles bundle, spawning ----
@pytest.mark.parametrize("kind", ["synctest", "p2p"])
@pytest.mark.parametrize("mode", [1, 2])
def test_particles_bundle_spawning_grows_and_matches_the_twin(kind, mode):
    """From 1024 rows past the one-wave size: both instances of k_particles_program run, the capacity grows at least
    four times, and every tick equals the twin's."""
    def script(w, cols, caps):
        w.trace_enable(256)
        sess = _session(kind)
        obs, kernels = [], set()
        for t in range(80):
            pressed = capi.BGR_INPUT_SPAWN if t < 70 else 0
            l0 = w.launch_count()
            out = _tick(w, sess, (pressed, 0), kind)
            k = w.last_kernel()
            kernels.add(k.stable_planes)
            obs.append((out, k.raw, w.launch_count() - l0, w.row_count(), w.active_count()))
            caps.append(w.capacity()[0])
        assert kernels == {False, True}  # the unstamped (one-wave) and the stamped instance both ran
        assert w.row_count() > ONE_WAVE_ROWS
        obs.append(w.trace_read(256)[:, 3])
        obs.append(_snapshots(w, cols))
        return obs
    _twins(_particles(mode), script, min_growths=4)


# ---- 2. / 3. the generic program and the stepwise path, growing through bgr_spawn ----
def _spawning_scores_script(w, cols, caps, ticks=24):
    sess = _session("synctest")
    score, health, tag = cols
    obs = []
    for t in range(ticks):
        obs.append(_tick(w, sess, ((t * 7) & 0xF, 3), "synctest"))
        obs.append((w.last_kernel().raw, w.row_count()))
        if t % 6 == 2:  # between ticks: the next tick's Load goes back to a frame saved before this growth (and its
            # rows, which no snapshot holds, go with it: each spawn needs more rows than the last)
            _populate_scores(w, cols, 60_000 << (t // 6), seed=t)
            w.insert_component(score, 17, np.array([99], np.uint32))
            w.remove_component(health, 5 + t)
        caps.append(w.capacity()[0])
    obs.append(_snapshots(w, cols))
    obs.append(_live(w, cols))
    return obs


def test_generic_program_grows_through_spawn(generic_kernel):
    _twins(_scores(), _spawning_scores_script, min_growths=3)


@pytest.mark.parametrize("tma", ["1", "0"])
def test_stepwise_path_grows_through_spawn(monkeypatch, tma):
    monkeypatch.setenv("BGR_TUNE_TMA", tma)
    _twins(_scores(), _spawning_scores_script, flags=capi.BGR_CFG_FORCE_STEPWISE, min_growths=3)


# ---- 4. queued submits ----
def _queued_script(grow, ticks=24, in_flight=4):
    """Request vectors submitted `in_flight` ahead of their collection; `grow(w, t)` runs between two submits."""
    def script(w, cols, caps):
        sess = _session("p2p")
        queued, obs = 0, []
        for t in range(ticks):
            for h in range(2):
                sess.add_local_input(h, capi.BGR_INPUT_SPAWN if (h == 0 and t >= 8) else 0)
            reqs = sess.advance_frame()
            w.submit_requests(sess.info(), reqs)
            queued += 1
            grow(w, t)
            caps.append(w.capacity()[0])
            if queued > in_flight:
                obs.append(w.collect())
                queued -= 1
        while queued:
            obs.append(w.collect())
            queued -= 1
        obs.append((w.row_count(), w.active_count()))
        obs.append(_snapshots(w, cols))
        return obs
    return script


def test_queued_submits_bundle_growth_inside_the_fifth_vector():
    """Four vectors in flight; the spawns of later ones force growths (default tile dependencies on the bundle)."""
    _twins(_particles(1, rate=4096), _queued_script(lambda w, t: None), min_growths=2)


def test_queued_submits_generated_kernel_with_tile_dependencies(monkeypatch):
    """The generated kernel with BGR_TUNE_JIT_TILEDEP=1: four vectors in flight while bgr_reserve grows the engine."""
    monkeypatch.setenv("BGR_TUNE_JIT", "2")
    monkeypatch.setenv("BGR_TUNE_JIT_TILEDEP", "1")

    def grow(w, t):
        if t in (6, 13):
            w.reserve(150_000 * (t // 6))

    _twins(_scores(5000), _queued_script(grow), min_growths=2)


# ---- 5. the deferred live image pending at a growth ----
@pytest.mark.parametrize("how", ["spawn", "reserve"])
def test_deferred_live_image_pending_at_a_growth(how):
    resumed = []

    def script(w, cols, caps):
        sess = _session("p2p")
        obs = []
        for t in range(30):
            obs.append(_tick(w, sess, (0, 0), "p2p"))
            k = w.last_kernel()
            obs.append(k.raw)
            if t in (10, 20):
                assert k.deferred_live
                if how == "spawn":
                    w.spawn(40_000 * (t // 10))    # materialises image 0, then grows and appends
                    obs.append(_live(w, cols))
                else:
                    w.reserve(80_000 * (t // 10))  # image 0 stays pending: the next vector starts from the base slot
            if t in (11, 21):
                resumed.append(k.from_deferred)
            caps.append(w.capacity()[0])
        obs.append(_live(w, cols))
        obs.append(_snapshots(w, cols))
        return obs
    _twins(_particles(1, rate=64), script, min_growths=2)
    if how == "reserve":  # a vector that did not start with its own Load started from the pending image's base slot
        assert any(resumed)


# ---- 6. desync capture and retention across a growth ----
def test_desync_reports_of_frames_saved_before_a_growth():
    def script(w, cols, caps):
        sess = _session("synctest")
        obs = []
        for t in range(24):
            obs.append(_tick(w, sess, (capi.BGR_INPUT_SPAWN if t % 3 == 0 else 0, 0), "synctest"))
            if t in (8, 16):
                frames = w.snapshot_frames()
                w.reserve(60_000 * (t // 8))
                for f in frames:
                    d = w.frame_digest(f)
                    obs.append((f, w.desync_diff(f), d))
                    if d is not None:
                        obs.append(w.export_blocks(f, list(range(d[0].n_blocks))))
            caps.append(w.capacity()[0])
        return obs
    _twins(_particles(2, rate=512), script, flags=capi.BGR_CFG_DESYNC_CAPTURE, min_growths=2)


# ---- 7. a change feed created before the growth ----
def test_change_feed_created_before_the_growth_reports_as_the_twin():
    def script(w, cols, caps):
        t_, v, l = cols
        fields = [(t_, 0, 12), (v, 0, 8), (l, 0, 8)]
        feed = w.feed_create(fields)
        cap = 400_000
        buf = w.feed_alloc(feed, cap)
        sess = _session("p2p")
        obs = []
        for t in range(40):
            obs.append(_tick(w, sess, (capi.BGR_INPUT_SPAWN if t < 30 else 0, 0), "p2p"))
            recs, info = w.feed_wait(w.feed_begin(feed, buf, cap))
            obs.append((recs, info))
            caps.append(w.capacity()[0])
        return obs
    _twins(_particles(1, rate=4096), script, min_growths=3)


# ---- 8. the generated kernel compiled when a growth crosses the JIT threshold ----
def test_growth_past_the_jit_threshold_compiles_the_generated_kernel(monkeypatch):
    monkeypatch.setenv("BGR_TUNE_JIT", "2")
    probe = Engine(max_entities=32, flags=0)
    _scores(16)(probe)
    monkeypatch.delenv("BGR_TUNE_JIT")  # the default: engines of >= 16384 rows compile the generated kernel
    nvrtc = probe.generic_specialised()
    probe.close()
    if not nvrtc:
        pytest.skip("NVRTC is not available: the interpreter kernel runs everywhere")

    def script(w, cols, caps):
        sess = _session("synctest")
        obs = []
        for t in range(12):
            obs.append(_tick(w, sess, (t & 3, 0), "synctest"))
            if t == 4:
                if w.capacity()[0] < 16384:
                    assert not w.generic_specialised()
                _populate_scores(w, cols, 20_000, seed=t)
            caps.append(w.capacity()[0])
        assert w.generic_specialised()
        assert w.last_kernel().kind == "generic_nvrtc"
        obs.append(_snapshots(w, cols))
        return obs
    _twins(_scores(1000), script, cap0=4096)


# ---- 9. errors and limits ----
def test_reserve_capacity_and_refusals():
    e = Engine(max_entities=1000, flags=GROW)
    _scores(100)(e)
    cap, ceiling = e.capacity()
    assert cap == 1000 and ceiling >= cap
    e.reserve(0)
    e.reserve(cap)
    assert e.capacity() == (cap, ceiling)            # at or below the capacity: no-op
    e.reserve(cap + 1)
    grown = e.capacity()[0]
    assert grown >= 2 * cap and grown % 512 == 0
    e.close()

    f = Engine(max_entities=1000)
    _scores(100)(f)
    assert f.capacity() == (1000, 1000)
    f.reserve(1000)
    with pytest.raises(BgrError) as ei:
        f.reserve(1001)
    assert ei.value.status == capi.BGR_ERR_UNSUPPORTED
    f.close()

    for flags, base in ((GROW | capi.BGR_CFG_SHARDED, 0), (GROW, 4096)):
        with pytest.raises(BgrError) as ei:
            Engine(max_entities=1000, flags=flags, order_base=base)
        assert ei.value.status == capi.BGR_ERR_UNSUPPORTED


def test_calls_past_the_ceiling_fail_and_change_nothing():
    """A wide schema with many frame slots has a small ceiling; the ceiling check maps nothing."""
    e = Engine(max_entities=512, max_depth=32, flags=GROW | capi.BGR_CFG_DESYNC_CAPTURE)
    cols = [e.rollback_component(f"Wide{i}", 1024) for i in range(16)]
    e.checksum_component(cols[0], 0, 16)
    e.build()
    e.spawn(100)
    cap, ceiling = e.capacity()
    assert cap == 512 and ceiling < (1 << 24)
    sess = _session("synctest")
    before = [_tick(e, sess, (0, 0), "synctest") for _ in range(3)]
    for call in (lambda: e.reserve(ceiling + 1), lambda: e.spawn(ceiling)):
        with pytest.raises(BgrError) as ei:
            call()
        assert ei.value.status == capi.BGR_ERR_CAPACITY
        assert e.capacity() == (cap, ceiling) and e.row_count() == 100
    after = [_tick(e, sess, (0, 0), "synctest") for _ in range(3)]  # the engine keeps ticking
    assert len(before) == len(after) == 3
    e.close()
