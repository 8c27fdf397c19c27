"""Replays (bgr_replay, Engine.replay): a recorded input log through a world in one call.  Every replay is held to the
request stream it stands for, run through bgr_handle_requests on a twin engine: [Save(f) at the checksum frames,
Advance] in vectors of at most BGR_MAX_REQUESTS.  The twin runs a spectator session, whose ring has depth 0, so its
Saves checksum and store nothing, as a replay's do.  Checksums, the live world (every column, alive and presence
bytes), the row count and the frame count must agree; ticking both on afterwards, with spawns, holds Time<GgrsTime>,
ParticleRng and the call counter to the stream too."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles

from test_gpu_batch import box_world, presence_world

pytestmark = pytest.mark.gpu
SPECTATOR = (capi.BGR_SESSION_SPECTATOR, 0, 0, 0)
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32


def counter_world(n, depth=4, flags=0):
    """Two call-count systems and a U32_ADD on an optional column: the counter reaches the checksums."""
    w = Engine(max_entities=n + 8, max_depth=depth, flags=flags)
    a = w.rollback_component("A", 4, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)
    b = w.rollback_component("B", 8, capi.BGR_STRATEGY_COPY)
    w.checksum_component(a, 0, 4)
    w.checksum_component(b, 0, 8)
    w.add_system(capi.BGR_SYS_U32_STORE_CALL_COUNT, [b], [0])
    w.add_system(capi.BGR_SYS_U32_ADD, [a], [0, 3])
    w.add_system(capi.BGR_SYS_U32_STORE_CALL_COUNT, [b], [4])
    w.build()
    w.spawn(n)
    w.write_component(a, 0, np.arange(n, dtype=np.uint32))
    for r in range(0, n, 7):
        w.remove_component(a, r)
    return w


def particles_world(n, rate=5, ttl=40, flags=0, cap=None, bundle=True, depth=4):
    """The particles example with spawn_particles; bundle=False registers a whole-Transform checksum, which the
    particles bundle does not take (the generic program runs it)."""
    w = Engine(max_entities=cap or n + rate * 400, max_depth=depth, flags=flags)
    ck = None if bundle else (lambda e, t, v: (e.checksum_component(t, 0, 40, FIN), e.checksum_component(v, 0, 12)))
    c = register_particles(w, spawn_rate=rate, spawn_ttl=ttl, rng_seed=0xC0FFEE, checksums=ck)
    w.build()
    populate(w, c, *synth_particles(n, 3, 2, 60, 0.2))
    return w


MAKERS = {
    "box": lambda: box_world(700, 4),
    "presence": lambda: presence_world(1300, 4),
    "counter": lambda: counter_world(600),
    "particles_bundle": lambda: particles_world(900),
    "particles_generic": lambda: particles_world(900, bundle=False),
}


def log_for(n_frames, n_players, seed, spawn_every=0):
    rng = np.random.default_rng(seed)
    log = rng.integers(0, 16, (n_frames, n_players), dtype=np.uint8)  # box_game's four direction bits
    if spawn_every:
        log[::spawn_every, 0] |= capi.BGR_INPUT_SPAWN
    return log


def stream_of(f0, log, k):
    """The request stream a replay stands for, in vectors of at most BGR_MAX_REQUESTS requests."""
    vecs, cur = [], []
    for j, row in enumerate(log):
        reqs = ([Request(SAVE, f0 + j)] if k and (f0 + j) % k == 0 else []) + [Request(ADVANCE, 0, [int(v) for v in row])]
        if len(cur) + len(reqs) > capi.BGR_MAX_REQUESTS:
            vecs.append(cur)
            cur = []
        cur += reqs
    if cur:
        vecs.append(cur)
    return vecs


def run_stream(e, f0, log, k):
    out, status = [], capi.BGR_OK
    for v in stream_of(f0, log, k):
        try:
            out += e.handle_requests(SPECTATOR, v)
        except BgrError as err:
            assert err.status == capi.BGR_ERR_NON_FINITE
            status = err.status
    return out, status


def live(e):
    """The observable live world.  A dead row's bytes are not observable (only a Load brings a row back, with its
    bytes): the particles bundle advances dead rows where the generated kernel leaves them, and a checkpoint restore
    zeroes them."""
    n = e.row_count()
    alive = e.read_alive(0, n)
    out = [e.rollback_frame_count(), n, e.active_count(), alive.tobytes()]
    for c in range(len(e.elem_bytes)):
        v = np.ascontiguousarray(e.read_component(c, 0, n)).reshape(n, -1).view(np.uint8).copy()
        v[alive == 0] = 0
        out.append(v.tobytes())
        out.append(e.has_component(c, 0, n).tobytes())
    return out


def tick_on(e, frames=12):
    """Frames after the replay through the request path: Time<GgrsTime>, ParticleRng and the counter show in them."""
    f = e.rollback_frame_count()
    log = log_for(frames, 2, 99, spawn_every=3)
    return run_stream(e, f, log, 1)[0]


def replay(e, log, k):
    try:
        return e.replay(log, k), capi.BGR_OK
    except BgrError as err:
        assert err.status == capi.BGR_ERR_NON_FINITE
        return str(err), err.status


@pytest.mark.parametrize("f0", [0, 7])
@pytest.mark.parametrize("k", [0, 1, 10, 1000])
@pytest.mark.parametrize("name", list(MAKERS))
def test_replay_equals_the_request_stream(name, k, f0):
    a, b = MAKERS[name](), MAKERS[name]()
    for e in (a, b):
        if f0:
            e.set_rollback_frame_count(f0)
    log = log_for(230, 2, seed=len(name) + k, spawn_every=11)
    got, st = replay(a, log, k)
    want, wst = run_stream(b, f0, log, k)
    assert st == wst == capi.BGR_OK
    assert got == want
    assert len(got) == sum(1 for j in range(230) if k and (f0 + j) % k == 0)
    assert a.last_kernel().replay
    assert live(a) == live(b)
    assert tick_on(a) == tick_on(b)
    assert live(a) == live(b)


def test_fast_path_is_byte_identical_to_the_chunked_fallback(monkeypatch):
    log = log_for(300, 2, seed=5, spawn_every=13)  # more than 80 frames, more than 40 checksum points
    fast = [particles_world(1500, bundle=False), counter_world(900)]
    monkeypatch.setenv("BGR_TUNE_JIT", "0")
    slow = [particles_world(1500, bundle=False), counter_world(900)]
    bundle_twin = particles_world(1500, bundle=True)  # the bundle engine's own fallback runs the bundle kernel
    monkeypatch.delenv("BGR_TUNE_JIT")
    bundle_fast = particles_world(1500, bundle=True)
    for f, s in zip(fast, slow):
        assert f.replay(log, 1) == s.replay(log, 1)
        assert f.last_kernel().replay and not s.last_kernel().replay
        assert live(f) == live(s)
    assert bundle_fast.replay(log, 1) == bundle_twin.replay(log, 1)
    assert bundle_fast.last_kernel().replay and bundle_twin.last_kernel().kind == "bundle"
    assert live(bundle_fast) == live(bundle_twin)


@pytest.mark.parametrize("name", ["box", "particles_generic", "counter"])
def test_two_replays_equal_one(name):
    a, b = MAKERS[name](), MAKERS[name]()
    log = log_for(500, 2, seed=11, spawn_every=7)
    one = a.replay(log, 10)
    two = b.replay(log[:123], 10) + b.replay(log[123:], 10)
    assert one == two
    assert live(a) == live(b)


def test_ring_and_rollback_across_a_replay():
    e = particles_world(800, bundle=False, depth=6)
    e.set_depth(6)
    saved = []
    for f in range(4):  # a few snapshots in the ring
        saved += e.handle_requests((capi.BGR_SESSION_NONE, 0, 0, 0), [Request(SAVE, f), Request(ADVANCE, 0, [1, 2])])
    before, frames, rows = live(e), e.snapshot_frames(), e.row_count()
    f_load = e.rollback_frame_count()
    e.handle_requests((capi.BGR_SESSION_NONE, 0, 0, 0), [Request(SAVE, f_load)])
    frames = e.snapshot_frames()
    e.replay(log_for(150, 2, seed=2, spawn_every=5), 10)
    assert e.snapshot_frames() == frames
    assert e.row_count() > rows
    e.handle_requests((capi.BGR_SESSION_NONE, 0, 0, 0), [Request(LOAD, f_load)])
    assert live(e) == before


def test_change_feed_reports_exactly_the_replayed_rows():
    a, b = box_world(600, 4), box_world(600, 4)
    fa, fb = a.feed_create([(1, 0, 12)]), b.feed_create([(1, 0, 12)])
    for e, fd in ((a, fa), (b, fb)):
        e.feed_wait(e.feed_begin(fd, e.feed_alloc(fd, 700), 700))
    log = log_for(90, 2, seed=4)
    a.replay(log, 10)
    run_stream(b, 0, log, 10)
    ra, ia = a.feed_wait(a.feed_begin(fa, a.feed_alloc(fa, 700), 700))
    rb, ib = b.feed_wait(b.feed_begin(fb, b.feed_alloc(fb, 700), 700))
    assert ia.n_records == ib.n_records > 0
    assert ra[: ia.n_records].tobytes() == rb[: ib.n_records].tobytes()


def test_growable_engine_grows_and_fixed_engine_refuses():
    g = particles_world(500, rate=40, cap=520, flags=capi.BGR_CFG_GROWABLE, bundle=False)
    ref = particles_world(500, rate=40, bundle=False)
    log = log_for(120, 2, seed=8, spawn_every=4)
    assert g.replay(log, 10) == ref.replay(log, 10)
    assert g.capacity()[0] >= g.row_count() == ref.row_count() == 500 + 40 * 30
    assert live(g) == live(ref)
    fixed = particles_world(500, rate=40, cap=520, bundle=False)
    before = live(fixed)
    with pytest.raises(BgrError) as ei:
        fixed.replay(log, 10)
    assert ei.value.status == capi.BGR_ERR_CAPACITY
    assert live(fixed) == before


@pytest.mark.parametrize("k", [1, 10])
def test_non_finite_checksum_frame(k):
    a, b = box_world(300, 4), box_world(300, 4)
    for e in (a, b):
        t = np.ascontiguousarray(e.read_component(1, 0, 1)).view(np.float32).copy()
        t.reshape(-1)[0] = np.nan  # a NaN translation stays NaN: every checksum frame is non-finite
        e.write_component(1, 0, t)
    log = log_for(60, 2, seed=1)
    text, st = replay(a, log, k)
    want, wst = run_stream(b, 0, log, k)
    assert st == wst == capi.BGR_ERR_NON_FINITE
    assert "frame 0)" in text
    assert live(a) == live(b)
    assert tick_on(a) == tick_on(b)


def test_refusals_change_nothing():
    e = box_world(200, 4)
    before = live(e)
    lib, h = e._lib, e._h
    import ctypes as C
    n = C.c_uint32()
    out = (capi.bgr_checksum * 8)()
    log = np.zeros((10, 9), np.uint8)
    for r, status in ((capi.bgr_replay(10, 9, 1, 0, log.ctypes.data), capi.BGR_ERR_INVALID_ARGUMENT),
                      (capi.bgr_replay(10, 2, 1, 0, None), capi.BGR_ERR_INVALID_ARGUMENT),
                      (capi.bgr_replay(10, 2, 1, 1, log.ctypes.data), capi.BGR_ERR_INVALID_ARGUMENT),
                      (capi.bgr_replay(capi.BGR_MAX_REPLAY_FRAMES + 1, 0, 1, 0, None), capi.BGR_ERR_INVALID_ARGUMENT)):
        assert lib.bgr_replay(h, C.byref(r), out, 8, C.byref(n)) == status
        assert live(e) == before
    e.set_rollback_frame_count(2**31 - 5)
    with pytest.raises(BgrError) as ei:
        e.replay(np.zeros((10, 2), np.uint8), 1)
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    e.set_rollback_frame_count(0)
    assert live(e) == before
    e.submit_requests(SPECTATOR, [Request(ADVANCE, 0, [1, 2])])
    with pytest.raises(BgrError) as ei:
        e.replay(np.zeros((10, 2), np.uint8), 1)
    assert ei.value.status == capi.BGR_ERR_STATE
    e.collect()
    s = Engine(max_entities=64, flags=capi.BGR_CFG_SHARDED)
    vel = s.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    s.checksum_component(vel, 0, 12)
    s.build()
    with pytest.raises(BgrError) as ei:
        s.replay(np.zeros((4, 1), np.uint8), 1)
    assert ei.value.status == capi.BGR_ERR_UNSUPPORTED


def test_checkpoint_then_replay_verifies_a_match():
    """A P2P-style match checkpointed at frame F: a fresh engine restored from the checkpoint replays the rest of the
    log, and its checksums at the interval frames equal the live engine's Saves."""
    live_e = particles_world(1200, bundle=False, depth=8)
    log = log_for(400, 2, seed=21, spawn_every=9)
    k, F = 10, 130
    recorded = {}
    for j, row in enumerate(log):
        f = live_e.rollback_frame_count()
        info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))
        reqs = ([Request(SAVE, f)] if f % k == 0 or f == F else []) + [Request(ADVANCE, 0, [int(v) for v in row])]
        for fr, cs in live_e.handle_requests(info, reqs):
            recorded[fr] = cs
        if f == F:
            blob = live_e.checkpoint(F)
    assert blob is not None
    fresh = particles_world(1200, bundle=False, depth=8)
    fresh.restore(blob)
    assert fresh.rollback_frame_count() == F
    got = fresh.replay(log[F:], k)
    assert got == [(f, recorded[f]) for f in range(F, 400) if f % k == 0]
    assert live(fresh) == live(live_e)


def test_retained_frames_and_desync_witnesses_are_untouched():
    """A SyncTest engine with desync capture and retention of confirmed frames: the frames it keeps, and every byte
    of them, are the same after a replay."""
    from bevy_ggrs_b200.session import SyncTestSession
    e = Engine(max_entities=708, max_depth=9, flags=capi.BGR_CFG_DESYNC_CAPTURE)
    e.retain_confirmed(2, 4)
    vel = e.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    tf = e.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
    e.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
    e.checksum_component(tf, 0, 12, FIN)
    e.checksum_component(vel, 0, 12)
    e.build()
    e.spawn(700)
    rng = np.random.default_rng(3)
    t = np.zeros((700, 10), np.float32)
    t[:, 0:3] = rng.uniform(-2, 2, (700, 3)); t[:, 6] = 1.0; t[:, 7:10] = 1.0
    e.write_component(tf, 0, t)
    sess = SyncTestSession(2, 3, 8)
    for tick in range(16):
        for h in range(2):
            sess.add_local_input(h, (tick * 5 + 3 * h) % 16)
        for f, cs in e.handle_requests(sess.info(), sess.advance_frame()):
            sess.save_cell(f, cs)

    def kept():
        n = e.row_count()
        out = [e.snapshot_frames(), e.retained_frames(), e.desync_frames(), e.confirmed_frame_count()]
        for f in e.snapshot_frames():
            out.append([e.peek(f, c, 0, n)[0].tobytes() for c in (vel, tf)])
        for f in e.desync_frames():
            out.append([e.peek_first(f, c, 0, n)[0].tobytes() for c in (vel, tf)])
        return out
    before = kept()
    assert before[1] and before[2], "the setup keeps retained frames and desync witnesses"
    e.replay(log_for(120, 2, seed=6), 10)
    assert kept() == before


def test_growable_engine_refuses_spawns_past_its_ceiling():
    rate = 4096  # the largest rate spawn_particles takes
    e = particles_world(300, rate=rate, cap=400, flags=capi.BGR_CFG_GROWABLE, bundle=False)
    cap_before, ceiling = e.capacity()
    log = np.full((ceiling // rate + 2, 1), capi.BGR_INPUT_SPAWN, np.uint8)  # spawns past the ceiling
    assert log.shape[0] <= capi.BGR_MAX_REPLAY_FRAMES
    before = live(e)
    with pytest.raises(BgrError) as ei:
        e.replay(log, 10)
    assert ei.value.status == capi.BGR_ERR_CAPACITY
    assert live(e) == before and e.capacity() == (cap_before, ceiling)
