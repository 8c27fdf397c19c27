"""Replay keyframes (bgr_replay_keyframes, Engine.replay_keyframes; the batch call): a replay that also writes a world
checkpoint every K frames.  Each keyframe is held to bgr_checkpoint_save on a twin engine that ran the equivalent
request stream with a Save at that frame, byte for byte; the checksums, live world, Time<GgrsTime>, ParticleRng and the
call counter are held to a plain bgr_replay on a third twin.  Every test runs on the interpreter (the chunked
fallback), the generated kernel with whole tiles and with 128-row items."""
import ctypes as C

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine, EngineBatch
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles

from test_gpu_batch import box_world, presence_world
from test_gpu_generic_spawn import spawn_world, whole_transform
from test_gpu_replay import FIN, live, log_for, particles_world, tick_on

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]

MAKERS = {
    "box": lambda: box_world(700, 4),
    "presence": lambda: presence_world(1300, 4),
    "spawning_fixed": lambda: particles_world(900, rate=37, bundle=False),
    "spawning_growable": lambda: particles_world(500, rate=40, cap=520, flags=capi.BGR_CFG_GROWABLE, bundle=False),
    "stress_15_words": lambda: particles_world(1500),
}


def stream_blobs(e, f0, log, kk):
    """The keyframes of `log` by the request stream: at each keyframe frame a Save, then bgr_checkpoint_save.  A P2P
    session that confirms every frame before the current one keeps the ring from filling up."""
    blobs = []
    for j, row in enumerate(log):
        f = f0 + j
        info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))
        if f % kk == 0:
            try:
                e.handle_requests(info, [Request(SAVE, f)])
            except BgrError as err:  # a non-finite checksum: the Save still stored the frame
                assert err.status == capi.BGR_ERR_NON_FINITE
            blobs.append((f, e.checkpoint(f)))
        e.handle_requests(info, [Request(ADVANCE, 0, [int(v) for v in row])])
    return blobs


def expected_frames(f0, n, kk):
    return [f0 + j for j in range(n) if (f0 + j) % kk == 0]


@pytest.mark.parametrize("f0,n,k,kk", [(0, 150, 10, 10), (7, 150, 10, 25), (3, 40, 0, 1), (5, 60, 7, 200),
                                       (60, 130, 60, 60)])
@pytest.mark.parametrize("name", list(MAKERS))
def test_keyframes_equal_the_request_stream(name, f0, n, k, kk):
    a, b, c = MAKERS[name](), MAKERS[name](), MAKERS[name]()
    for e in (a, b, c):
        e.set_rollback_frame_count(f0)
    log = log_for(n, 2, seed=len(name) + kk, spawn_every=9)
    cs, kfs = a.replay_keyframes(log, k, kk)
    assert [f for f, _ in kfs] == expected_frames(f0, n, kk)
    assert kfs == stream_blobs(b, f0, log, kk)
    assert cs == c.replay(log, k)
    assert live(a) == live(c) == live(b)
    assert a.last_kernel().replay == c.last_kernel().replay
    assert tick_on(a) == tick_on(c)


def rate_world(n, fps, stream=None, seed=0, spawn_rate=0):
    """box_game (spawn_rate 0) or spawning particles at `fps`: Time<GgrsTime>'s step and the systems' dt follow it."""
    w = Engine(max_entities=n + 8 + spawn_rate * 64, max_depth=4, fps=fps, stream=stream)
    if spawn_rate:
        c = register_particles(w, spawn_rate=spawn_rate, spawn_ttl=11, rng_seed=0xC0FFEE + seed, checksums=whole_transform)
        w.build()
        populate(w, c, *synth_particles(n, seed, 2, 30, 0.2))
        return w
    vel = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    tf = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
    w.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
    w.checksum_component(tf, 0, 12, FIN)
    w.checksum_component(vel, 0, 12)
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(seed)
    t = np.zeros((n, 10), np.float32)
    t[:, 0:3] = rng.uniform(-2, 2, (n, 3)); t[:, 6] = 1.0; t[:, 7:10] = 1.0
    w.write_component(tf, 0, t)
    w.write_component(vel, 0, rng.uniform(-1, 1, (n, 3)).astype(np.float32))
    return w


@pytest.mark.parametrize("spawn_rate", [0, 13])
@pytest.mark.parametrize("fps", [7, 144])
def test_keyframes_of_a_restored_world_at_other_rates(fps, spawn_rate):
    """A keyframe replay from a restored world whose Time<GgrsTime> is not its frame's runtime (a checkpoint taken after
    bgr_set_rollback_frame_count), so the first keyframe carries the restored Time and the later ones the runtime at
    this rate; held to the request stream and a plain replay on twins restored from the same blob."""
    src = rate_world(600, fps, spawn_rate=spawn_rate)
    src.set_rollback_frame_count(33)  # Time<GgrsTime> stays 0
    _, first = src.replay_keyframes(log_for(40, 2, seed=1, spawn_every=7), 0, 11)
    assert first[0][0] == 33
    a, b, c = (rate_world(600, fps, spawn_rate=spawn_rate) for _ in range(3))
    for e in (a, b, c):
        e.restore(first[0][1])
    log = log_for(130, 2, seed=fps + spawn_rate, spawn_every=9)
    cs, kfs = a.replay_keyframes(log, 10, 11)
    assert [f for f, _ in kfs] == expected_frames(33, 130, 11)
    assert kfs[0][1] == first[0][1]
    assert kfs == stream_blobs(b, 33, log, 11)
    assert cs == c.replay(log, 10)
    assert live(a) == live(b) == live(c)


def test_query_runs_nothing_and_bounds_the_blobs():
    e = particles_world(900, rate=37, bundle=False)
    before = live(e)
    log = log_for(100, 2, seed=4, spawn_every=5)
    r = capi.bgr_replay(100, 2, 10, 0, log.ctypes.data)
    kf = capi.bgr_keyframes(8, 0, 0, None, 0, None)
    n, n_kf, size = C.c_uint32(), C.c_uint32(), C.c_size_t()
    assert e._lib.bgr_replay_keyframes(e._h, C.byref(r), C.byref(kf), None, 0, C.byref(n), C.byref(n_kf), C.byref(size)) == 0
    assert live(e) == before
    assert n_kf.value == len(expected_frames(0, 100, 8))
    _, kfs = e.replay_keyframes(log, 10, 8)
    assert sum((len(b) + 7) // 8 * 8 for _, b in kfs) <= size.value


@pytest.mark.parametrize("name", ["box", "spawning_fixed"])
def test_seeking_from_a_keyframe_equals_a_full_replay(name):
    a = MAKERS[name]()
    log = log_for(300, 2, seed=11, spawn_every=13)
    kk, k = 40, 10
    cs, kfs = a.replay_keyframes(log, k, kk)
    blobs = dict(kfs)
    rng = np.random.default_rng(5)
    for target in sorted(rng.integers(0, 300, 4).tolist()) + [299, 0]:
        full = MAKERS[name]()
        full.replay(log[:target], k)
        seek = MAKERS[name]()
        base = target // kk * kk
        seek.restore(blobs[base])
        seek.replay(log[base:target], k)
        assert live(seek) == live(full), target
        assert seek.replay(log[target:], k) == [x for x in cs if x[0] >= target]
        assert live(seek) == live(a)


@pytest.mark.parametrize("name", ["presence", "spawning_growable"])
def test_two_keyframe_replays_equal_one(name):
    a, b = MAKERS[name](), MAKERS[name]()
    log = log_for(170, 2, seed=3, spawn_every=7)
    cs1, kf1 = a.replay_keyframes(log[:83], 10, 6)
    cs2, kf2 = a.replay_keyframes(log[83:], 10, 6)
    cs, kf = b.replay_keyframes(log, 10, 6)
    assert cs1 + cs2 == cs and kf1 + kf2 == kf
    assert live(a) == live(b)


@pytest.mark.parametrize("points", [None, "3"])
def test_many_launches_give_the_same_bytes(monkeypatch, points):
    log = log_for(200, 2, seed=9, spawn_every=6)
    ref = particles_world(900, rate=37, bundle=False)
    want = ref.replay_keyframes(log, 4, 5)
    monkeypatch.setenv("BGR_TUNE_KEYFRAME_BYTES", "1")
    if points:
        monkeypatch.setenv("BGR_TUNE_REPLAY_POINTS", points)
    e = particles_world(900, rate=37, bundle=False)
    assert e.replay_keyframes(log, 4, 5) == want
    assert live(e) == live(ref)


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


ROWS = [1, 127, 700, 2000, 129, 40]


@pytest.mark.parametrize("make", [box_world, spawn_world, rate_world])
def test_batched_keyframes_equal_each_worlds_own(stream, make):
    def member(i, s):
        if make is spawn_world:
            return spawn_world(ROWS[i % 6], 4, stream=s, seed=i, rate=10 + i)
        if make is rate_world:  # spawning members at different rates and spawn rates
            return rate_world(ROWS[i % 6], [60, 7, 144, 30][i % 4], stream=s, seed=i, spawn_rate=5 + i)
        return box_world(ROWS[i % 6], 4, stream=s, seed=i, order_base=i * 1000)
    members = [member(i, stream) for i in range(7)]
    twins = [member(i, None) for i in range(7)]
    for i, (m, t) in enumerate(zip(members, twins)):
        m.set_rollback_frame_count(5 * i)
        t.set_rollback_frame_count(5 * i)
    batch = EngineBatch(members)
    rng = np.random.default_rng(1)
    for rnd in range(3):
        subset = sorted(rng.choice(7, size=int(rng.integers(1, 8)), replace=False).tolist())
        calls = [(w, log_for(int(rng.integers(0, 90)), 1 + w % 3, seed=10 * rnd + w, spawn_every=11), int(rng.integers(0, 12)),
                  int(rng.integers(1, 30))) for w in subset]
        res = batch.replay_keyframes(calls)
        for (w, log, k, kk), (status, cs, kfs) in zip(calls, res):
            assert status == capi.BGR_OK
            assert (cs, kfs) == twins[w].replay_keyframes(log, k, kk), f"world {w} round {rnd}"
    for w, (m, t) in enumerate(zip(members, twins)):
        assert live(m) == live(t), f"world {w}"


def test_batch_refusals_change_no_world(stream):
    members = [box_world(ROWS[i], 4, stream=stream, seed=i) for i in range(3)]
    batch = EngineBatch(members)
    before = [live(m) for m in members]
    log = log_for(50, 2, seed=1)
    n = 3
    worlds = (C.c_uint32 * n)(0, 1, 2)
    reps = (capi.bgr_replay * n)(*[capi.bgr_replay(50, 2, 10, 0, log.ctypes.data)] * n)
    bufs = [np.zeros(1 << 20, np.uint8) for _ in range(n)]
    idx = [(capi.bgr_keyframe * 64)() for _ in range(n)]
    out = (capi.bgr_checksum * 64)()
    n_cs, n_kf, status = (C.c_uint32 * n)(), (C.c_uint32 * n)(), (C.c_int32 * n)()
    for field, value, code in (("interval", 0, capi.BGR_ERR_INVALID_ARGUMENT), ("reserved", 1, capi.BGR_ERR_INVALID_ARGUMENT),
                               ("index_cap", 1, capi.BGR_ERR_CAPACITY), ("dst_cap", 64, capi.BGR_ERR_CAPACITY)):
        kfs = (capi.bgr_keyframes * n)(*[capi.bgr_keyframes(5, 64, 0, bufs[i].ctypes.data, bufs[i].size, idx[i]) for i in range(n)])
        setattr(kfs[1], field, value)
        rc = batch._lib.bgr_batch_replay_keyframes(batch._h, worlds, n, reps, kfs, out, 64, n_cs, n_kf, status)
        assert rc == code and status[1] == code, field
        assert batch._lib.bgr_last_error().decode().startswith("world 1: ")
        assert [live(m) for m in members] == before


def test_refusals_change_nothing():
    e = box_world(300, 4)
    before = live(e)
    log = log_for(50, 2, seed=2)
    r = capi.bgr_replay(50, 2, 10, 0, log.ctypes.data)
    buf = np.zeros(1 << 20, np.uint8)
    idx = (capi.bgr_keyframe * 64)()
    n, n_kf, size = C.c_uint32(), C.c_uint32(), C.c_size_t()
    out = (capi.bgr_checksum * 64)()

    def call(kf, rr=r):
        return e._lib.bgr_replay_keyframes(e._h, C.byref(rr), C.byref(kf), out, 64, C.byref(n), C.byref(n_kf), C.byref(size))
    assert call(capi.bgr_keyframes(0, 64, 0, buf.ctypes.data, buf.size, idx)) == capi.BGR_ERR_INVALID_ARGUMENT
    assert call(capi.bgr_keyframes(5, 64, 1, buf.ctypes.data, buf.size, idx)) == capi.BGR_ERR_INVALID_ARGUMENT
    assert call(capi.bgr_keyframes(5, 9, 0, buf.ctypes.data, buf.size, idx)) == capi.BGR_ERR_CAPACITY  # 10 keyframes
    assert call(capi.bgr_keyframes(5, 64, 0, buf.ctypes.data, 1000, idx)) == capi.BGR_ERR_CAPACITY
    bad = capi.bgr_replay(50, 2, 10, 1, log.ctypes.data)
    assert call(capi.bgr_keyframes(5, 64, 0, buf.ctypes.data, buf.size, idx), bad) == capi.BGR_ERR_INVALID_ARGUMENT
    assert live(e) == before
    s = Engine(max_entities=64, flags=capi.BGR_CFG_SHARDED)
    vel = s.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    s.checksum_component(vel, 0, 12)
    s.build()
    with pytest.raises(BgrError) as ei:
        s.replay_keyframes(np.zeros((4, 1), np.uint8), 1, 2)
    assert ei.value.status == capi.BGR_ERR_UNSUPPORTED


def test_non_finite_checksum_frame_still_writes_the_keyframes():
    a, b = box_world(300, 4), box_world(300, 4)
    for e in (a, b):
        t = np.ascontiguousarray(e.read_component(1, 0, 1)).view(np.float32).copy()
        t.reshape(-1)[0] = np.nan
        e.write_component(1, 0, t)
    log = log_for(60, 2, seed=1)
    lib, h = a._lib, a._h
    r = capi.bgr_replay(60, 2, 10, 0, log.ctypes.data)
    buf = np.zeros(1 << 22, np.uint8)
    idx = (capi.bgr_keyframe * 16)()
    kf = capi.bgr_keyframes(15, 16, 0, buf.ctypes.data, buf.size, idx)
    n, n_kf, size = C.c_uint32(), C.c_uint32(), C.c_size_t()
    out = (capi.bgr_checksum * 16)()
    assert lib.bgr_replay_keyframes(h, C.byref(r), C.byref(kf), out, 16, C.byref(n), C.byref(n_kf), C.byref(size)) == \
        capi.BGR_ERR_NON_FINITE
    assert n.value == 6 and n_kf.value == 4
    got = [(idx[i].frame, buf[idx[i].offset: idx[i].offset + idx[i].bytes].tobytes()) for i in range(4)]
    assert got == stream_blobs(b, 0, log, 15)


def test_retained_frames_and_desync_witnesses_are_untouched():
    from bevy_ggrs_b200.session import SyncTestSession
    e = Engine(max_entities=708, max_depth=9, flags=capi.BGR_CFG_DESYNC_CAPTURE)
    e.retain_confirmed(2, 4)
    vel = e.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    tf = e.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
    e.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
    e.checksum_component(tf, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
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
    assert before[1] and before[2]
    _, kfs = e.replay_keyframes(log_for(120, 2, seed=6), 10, 30)
    assert len(kfs) == 4
    assert kept() == before
