"""Replay traces (bgr_replay_trace, Engine.replay_trace; the batch call): a replay that also records chosen fields of a
row range every T frames.  Each sample's records are held byte for byte to a twin engine that replays the same log in
pieces ending at each sample frame and reads the traced rows back with bgr_read_component / bgr_has_component /
bgr_read_alive / bgr_row_count; the checksums and the end state are held to a plain bgr_replay.  Every test runs on the
interpreter (BGR_TUNE_JIT=0: the chunked fallback and k_trace_gather), the generated kernel with whole tiles and with
128-row items."""
import ctypes as C

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import EngineBatch
from bevy_ggrs_b200.session import ADVANCE, Request

from test_gpu_batch import box_world, presence_world
from test_gpu_replay import live, log_for, particles_world, tick_on

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]

# name -> (maker, fields [(column, byte_offset, byte_len)], traced rows (first_row, n_rows))
WORLDS = {
    # Velocity and Transform's translation; the range runs past the 700 rows
    "box": (lambda: box_world(700, 4), [(1, 0, 12), (0, 0, 12)], (650, 58)),
    # both optional columns and the tag, every row
    "presence": (lambda: presence_world(1300, 4), [(0, 0, 4), (1, 0, 4), (2, 4, 8)], (0, 1308)),
    # rows are born into the range as the replay runs, and the engine grows past 520
    "spawning_growable": (lambda: particles_world(500, rate=40, cap=520, flags=capi.BGR_CFG_GROWABLE, bundle=False),
                          [(0, 0, 12), (1, 0, 12), (2, 0, 4)], (480, 700)),
}


def expected(w, fields, first_row, n_rows):
    """The records of rows [first_row, first_row + n_rows) read back from a world (an engine or the oracle)."""
    rb = 8 + sum(ln for _, _, ln in fields)
    out = np.zeros((n_rows, rb), np.uint8)
    out[:, 0:4] = np.arange(first_row, first_row + n_rows, dtype="<u4").view(np.uint8).reshape(-1, 4)
    m = max(0, min(first_row + n_rows, w.row_count()) - first_row)
    if m:
        state = (np.asarray(w.read_alive(first_row, m)) != 0).astype("<u4")
        at = 8
        for k, (c, off, ln) in enumerate(fields):
            has = np.asarray(w.has_component(c, first_row, m)) != 0
            state |= has.astype("<u4") << (1 + k)
            v = np.ascontiguousarray(w.read_component(c, first_row, m)).view(np.uint8).reshape(m, -1)[:, off:off + ln].copy()
            v[~has] = 0
            out[:m, at:at + ln] = v
            at += ln
        out[:m, 4:8] = state.view(np.uint8).reshape(-1, 4)
    return out


def pieces(e, f0, log, k, tt, fields, first_row, n_rows):
    """What a trace stands for: bgr_replay in pieces that end at each sample frame, the rows read back there."""
    cs, samples, recs, at = [], [], [], 0
    for j in range(len(log)):
        if (f0 + j) % tt == 0:
            cs += e.replay(log[at:j], k)
            at = j
            samples.append((f0 + j, e.row_count()))
            recs.append(expected(e, fields, first_row, n_rows))
    cs += e.replay(log[at:], k)
    rb = 8 + sum(ln for _, _, ln in fields)
    return cs, samples, np.array(recs, np.uint8).reshape(len(recs), n_rows, rb)


@pytest.mark.parametrize("f0,n,k,tt", [(0, 90, 10, 1), (7, 150, 10, 7), (3, 130, 0, 60), (5, 40, 4, 500)])
@pytest.mark.parametrize("name", list(WORLDS))
def test_trace_equals_a_twin_read_back_and_a_plain_replay(name, f0, n, k, tt):
    make, fields, (first_row, n_rows) = WORLDS[name]
    a, b, c = make(), make(), make()
    for e in (a, b, c):
        e.set_rollback_frame_count(f0)
    log = log_for(n, 2, seed=len(name) + tt, spawn_every=9)
    cs, samples, recs = a.replay_trace(log, k, tt, fields, first_row, n_rows)
    assert [f for f, _ in samples] == [f0 + j for j in range(n) if (f0 + j) % tt == 0]
    want = pieces(b, f0, log, k, tt, fields, first_row, n_rows)
    assert cs == want[0]
    assert samples == want[1]
    assert recs.shape == want[2].shape and np.array_equal(recs, want[2])
    assert cs == c.replay(log, k)
    assert live(a) == live(b) == live(c)
    assert a.last_kernel().replay == c.last_kernel().replay
    assert tick_on(a) == tick_on(c)


@pytest.mark.parametrize("name", list(WORLDS))
def test_two_traces_equal_one(name):
    make, fields, (first_row, n_rows) = WORLDS[name]
    a, b = make(), make()
    log = log_for(140, 2, seed=5, spawn_every=8)
    cs1, s1, r1 = a.replay_trace(log[:61], 10, 6, fields, first_row, n_rows)
    cs2, s2, r2 = a.replay_trace(log[61:], 10, 6, fields, first_row, n_rows)
    cs, s, r = b.replay_trace(log, 10, 6, fields, first_row, n_rows)
    assert (cs1 + cs2, s1 + s2) == (cs, s)
    assert np.array_equal(np.concatenate([r1, r2]), r)
    assert live(a) == live(b)


@pytest.mark.parametrize("points", [None, "7"])
def test_many_launches_give_the_same_bytes(monkeypatch, points):
    make, fields, (first_row, n_rows) = WORLDS["spawning_growable"]
    log = log_for(200, 2, seed=9, spawn_every=6)
    ref = make()
    want = ref.replay_trace(log, 3, 2, fields, first_row, n_rows)
    monkeypatch.setenv("BGR_TUNE_TRACE_BYTES", str(3 * n_rows * 36 + 1))  # three samples per launch
    if points:
        monkeypatch.setenv("BGR_TUNE_REPLAY_POINTS", points)
    e = make()
    got = e.replay_trace(log, 3, 2, fields, first_row, n_rows)
    assert got[:2] == want[:2] and np.array_equal(got[2], want[2])
    assert live(e) == live(ref)


@pytest.mark.parametrize("name", list(WORLDS))
def test_the_fallback_writes_the_kernels_bytes(monkeypatch, name):
    make, fields, (first_row, n_rows) = WORLDS[name]
    log = log_for(100, 2, seed=3, spawn_every=7)
    a = make()
    want = a.replay_trace(log, 10, 3, fields, first_row, n_rows)
    monkeypatch.setenv("BGR_TUNE_JIT", "0")
    b = make()
    got = b.replay_trace(log, 10, 3, fields, first_row, n_rows)
    assert not b.last_kernel().replay
    assert got[:2] == want[:2] and np.array_equal(got[2], want[2])
    assert live(a) == live(b)


def test_query_runs_nothing_and_refusals_change_nothing():
    e = box_world(300, 4)
    before = live(e)
    log = log_for(50, 2, seed=2)
    r = capi.bgr_replay(50, 2, 10, 0, log.ctypes.data)
    fa = (capi.bgr_feed_field * 2)(capi.bgr_feed_field(1, 0, 12), capi.bgr_feed_field(0, 4, 8))
    buf = np.zeros(1 << 20, np.uint8)
    smp = (capi.bgr_trace_sample * 64)()
    n, n_s, size = C.c_uint32(), C.c_uint32(), C.c_size_t()
    out = (capi.bgr_checksum * 64)()

    def trace(**kw):
        t = dict(interval=5, first_row=0, n_rows=300, n_fields=2, fields=C.cast(fa, C.POINTER(capi.bgr_feed_field)),
                 dst=buf.ctypes.data, dst_cap=buf.size, samples=C.cast(smp, C.POINTER(capi.bgr_trace_sample)),
                 samples_cap=64, reserved=0)
        t.update(kw)
        return capi.bgr_trace(**t)

    def call(t, rr=r):
        return e._lib.bgr_replay_trace(e._h, C.byref(rr), C.byref(t), out, 64, C.byref(n), C.byref(n_s), C.byref(size))
    assert call(trace(dst=None)) == capi.BGR_OK
    assert (n_s.value, size.value) == (10, 10 * 300 * 28)
    assert live(e) == before and e.rollback_frame_count() == 0
    bad_field = (capi.bgr_feed_field * 1)(capi.bgr_feed_field(0, 4, 12))  # past Velocity's 12 bytes
    bad_col = (capi.bgr_feed_field * 1)(capi.bgr_feed_field(5, 0, 4))
    for t, code in ((trace(interval=0), capi.BGR_ERR_INVALID_ARGUMENT), (trace(reserved=1), capi.BGR_ERR_INVALID_ARGUMENT),
                    (trace(n_rows=0), capi.BGR_ERR_INVALID_ARGUMENT), (trace(first_row=9), capi.BGR_ERR_INVALID_ARGUMENT),
                    (trace(n_fields=9), capi.BGR_ERR_CAPACITY),
                    (trace(n_fields=1, fields=C.cast(bad_field, C.POINTER(capi.bgr_feed_field))), capi.BGR_ERR_INVALID_ARGUMENT),
                    (trace(n_fields=1, fields=C.cast(bad_col, C.POINTER(capi.bgr_feed_field))), capi.BGR_ERR_INVALID_ARGUMENT),
                    (trace(samples_cap=9), capi.BGR_ERR_CAPACITY), (trace(dst_cap=10 * 300 * 28 - 1), capi.BGR_ERR_CAPACITY)):
        assert call(t) == code, e._lib.bgr_last_error()
    assert call(trace(first_row=8), capi.bgr_replay(50, 2, 10, 1, log.ctypes.data)) == capi.BGR_ERR_INVALID_ARGUMENT
    assert live(e) == before and e.rollback_frame_count() == 0
    assert call(trace(first_row=8)) == capi.BGR_OK  # rows [8, 308): the engine's last row
    assert n_s.value == 10 and smp[9].frame == 45 and smp[9].rows == 300


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


ROWS = [1, 127, 700, 2000, 129, 40]
BOX_FIELDS = [(1, 0, 12), (0, 0, 12)]


def test_batched_traces_equal_each_worlds_own(stream):
    members = [box_world(ROWS[i % 6], 4, stream=stream, seed=i, order_base=i * 1000) for i in range(7)]
    twins = [box_world(ROWS[i % 6], 4, seed=i, order_base=i * 1000) for i in range(7)]
    for i, (m, t) in enumerate(zip(members, twins)):
        m.set_rollback_frame_count(5 * i)
        t.set_rollback_frame_count(5 * i)
    batch = EngineBatch(members)
    rng = np.random.default_rng(1)
    for rnd in range(3):
        subset = sorted(rng.choice(7, size=int(rng.integers(1, 8)), replace=False).tolist())
        calls = []
        for w in subset:
            rows = ROWS[w % 6] + 8
            a = int(rng.integers(0, rows))
            calls.append((w, log_for(int(rng.integers(0, 90)), 1 + w % 3, seed=10 * rnd + w), int(rng.integers(0, 12)),
                          int(rng.integers(1, 30)), a, int(rng.integers(1, rows - a + 1))))
        res = batch.replay_trace(calls, BOX_FIELDS)
        for (w, log, k, tt, a, nr), (status, cs, samples, recs) in zip(calls, res):
            assert status == capi.BGR_OK
            want = twins[w].replay_trace(log, k, tt, BOX_FIELDS, a, nr)
            assert (cs, samples) == want[:2], f"world {w} round {rnd}"
            assert np.array_equal(recs, want[2]), f"world {w} round {rnd}"
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
    fa = (capi.bgr_feed_field * 2)(*[capi.bgr_feed_field(*f) for f in BOX_FIELDS])
    other = (capi.bgr_feed_field * 2)(capi.bgr_feed_field(1, 0, 12), capi.bgr_feed_field(0, 0, 8))
    bufs = [np.zeros(1 << 20, np.uint8) for _ in range(n)]
    smp = [(capi.bgr_trace_sample * 64)() for _ in range(n)]
    out = (capi.bgr_checksum * 64)()
    n_cs, n_s, status = (C.c_uint32 * n)(), (C.c_uint32 * n)(), (C.c_int32 * n)()

    def traces():
        return (capi.bgr_trace * n)(*[capi.bgr_trace(5, 0, ROWS[i], 2, C.cast(fa, C.POINTER(capi.bgr_feed_field)),
                                                     bufs[i].ctypes.data, bufs[i].size,
                                                     C.cast(smp[i], C.POINTER(capi.bgr_trace_sample)), 64, 0) for i in range(n)])
    cases = [("interval", 0, capi.BGR_ERR_INVALID_ARGUMENT), ("reserved", 1, capi.BGR_ERR_INVALID_ARGUMENT),
             ("n_rows", ROWS[1] + 9, capi.BGR_ERR_INVALID_ARGUMENT), ("samples_cap", 1, capi.BGR_ERR_CAPACITY),
             ("dst_cap", 64, capi.BGR_ERR_CAPACITY), ("fields", C.cast(other, C.POINTER(capi.bgr_feed_field)), capi.BGR_ERR_INVALID_ARGUMENT)]
    for field, value, code in cases:
        trs = traces()
        setattr(trs[1], field, value)
        rc = batch._lib.bgr_batch_replay_trace(batch._h, worlds, n, reps, trs, out, 64, n_cs, n_s, status)
        assert rc == code and status[1] == code, field
        assert batch._lib.bgr_last_error().decode().startswith("world 1: ")
        assert [live(m) for m in members] == before
    members[1].submit_requests((capi.BGR_SESSION_SPECTATOR, 0, 0, 0), [Request(ADVANCE, 0, [1, 2])])
    rc = batch._lib.bgr_batch_replay_trace(batch._h, worlds, n, reps, traces(), out, 64, n_cs, n_s, status)
    assert rc == capi.BGR_ERR_STATE and status[1] == capi.BGR_ERR_STATE
    members[1].collect()
    assert [live(m) for m in members][::2] == before[::2]


def test_batched_launches_do_not_depend_on_the_world_count(stream):
    log = log_for(120, 2, seed=4)
    counts = []
    for n in (1, 4, 16):
        members = [box_world(700, 4, stream=stream, seed=i) for i in range(n)]
        batch = EngineBatch(members)
        l0 = members[0].launch_count()
        res = batch.replay_trace([(w, log, 10, 1, 0, 700) for w in range(n)], BOX_FIELDS)
        assert all(r[0] == capi.BGR_OK and r[3].shape == (120, 700, 32) for r in res)
        counts.append(members[0].launch_count() - l0)
        batch.close()
    assert counts[0] == counts[1] == counts[2], counts


def test_non_finite_checksum_frame_still_writes_every_sample():
    make, fields, (first_row, n_rows) = WORLDS["box"]
    a, b, c = make(), make(), make()
    tf = a.read_component(1, 3, 1).view(np.float32).copy()
    tf[0, 0:3] = np.nan   # Transform's translation of row 3: finite-asserted
    for e in (a, b, c):
        e.write_component(1, 3, tf)
    log = log_for(30, 2, seed=6)
    with pytest.raises(BgrError) as ei:
        a.replay_trace(log, 10, 4, [(1, 0, 12)], 0, 8)
    assert ei.value.status == capi.BGR_ERR_NON_FINITE
    lib, r = a._lib, capi.bgr_replay(30, 2, 10, 0, log.ctypes.data)
    fa = (capi.bgr_feed_field * 1)(capi.bgr_feed_field(1, 0, 12))
    buf = np.zeros(8 * 8 * 20, np.uint8)
    smp = (capi.bgr_trace_sample * 8)()
    t = capi.bgr_trace(4, 0, 8, 1, C.cast(fa, C.POINTER(capi.bgr_feed_field)), buf.ctypes.data, buf.size,
                       C.cast(smp, C.POINTER(capi.bgr_trace_sample)), 8, 0)
    n, n_s, size = C.c_uint32(), C.c_uint32(), C.c_size_t()
    out = (capi.bgr_checksum * 8)()
    assert lib.bgr_replay_trace(b._h, C.byref(r), C.byref(t), out, 8, C.byref(n), C.byref(n_s), C.byref(size)) == capi.BGR_ERR_NON_FINITE
    assert n_s.value == 8 and size.value == buf.size
    want = pieces(c, 0, log, 0, 4, [(1, 0, 12)], 0, 8)[2]
    assert np.array_equal(buf.reshape(8, 8, 20), want)
