"""World batches (bgr_batch_*, EngineBatch): the request vectors of many engines with one registration in ONE launch.
Every member has a twin engine ticked alone by bgr_handle_requests with the same vectors; checksums, frame counters,
rings, peeks and live worlds must agree bit for bit, on the generated kernel (one launch) and on the interpreter
(BGR_TUNE_JIT=0: the batch runs its worlds one after another)."""
import struct

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import EDIT_DTYPE, Engine, EngineBatch
from bevy_ggrs_b200.plugin import (App, GgrsPlugin, GgrsSchedule, LocalInputs, ReadInputs, ResourceSystem, Session,
                                   Startup, SyncTestMismatch, System, step_batch)
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, P2PTraceSession, Request, SyncTestSession
from bevy_ggrs_b200.stress import register_particles

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]
OPT = capi.BGR_STRATEGY_OPTIONAL
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
SEQ = [0b0001, 0b1000, 0b0101, 0, 0b0010, 0b1010, 0b0100, 0b1001]
ROWS = [1, 127, 128, 129, 700, 2000]


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


# ---- registrations (every member of a batch has the same one) ----
def presence_world(n, depth, stream=None, flags=0, order_base=0, seed=0):
    """Score (optional, +1 per frame), Health (optional, satsub-despawn), Tag (12 B), all checksummed."""
    w = Engine(max_entities=n + 8, max_depth=depth, flags=flags, order_base=order_base, stream=stream)
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = w.rollback_component("Tag", 12, capi.BGR_STRATEGY_COPY)
    w.checksum_component(score, 0, 4)
    w.checksum_component(tag, 0, 12)
    w.checksum_component(health, 0, 4)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(seed)
    w.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    w.write_component(health, 0, rng.integers(3, 90, n, dtype=np.uint32))
    w.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in rng.choice(n, n // 5, replace=False):
        w.remove_component((score, health)[int(r) % 2], int(r))
    return w


def box_world(n, depth, stream=None, flags=0, order_base=0, seed=0):
    """box_game's Velocity / Transform with move_cube_system, both checksummed, the translation asserting finite."""
    w = Engine(max_entities=n + 8, max_depth=depth, flags=flags, order_base=order_base, stream=stream)
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


# ---- sessions: each world's vectors, fed back with the batch's checksums ----
class SyncDriver:
    def __init__(self, d):
        self.sess, self.depth = SyncTestSession(2, d, 9), 9

    def next(self, tick):
        for h in range(2):
            self.sess.add_local_input(h, SEQ[(tick + 3 * h) % len(SEQ)])
        return self.sess.info(), self.sess.advance_frame()

    def saved(self, checksums):
        for f, cs in checksums:
            self.sess.save_cell(f, cs)


class P2PDriver(SyncDriver):
    def __init__(self, mp, seed):
        self.sess, self.depth = P2PTraceSession(2, max_prediction=mp, input_delay=2, seed=seed), mp + 1

    def next(self, tick):
        self.sess.add_local_input(0, SEQ[tick % len(SEQ)])
        return self.sess.info(), self.sess.advance_frame()


class SpectatorDriver:
    depth = 4

    def next(self, tick):
        return (capi.BGR_SESSION_SPECTATOR, 0, 0, 0), [Request(ADVANCE, 0, [SEQ[tick % 8], SEQ[(tick + 5) % 8]])]

    def saved(self, checksums):
        pass


class NoSessionDriver(SpectatorDriver):
    depth = 8

    def __init__(self):
        self.frame = 0

    def next(self, tick):
        reqs = ([Request(SAVE, self.frame)] if tick < 5 else []) + [Request(ADVANCE, 0, [SEQ[tick % 8]])]
        self.frame += 1
        return (capi.BGR_SESSION_NONE, 0, 0, 0), reqs


def driver(i):
    kind = i % 4
    if kind == 0:
        return SyncDriver(1 + (3 * (i // 4)) % 8)
    if kind == 1:
        return P2PDriver(3 + i % 6, seed=0xB200 + i)
    return SpectatorDriver() if kind == 2 else NoSessionDriver()


class Fleet:
    """A batch of members on one stream and their twins, each on its own engine stream."""

    def __init__(self, make, stream, n_worlds=10):
        self.drivers = [driver(i) for i in range(n_worlds)]
        # engines may differ in capacity, depth, rows, session, desync capture, growth and order_base
        opts = [dict(), dict(flags=capi.BGR_CFG_DESYNC_CAPTURE), dict(flags=capi.BGR_CFG_GROWABLE), dict(order_base=4096), dict()]
        self.members, self.twins = [], []
        for i, d in enumerate(self.drivers):
            kw = dict(opts[i % len(opts)], seed=i)
            self.members.append(make(ROWS[i % len(ROWS)], d.depth, stream=stream, **kw))
            self.twins.append(make(ROWS[i % len(ROWS)], d.depth, **kw))
        self.batch = EngineBatch(self.members)
        self.tick_no = [0] * n_worlds

    def tick(self, worlds=None):
        worlds = list(range(len(self.members))) if worlds is None else worlds
        calls = []
        for w in worlds:
            info, reqs = self.drivers[w].next(self.tick_no[w])
            self.tick_no[w] += 1
            calls.append((w, info, reqs))
        l_m = [self.members[w].launch_count() for w in worlds]
        l_t = [self.twins[w].launch_count() for w in worlds]
        res = self.batch.handle_requests(calls)
        for (w, info, reqs), (status, cs) in zip(calls, res):
            assert status == capi.BGR_OK
            assert cs == self.twins[w].handle_requests(info, reqs), f"world {w} tick {self.tick_no[w]}"
            self.drivers[w].saved(cs)
        for k, w in enumerate(worlds):
            assert self.members[w].launch_count() - l_m[k] == self.twins[w].launch_count() - l_t[k]
            lk = self.members[w].last_kernel()
            if self.batch.specialised():
                assert lk.batched and lk.kind == "generic_nvrtc"
            else:
                assert not lk.batched
        return res


def image(e):
    """Everything observable of a world: counters, ring, every stored frame's peek, the live image."""
    n = e.row_count()
    out = [e.rollback_frame_count(), e.confirmed_frame_count(), e.snapshot_frames(), n, e.active_count(),
           e.read_alive(0, n).tobytes()]
    for c in range(len(e.elem_bytes)):
        out.append(e.read_component(c, 0, n).tobytes())
        for f in e.snapshot_frames():
            p = e.peek(f, c, 0, n)
            out.append((f, None if p is None else (p[0].tobytes(), p[1].tobytes())))
    return out


def assert_fleet_equal(fl):
    for w, (m, t) in enumerate(zip(fl.members, fl.twins)):
        assert image(m) == image(t), f"world {w}"


@pytest.mark.parametrize("make", [presence_world, box_world])
def test_parity_with_twins(generic_kernel, stream, make):
    fl = Fleet(make, stream, n_worlds=16)
    assert fl.batch.specialised() == (generic_kernel != "interpreter")
    for _ in range(64):
        res = fl.tick()
    if fl.batch.specialised():
        assert {m.last_kernel().item_rows for m in fl.members} == {512 if generic_kernel == "jit" else 128}
    assert sum(len(cs) for _, cs in res) > 0
    assert_fleet_equal(fl)


def test_subsets_leave_other_worlds_untouched(stream):
    fl = Fleet(presence_world, stream, n_worlds=8)
    for _ in range(12):
        fl.tick()
    for part in ([0, 2, 4, 6], [7, 1], [3]):
        before = {w: image(fl.members[w]) for w in range(8) if w not in part}   # reads launch kernels of their own
        launches = {w: fl.members[w].launch_count() for w in before}
        for _ in range(3):
            fl.tick(part)
        for w in before:
            assert fl.members[w].launch_count() == launches[w], f"world {w}"
            assert image(fl.members[w]) == before[w], f"world {w}"
    assert_fleet_equal(fl)


def test_a_refused_call_executes_nothing(stream):
    fl = Fleet(box_world, stream, n_worlds=4)
    for _ in range(10):
        fl.tick()
    before = [image(m) for m in fl.members]           # reads launch kernels of their own
    launches = [m.launch_count() for m in fl.members]
    info, reqs = fl.drivers[0].next(fl.tick_no[0])   # a valid vector for world 0 ...
    calls = [(0, info, reqs), (1, (capi.BGR_SESSION_NONE, 0, 0, 0), [Request(LOAD, 99), Request(ADVANCE, 0, [0, 0])]),
             (2, (capi.BGR_SESSION_SPECTATOR, 0, 0, 0), [Request(ADVANCE, 0, [0, 0])])]
    with pytest.raises(BgrError) as ei:
        fl.batch.handle_requests(calls)                # ... but world 1 loads a frame it never saved
    assert ei.value.status == capi.BGR_ERR_NO_SNAPSHOT and str(ei.value).startswith("world 1: ")
    assert [m.launch_count() for m in fl.members] == launches
    assert [image(m) for m in fl.members] == before
    for _ in range(4):                                 # world 0's session moved on without it: leave it out

        fl.tick([1, 2, 3])
    assert_fleet_equal(fl)


def test_refused_calls_and_members(stream):
    fl = Fleet(presence_world, stream, n_worlds=3)
    sp = (capi.BGR_SESSION_SPECTATOR, 0, 0, 0)
    adv = [Request(ADVANCE, 0, [0])]
    with pytest.raises(BgrError) as ei:                # duplicate world
        fl.batch.handle_requests([(1, sp, adv), (1, sp, adv)])
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and "world 1" in str(ei.value)
    with pytest.raises(BgrError) as ei:                # out of range
        fl.batch.handle_requests([(3, sp, adv)])
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    fl.members[2].submit_requests(sp, adv)             # pending submit
    with pytest.raises(BgrError) as ei:
        fl.batch.handle_requests([(0, sp, adv), (2, sp, adv)])
    assert ei.value.status == capi.BGR_ERR_STATE and str(ei.value).startswith("world 2: ")
    fl.members[2].collect()
    fl.twins[2].handle_requests(sp, adv)
    assert image(fl.members[2]) == image(fl.twins[2])

    def refused(engines, status):
        with pytest.raises(BgrError) as ei:
            EngineBatch(engines)
        assert ei.value.status == status, str(ei.value)
    a = presence_world(100, 8, stream=stream)
    refused([a, box_world(100, 8, stream=stream)], capi.BGR_ERR_INVALID_ARGUMENT)       # registrations differ
    refused([a, presence_world(100, 8)], capi.BGR_ERR_INVALID_ARGUMENT)                 # streams differ
    refused([presence_world(100, 8), presence_world(100, 8)], capi.BGR_ERR_INVALID_ARGUMENT)  # no shared stream
    refused([a, presence_world(100, 8, stream=stream, flags=capi.BGR_CFG_FORCE_STEPWISE)], capi.BGR_ERR_UNSUPPORTED)
    refused([a, presence_world(100, 8, stream=stream, flags=capi.BGR_CFG_SHARDED)], capi.BGR_ERR_UNSUPPORTED)
    bundles = []
    for _ in range(2):
        b = Engine(max_entities=64, max_depth=8, stream=stream)
        register_particles(b)
        b.build()
        bundles.append(b)
    refused(bundles, capi.BGR_ERR_UNSUPPORTED)                                          # the particles bundle
    refused([a, a], capi.BGR_ERR_INVALID_ARGUMENT)


def test_non_finite_fails_only_its_world(stream):
    fl = Fleet(box_world, stream, n_worlds=4)
    for _ in range(6):
        fl.tick()
    nan = np.zeros((1, 10), np.float32); nan[0, 0] = np.nan; nan[0, 6] = 1.0
    for e in (fl.members[2], fl.twins[2]):           # world 2 is a spectator: no rollback undoes the NaN
        e.write_component(1, 0, nan)
    calls = [(w,) + fl.drivers[w].next(fl.tick_no[w]) for w in (0, 1, 3)]
    calls.insert(2, (2, (capi.BGR_SESSION_SPECTATOR, 0, 0, 0), [Request(SAVE, 0), Request(ADVANCE, 0, [0, 0])]))
    res = fl.batch.handle_requests(calls)
    for (w, info, reqs), (status, cs) in zip(calls, res):
        if w == 2:
            assert status == capi.BGR_ERR_NON_FINITE
            with pytest.raises(BgrError) as ei:
                fl.twins[w].handle_requests(info, reqs)
            assert ei.value.status == capi.BGR_ERR_NON_FINITE
        else:
            assert status == capi.BGR_OK and cs == fl.twins[w].handle_requests(info, reqs)
            fl.drivers[w].saved(cs)


def test_members_stay_ordinary_engines(stream):
    fl = Fleet(presence_world, stream, n_worlds=8)
    feeds = [(e.feed_create([(0, 0, 4), (2, 0, 12)]), e) for e in (fl.members[4], fl.twins[4])]
    rng = np.random.default_rng(3)
    for step in range(24):
        fl.tick()
        m, t = fl.members, fl.twins
        k = step % 6
        if k == 0:                                   # a live read of a SyncTest world whose image is deferred
            assert step == 0 or m[0].last_kernel().deferred_live
            assert np.array_equal(m[0].read_component(2, 0, m[0].row_count()), t[0].read_component(2, 0, t[0].row_count()))
        elif k == 1:                                 # host edits: despawn a row, write a Tag
            rows = m[1].row_count()
            r = int(rng.integers(rows - 1))
            ed = np.zeros(2, EDIT_DTYPE)
            ed[0] = (capi.BGR_EDIT_DESPAWN, 0, r, 0, 0, 0, 0, 0)
            ed[1] = (capi.BGR_EDIT_WRITE, 2, rows - 1, 1, 0, 12, 0, 0)
            vals = rng.integers(0, 2**32, 3, dtype=np.uint32).tobytes()
            for e in (m[1], t[1]):
                e.apply_edits(ed, vals)
        elif k == 2:                                 # spawn, write, despawn
            for e in (m[2], t[2]):
                first = e.spawn(3)
                e.write_component(2, first, np.arange(9, dtype=np.uint32).reshape(3, 3) + step)
                e.despawn(0)
        elif k == 3:                                 # a checkpoint restore of a world without a session (its ring is its own)
            for e in (m[7], t[7]):
                e.restore(e.checkpoint(e.snapshot_frames()[-1]))
        elif k == 4:                                 # a change-feed report
            recs = []
            for feed, e in feeds:
                buf = e.feed_alloc(feed, 4096)
                recs.append(e.feed_wait(e.feed_begin(feed, buf, 4096)))
            assert recs[0][0].tobytes() == recs[1][0].tobytes() and recs[0][1] == recs[1][1]
        else:                                        # remove / insert an optional component on live rows
            n = t[3].row_count()
            alive = t[3].read_alive(0, n).astype(bool)
            with_score = np.flatnonzero(alive & t[3].has_component(0, 0, n).astype(bool))
            without_health = np.flatnonzero(alive & ~t[3].has_component(1, 0, n).astype(bool))
            for e in (m[3], t[3]):
                if len(with_score):
                    e.remove_component(0, int(with_score[0]))
                if len(without_health):
                    e.insert_component(1, int(without_health[0]), np.array([50], np.uint32))
    assert_fleet_equal(fl)


def _box_app(backend, counter_rows, native_resource=False):
    """box_game (2 players, SyncTest d=8, FrameCount checksummed on the host) with an optional, checksummed Counter
    column bound to the non-deterministic store_call_count system (tests/synctest.rs:83-125); only the rows in
    ``counter_rows`` keep the component."""
    app = App(backend)
    app.insert_resource(Session.SyncTest(SyncTestSession(2, 8, 9, input_delay=2)))
    app.add_plugins(GgrsPlugin())
    app.add_systems(ReadInputs, lambda a: a.insert_resource(
        LocalInputs({h: SEQ[(a.ticks + 3 * h) % len(SEQ)] for h in a.local_players.handles})))
    vel = app.rollback_component_with_copy("Velocity", 12)
    tf = app.rollback_component_with_clone("Transform", 40)
    counter = app.rollback_optional_component_with_copy("Counter", 4)
    app.checksum_component_with_hash(counter)
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_BOX_MOVE, [tf, vel]))
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_U32_STORE_CALL_COUNT, [counter], [0]))
    if native_resource:
        from oracle_backend import ORC_SYS_RESOURCE_U32_ADD
        fc = backend.rollback_resource("FrameCount", bytes(4), checksum=True)
        app.add_systems(GgrsSchedule, System(ORC_SYS_RESOURCE_U32_ADD, [], [fc]))
    else:
        app.rollback_resource_with_copy("FrameCount", bytes(4)).checksum_resource_with_hash("FrameCount")

        def increase_frame_system(res):  # box_game.rs:146-148
            res["FrameCount"][:] = struct.pack("<I", (struct.unpack("<I", res["FrameCount"])[0] + 1) & 0xFFFFFFFF)
        app.add_systems(GgrsSchedule, ResourceSystem(increase_frame_system))

    def setup(a):
        first = a.world.spawn(2)
        t = np.zeros((2, 10), np.float32)
        for h in range(2):
            rot = np.float32(h) / np.float32(2) * np.float32(2.0) * np.float32(np.pi)
            t[h, 0] = 1.25 * np.cos(rot); t[h, 1] = 0.1; t[h, 2] = 1.25 * np.sin(rot)
            t[h, 6] = 1.0; t[h, 7:10] = 1.0
        a.world.write_component(tf, first, t)
        for r in range(2):
            if r not in counter_rows:
                a.world.remove_component(counter, first + r)
    app.add_systems(Startup, setup)
    bad = []
    app.add_observer(SyncTestMismatch, lambda ev: bad.append(ev))
    return app, bad


def test_step_batch_apps(stream):
    from oracle_backend import OracleWorld
    apps = [_box_app(Engine(max_entities=4, max_depth=9, stream=stream), rows) for rows in ([], [1], [])]
    oracle, bad_o = _box_app(OracleWorld(), [], native_resource=True)
    for app, _ in apps:
        app.finish()
    batch = EngineBatch([app.world for app, _ in apps])
    for _ in range(60):
        step_batch([app for app, _ in apps], batch)
        oracle.step()
        assert apps[0][0].last_checksums == oracle.last_checksums
    assert not apps[0][1] and not apps[2][1] and not bad_o
    assert apps[1][1]                                    # only the App whose entity has a Counter mismatches
    assert apps[0][0].rollback_frame_count() == oracle.rollback_frame_count() == apps[0][0].ticks
    assert struct.unpack("<I", apps[0][0].resources["FrameCount"])[0] == apps[0][0].ticks
    if batch.specialised():
        assert apps[0][0].world.last_kernel().batched


def test_one_batched_call_is_one_kernel(generic_kernel, stream):
    torch = pytest.importorskip("torch")
    if generic_kernel == "interpreter":
        pytest.skip("the interpreter batch runs its worlds one after another")
    members = [box_world(2, 9, stream=stream, seed=i) for i in range(64)]
    batch = EngineBatch(members)
    drivers = [SyncDriver(7) for _ in members]

    def call(tick):
        calls = [(w,) + d.next(tick) for w, d in enumerate(drivers)]
        for (w, _, _), (status, cs) in zip(calls, batch.handle_requests(calls)):
            assert status == capi.BGR_OK
            drivers[w].saved(cs)
    for tick in range(12):                               # past the ring fill: every vector starts with its own Load
        call(tick)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]):
        call(12)                                         # the first session of a process sets the tracer up
        torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call(13)
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset"))]
    assert kernels == ["k_generic_jit_batch"], kernels
