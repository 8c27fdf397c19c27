"""App replays (App.replay / replay_keyframes / replay_trace, and replay_batch / replay_keyframes_batch /
replay_trace_batch) of box_game with its FrameCount rollback resource, checksummed on the host as box_game_p2p.rs
registers it.  A replay must leave the App as the host half of handle_requests leaves it after the equivalent stream
[Save(f) if f % k == 0, Advance(inputs[j])], except that no snapshot is pushed: checksums with the resource parts,
resources, resource frame and world, with the resource store and ring left alone.  Every test runs on the generated
kernel, the interpreter (BGR_TUNE_JIT=0) and BGR_CFG_FORCE_STEPWISE, except the batch tests: a world batch does not take
BGR_CFG_FORCE_STEPWISE engines."""
import struct

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine, EngineBatch
from bevy_ggrs_b200.plugin import (App, GgrsPlugin, GgrsSchedule, LocalInputs, ReadInputs, ResourceSystem, Session,
                                   Startup, System, replay_batch, replay_keyframes_batch, replay_trace_batch)
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, P2PTraceSession, Request, SyncTestSession

pytestmark = pytest.mark.gpu
SEQ = [0b0001, 0b1000, 0b0101, 0, 0b0010, 0b1010, 0b0100, 0b1001]
SPECTATOR = (capi.BGR_SESSION_SPECTATOR, 0, 0, 0)
VEL, TF = 0, 1  # box_app's columns


def path_flags(path, monkeypatch):
    """The engine flags of a kernel path: the registration's generated kernel, the interpreter, or stepwise launches."""
    if path == "stepwise":
        return capi.BGR_CFG_FORCE_STEPWISE
    monkeypatch.setenv("BGR_TUNE_JIT", "0" if path == "interpreter" else "2")
    return 0


@pytest.fixture(params=["jit", "interpreter", "stepwise"])
def flags(request, monkeypatch):
    return path_flags(request.param, monkeypatch)


@pytest.fixture(params=["jit", "interpreter"])
def batch_flags(request, monkeypatch):
    """A world batch takes only engines that run the generic one-launch program: BGR_CFG_FORCE_STEPWISE engines cannot be
    batched (bgr_batch_create refuses them)."""
    return path_flags(request.param, monkeypatch)


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


class SessionInfo:
    """A session that only supplies handle_requests' session info and keeps no cells: the twin Apps run a request stream
    through the App's host half under it (the Python mirror has no spectator session)."""

    def __init__(self, info):
        self.value = info

    def info(self):
        return self.value

    def save_cell(self, frame, checksum):
        pass


def increase_frame_system(res):  # box_game.rs:146-148
    res["FrameCount"][:] = struct.pack("<I", (struct.unpack("<I", res["FrameCount"])[0] + 1) & 0xFFFFFFFF)


def box_app(flags, session=None, stream=None):
    """box_game with FrameCount (rollback_resource_with_copy + checksum_resource_with_hash) and the translation checksummed
    as finite.  Returns (app, transform column, velocity column)."""
    app = App(Engine(max_entities=4, max_depth=9, flags=flags, stream=stream))
    if session is not None:
        app.insert_resource(session)
    app.add_plugins(GgrsPlugin())
    app.add_systems(ReadInputs, lambda a: a.insert_resource(
        LocalInputs({h: SEQ[(a.ticks + 3 * h) % len(SEQ)] for h in a.local_players.handles})))
    vel = app.rollback_component_with_copy("Velocity", 12)
    tf = app.rollback_component_with_clone("Transform", 40)
    app.checksum_component(tf, 0, 12, assert_finite=True)
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_BOX_MOVE, [tf, vel]))
    app.rollback_resource_with_copy("FrameCount", bytes(4)).checksum_resource_with_hash("FrameCount")
    app.add_systems(GgrsSchedule, ResourceSystem(increase_frame_system))

    def setup(a):
        first = a.world.spawn(2)
        t = np.zeros((2, 10), np.float32)
        for h in range(2):
            rot = np.float32(h) / np.float32(2) * np.float32(2.0) * np.float32(np.pi)
            t[h, 0] = 1.25 * np.cos(rot); t[h, 1] = 0.1; t[h, 2] = 1.25 * np.sin(rot)
            t[h, 6] = 1.0; t[h, 7:10] = 1.0
        a.world.write_component(tf, first, t)
    app.add_systems(Startup, setup)
    return app, tf, vel


def frame_count(app):
    return struct.unpack("<I", app.resources["FrameCount"])[0]


def source_checkpoint(flags, ticks=20):
    """The App checkpoint of a frame a SyncTest box_game App saved after ``ticks`` ticks: (blob, frame)."""
    app, _, _ = box_app(flags, Session.SyncTest(SyncTestSession(2, 8, 9, input_delay=2)))
    for _ in range(ticks):
        app.step()
    f = sorted(app.world.snapshot_frames())[-3]
    return app.checkpoint(f), f


def restored(blob, flags, session=None, stream=None):
    app, _, _ = box_app(flags, session, stream)
    app.finish()
    app.restore_checkpoint(blob)
    return app


def world(app):
    return app.world.rollback_frame_count(), app.world.read_component(VEL, 0, 2).tobytes(), app.world.read_component(TF, 0, 2).tobytes()


def resources(app):
    return {n: bytes(v) for n, v in app.resources.items()}, app._res_frame


def state(app):
    """Everything a replay may change, and the resource store and ring it must not."""
    return world(app), resources(app), dict(app._res_store), sorted(app.world.snapshot_frames())


def log_of(n, seed):
    return np.random.default_rng(seed).integers(0, 16, (n, 2), dtype=np.uint8)


def stream_vectors(f0, log, k):
    """The request stream a replay stands for, in vectors of at most BGR_MAX_REQUESTS requests."""
    vecs, cur = [], []
    for j, row in enumerate(log):
        reqs = ([Request(SAVE, f0 + j)] if k and (f0 + j) % k == 0 else []) + [Request(ADVANCE, 0, [int(v) for v in row])]
        if len(cur) + len(reqs) > capi.BGR_MAX_REQUESTS:
            vecs.append(cur)
            cur = []
        cur += reqs
    return vecs + ([cur] if cur else [])


class RecordingP2P(P2PTraceSession):
    """A P2P trace session that records the inputs of the frames it advances: the confirmed input log."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.log = {}

    def advance_frame(self):
        f = self.current_frame
        reqs = super().advance_frame()
        for r in reqs:
            if r.kind == LOAD:
                f = r.frame
            elif r.kind == ADVANCE:
                self.log[f] = list(r.inputs)
                f += 1
        return reqs


@pytest.mark.parametrize("interval", [5, 10])
def test_p2p_checksum_reports_equal_the_replay_of_the_match(flags, interval):
    sess = RecordingP2P(2, 8, seed=31 + interval, p_clean=0.4, desync_interval=interval)
    a, _, _ = box_app(flags, Session.P2PTrace(sess))
    reports = {}
    a.step()
    first = a.checkpoint(0)
    reports.update(sess.checksum_reports())
    for _ in range(119):
        a.step()
        reports.update(sess.checksum_reports())
    assert len(reports) >= 100 // interval
    log = np.array([sess.log[f] for f in range(120)], np.uint8)
    b = restored(first, flags)
    got = dict(b.replay(log[:47], interval) + b.replay(log[47:], interval))
    assert {f: got[f] for f in reports} == reports
    assert frame_count(b) == frame_count(a) == 120 and world(b) == world(a)
    # without the resource parts, the same replay's checksums cannot equal the peers'
    c = restored(first, flags)
    engine_only = dict(c.world.replay(log, interval))
    assert all(engine_only[f] != reports[f] for f in reports)
    assert world(c) == world(a)


@pytest.mark.parametrize("interval", [1, 7, 10])
def test_replay_equals_the_request_stream_through_the_host_half(flags, interval):
    blob, f0 = source_checkpoint(flags)
    a = restored(blob, flags)
    whole = restored(blob, flags)
    twin = restored(blob, flags, Session(Session.SPECTATOR, SessionInfo(SPECTATOR)))
    before_store = dict(a._res_store)
    log = log_of(230, interval)
    cuts = [0, 1, 2, 40, 97, 170, 230]
    cs = []
    for s, e in zip(cuts, cuts[1:]):
        cs += a.replay(log[s:e], interval)
        stream_cs = []
        for v in stream_vectors(f0 + s, log[s:e], interval):
            twin.handle_requests(v)
            stream_cs += twin.last_checksums
        assert cs[len(cs) - len(stream_cs):] == stream_cs
        assert world(a) == world(twin) and resources(a) == resources(twin)
        assert a._res_frame == a.rollback_frame_count() == f0 + e
    assert cs == whole.replay(log, interval)
    assert state(whole) == state(a)
    assert [f for f, _ in cs] == [f for f in range(f0, f0 + 230) if f % interval == 0]
    assert frame_count(a) == f0 + 230 and a._res_store == before_store and a.world.snapshot_frames() == [f0]


def test_keyframes_are_the_checkpoints_of_a_ticking_twin(flags):
    blob, f0 = source_checkpoint(flags)
    a = restored(blob, flags)
    plain = restored(blob, flags)
    info = SessionInfo(None)
    twin = restored(blob, flags, Session(Session.P2P, info))
    log = log_of(130, 3)
    cs, kfs = a.replay_keyframes(log, 10, 11)
    assert cs == plain.replay(log, 10) and state(a) == state(plain)
    expected = []
    for j, row in enumerate(log):
        f = f0 + j
        info.value = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))  # confirms every frame before the current one
        if f % 11 == 0:
            twin.handle_requests([Request(SAVE, f)])
            expected.append((f, twin.checkpoint(f)))
        twin.handle_requests([Request(ADVANCE, 0, [int(v) for v in row])])
    assert [f for f, _ in kfs] == [f for f in range(f0, f0 + 130) if f % 11 == 0]
    assert kfs == expected
    assert world(twin) == world(a) and resources(twin) == resources(a)
    seek = restored(blob, flags)
    for f, kf in (kfs[0], kfs[len(kfs) // 2], kfs[-1]):
        seek.restore_checkpoint(kf)
        assert seek.replay(log[f - f0:], 10) == [c for c in cs if c[0] >= f]
        assert world(seek) == world(a) and resources(seek) == resources(a)


def test_trace_records_the_world_and_checksums_the_resources(flags):
    blob, f0 = source_checkpoint(flags)
    a, b = restored(blob, flags), restored(blob, flags)
    log = log_of(90, 4)
    cs, samples, records = a.replay_trace(log, 10, 6, [(TF, 0, 12)], 0, 2)
    engine_cs, engine_samples, engine_records = b.world.replay_trace(log, 10, 6, [(TF, 0, 12)], 0, 2)
    assert samples == engine_samples and np.array_equal(records, engine_records)
    assert [f for f, _ in cs] == [f for f, _ in engine_cs] and all(x != y for (_, x), (_, y) in zip(cs, engine_cs))
    assert cs == restored(blob, flags).replay(log, 10)
    assert frame_count(a) == f0 + 90 and a._res_frame == f0 + 90


def test_a_frame_saved_before_a_replay_still_loads_with_its_resources(flags):
    app, _, _ = box_app(flags, Session.SyncTest(SyncTestSession(2, 8, 9, input_delay=2)))
    for _ in range(20):
        app.step()
    f = sorted(app.world.snapshot_frames())[-2]
    twin = restored(app.checkpoint(f), flags)
    app.replay(log_of(50, 5), 10)
    app.handle_requests([Request(LOAD, f)])
    assert resources(app) == resources(twin) and app._res_frame == f and world(app) == world(twin)
    log = log_of(30, 6)
    assert app.replay(log, 10) == twin.replay(log, 10)
    assert world(app) == world(twin) and resources(app) == resources(twin)


def test_refused_replays_change_nothing(flags):
    blob, f0 = source_checkpoint(flags)
    app = restored(blob, flags)
    log = log_of(40, 7)
    before = state(app)
    calls = [lambda x: app.replay(x, 10), lambda x: app.replay_keyframes(x, 10, 8),
             lambda x: app.replay_trace(x, 10, 4, [(TF, 0, 12)], 0, 2)]
    # the App's resources out of step with its world
    app.world.set_rollback_frame_count(f0 + 3)
    for call in calls:
        with pytest.raises(BgrError) as e:
            call(log)
        assert e.value.status == capi.BGR_ERR_STATE
    app.world.set_rollback_frame_count(f0)
    assert state(app) == before
    # un-collected submits: the engine refuses after the resources were stepped on their copy
    app.world.submit_requests((capi.BGR_SESSION_NONE, 0, 0, 0), [Request(SAVE, f0)])
    for call in calls:
        with pytest.raises(BgrError) as e:
            call(log)
        assert e.value.status == capi.BGR_ERR_STATE
        assert resources(app) == before[1] and app._res_store == before[2]
    app.world.collect()
    assert state(app) == before
    # a log the engine refuses (n_players > BGR_MAX_PLAYERS)
    for call in calls:
        with pytest.raises(BgrError) as e:
            call(np.zeros((5, 9), np.uint8))
        assert e.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    assert state(app) == before
    # host-side component tables
    hosted, _, _ = box_app(flags)
    hosted.rollback_component_with_clone("Sprite")
    hosted.finish()
    hosted_before = state(hosted)
    for call in (lambda: hosted.replay(log, 10), lambda: hosted.replay_keyframes(log, 10, 8),
                 lambda: hosted.replay_trace(log, 10, 4, [(TF, 0, 12)], 0, 2)):
        with pytest.raises(BgrError, match="host-side component tables") as e:
            call()
        assert e.value.status == capi.BGR_ERR_UNSUPPORTED
    assert state(hosted) == hosted_before
    # the replay still runs and is equal to a twin's
    assert app.replay(log, 10) == restored(blob, flags).replay(log, 10)


def test_non_finite_replay_commits_the_resources(flags):
    blob, f0 = source_checkpoint(flags)
    app, plain = restored(blob, flags), restored(blob, flags)
    for a in (app, plain):
        t = a.world.read_component(TF, 0, 2).view(np.float32).copy()
        t[1, 0] = np.nan
        a.world.write_component(TF, 0, t)
    log = log_of(25, 8)
    with pytest.raises(BgrError) as e:
        app.replay(log, 1)
    assert e.value.status == capi.BGR_ERR_NON_FINITE
    with pytest.raises(BgrError):
        plain.world.replay(log, 1)
    assert world(app) == world(plain)
    assert app._res_frame == app.rollback_frame_count() == f0 + 25 and frame_count(app) == f0 + 25


def test_batches_equal_each_apps_own_replay(batch_flags, stream):
    flags = batch_flags
    blob, f0 = source_checkpoint(flags)
    apps = [restored(blob, flags, stream=stream) for _ in range(16)]
    twins = [restored(blob, flags) for _ in range(16)]
    batch = EngineBatch([a.world for a in apps])
    rng = np.random.default_rng(9)
    fields = [(0, 0, 12), (1, 0, 12)]
    for rnd in range(6):
        subset = [int(i) for i in rng.choice(16, int(rng.integers(1, 17)), replace=False)]
        logs = {i: log_of(int(rng.integers(1, 70)), 100 * rnd + i) for i in subset}
        ks = {i: int(rng.choice([0, 1, 7, 10])) for i in subset}
        if rnd % 3 == 0:
            got = replay_batch([(apps[i], logs[i], ks[i]) for i in subset], batch)
            want = [twins[i].replay(logs[i], ks[i]) for i in subset]
        elif rnd % 3 == 1:
            got = replay_keyframes_batch([(apps[i], logs[i], ks[i], 1 + i) for i in subset], batch)
            want = [twins[i].replay_keyframes(logs[i], ks[i], 1 + i) for i in subset]
        else:
            got = replay_trace_batch([(apps[i], logs[i], ks[i], 1 + i % 5, i % 2, 2 - i % 2) for i in subset], batch, fields)
            want = [twins[i].replay_trace(logs[i], ks[i], 1 + i % 5, fields, i % 2, 2 - i % 2) for i in subset]
            got = [(cs, s, r.tobytes()) for cs, s, r in got]
            want = [(cs, s, r.tobytes()) for cs, s, r in want]
        assert got == want, f"round {rnd}"
        for i in range(16):
            assert state(apps[i]) == state(twins[i]), f"round {rnd}, App {i}"


def test_batch_commits_every_app_before_raising_non_finite(batch_flags, stream):
    flags = batch_flags
    blob, f0 = source_checkpoint(flags)
    apps = [restored(blob, flags, stream=stream) for _ in range(4)]
    t = apps[2].world.read_component(TF, 0, 2).view(np.float32).copy()
    t[0, 1] = np.inf
    apps[2].world.write_component(TF, 0, t)
    batch = EngineBatch([a.world for a in apps])
    logs = [log_of(33, 20 + i) for i in range(4)]
    with pytest.raises(BgrError) as e:
        replay_batch([(apps[i], logs[i], 1) for i in range(4)], batch)
    assert e.value.status == capi.BGR_ERR_NON_FINITE and "world 2" in str(e.value)
    for i in range(4):
        assert apps[i]._res_frame == apps[i].rollback_frame_count() == f0 + 33 and frame_count(apps[i]) == f0 + 33
    # a refused batch (an App listed twice) commits nothing
    before = [state(a) for a in apps]
    with pytest.raises(BgrError):
        replay_batch([(apps[0], logs[0], 1), (apps[0], logs[1], 1)], batch)
    assert [state(a) for a in apps] == before
