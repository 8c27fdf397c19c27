"""The host half of App replays (plugin.py: App.replay / replay_keyframes / replay_trace and the batch calls) over a
stand-in engine whose world is its frame counter, so it runs without a GPU.  A replay must leave the App as the host half
of handle_requests leaves it after [Save(f) if f % k == 0, Advance(inputs[j])]: resource parts XORed into the engine's
checksums, keyframes that are App checkpoints, resources committed when the engine ran the log (BGR_OK or
BGR_ERR_NON_FINITE) and untouched by every refusal.  tests/test_gpu_app_replay.py holds the same on the engine."""
import struct

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.plugin import (App, GgrsSchedule, ResourceSystem, Session, replay_batch, replay_keyframes_batch,
                                   replay_trace_batch)
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request

MASK = (1 << 128) - 1


def engine_checksum(f):
    return (f * 0x9E3779B97F4A7C15_5851F42D4C957F2D) & MASK


class FrameEngine:
    """The Engine calls an App's replay makes, over a world that is only RollbackFrameCount.  ``refuse`` makes the next
    replay raise that status before running; ``non_finite`` makes replays run and then raise BGR_ERR_NON_FINITE."""

    def __init__(self):
        self.frame, self.ring, self.refuse, self.non_finite = 0, set(), None, False

    def build(self):
        pass

    def rollback_frame_count(self):
        return self.frame

    def snapshot_frames(self):
        return sorted(self.ring)

    def handle_requests(self, info, requests):
        out = []
        for r in requests:
            if r.kind == SAVE:
                self.ring.add(self.frame)
                out.append((self.frame, engine_checksum(self.frame)))
            else:
                self.frame += 1
        return out

    def checkpoint(self, f):
        return b"engine blob %d|" % f if f in self.ring else None

    def _run(self, n, k):
        if self.refuse is not None:
            raise BgrError(self.refuse, "refused")
        f0, self.frame = self.frame, self.frame + n
        if self.non_finite:
            raise BgrError(capi.BGR_ERR_NON_FINITE, "Hashing is not stable for NaN f32 values.")
        return [(f, engine_checksum(f)) for f in range(f0, f0 + n) if k and f % k == 0]

    def replay(self, inputs, k=0):
        return self._run(len(inputs), k)

    def replay_keyframes(self, inputs, k, kk):
        f0 = self.frame
        return self._run(len(inputs), k), [(f, b"engine blob %d|" % f) for f in range(f0, f0 + len(inputs)) if f % kk == 0]

    def replay_trace(self, inputs, k, tt, fields, first_row, n_rows):
        f0 = self.frame
        frames = [f for f in range(f0, f0 + len(inputs)) if f % tt == 0]
        return self._run(len(inputs), k), [(f, n_rows) for f in frames], np.zeros((len(frames), n_rows, 8), np.uint8)


class FrameBatch:
    """EngineBatch's replay calls over FrameEngines: per-world (status, results...), a refusal raising for all."""

    def __init__(self, engines):
        self.engines = list(engines)

    def _each(self, calls, fn, empty):
        if len({c[0] for c in calls}) != len(calls):
            raise BgrError(capi.BGR_ERR_INVALID_ARGUMENT, "listed twice in one call")
        out = []
        for c in calls:
            try:
                r = fn(self.engines[c[0]], *c[1:])
                out.append((capi.BGR_OK,) + (r if isinstance(r, tuple) else (r,)))
            except BgrError as e:
                out.append((e.status,) + empty)
        return out

    def replay(self, calls):
        return self._each(calls, FrameEngine.replay, ([],))

    def replay_keyframes(self, calls):
        return self._each(calls, FrameEngine.replay_keyframes, ([], []))

    def replay_trace(self, calls, fields):
        return self._each([c[:4] + (fields,) + c[4:] for c in calls], FrameEngine.replay_trace, ([], [], None))


def bump(res, frame):  # increase_frame_system with the frame the tick's host half passes
    res["FrameCount"][:] = struct.pack("<I", struct.unpack("<I", res["FrameCount"])[0] + 1)
    res["Seen"][:] = struct.pack("<I", frame)


def app_of(engine=None):
    app = App(engine or FrameEngine())
    app.rollback_resource_with_copy("FrameCount", bytes(4)).checksum_resource_with_hash("FrameCount")
    app.rollback_resource_with_copy("Seen", bytes(4))
    app.rollback_resource_with_copy("Absent")
    app.add_systems(GgrsSchedule, ResourceSystem(bump))
    return app.finish()


class Info:
    def info(self):
        return (capi.BGR_SESSION_NONE, 0, 0, 0)

    def save_cell(self, frame, checksum):
        pass


def streamed(app, f0, n, k, kk=0):
    """The equivalent request stream through the App's host half, with App.checkpoint at the keyframe frames."""
    app.insert_resource(Session(Session.P2P, Info()))
    cs, kfs = [], []
    for f in range(f0, f0 + n):
        if (k and f % k == 0) or (kk and f % kk == 0):
            app.handle_requests([Request(SAVE, f)])
            if k and f % k == 0:
                cs += app.last_checksums
            if kk and f % kk == 0:
                kfs.append((f, app.checkpoint(f)))
        app.handle_requests([Request(ADVANCE, 0, [0, 0])])
    return cs, kfs


def host_state(app):
    return {n: bytes(v) for n, v in app.resources.items()}, app._res_frame, app.world.frame


@pytest.mark.parametrize("k,kk", [(1, 1), (7, 3), (10, 11), (0, 4)])
def test_replays_equal_the_stream_through_the_host_half(k, kk):
    a, b, c = app_of(), app_of(), app_of()
    log = np.zeros((95, 2), np.uint8)
    cs = a.replay(log[:30], k) + a.replay(log[30:], k)
    cs_b, _ = streamed(b, 0, 95, k)
    assert cs == cs_b and host_state(a) == host_state(b)
    assert struct.unpack("<I", a.resources["Seen"])[0] == 95 and "Absent" not in a.resources
    assert all(c != engine_checksum(f) for f, c in cs)
    assert a._res_store == {}                     # no snapshot was pushed
    cs_c, kfs = c.replay_keyframes(log, k, kk)
    twin = app_of()
    _, kfs_twin = streamed(twin, 0, 95, 0, kk)
    assert cs_c == cs and kfs == kfs_twin and host_state(c) == host_state(a)
    d = app_of()
    cs_d, samples, records = d.replay_trace(log, k, 5, [(0, 0, 8)], 0, 2)
    assert cs_d == cs and [f for f, _ in samples] == list(range(0, 95, 5)) and host_state(d) == host_state(a)


def test_restoring_a_keyframe_and_replaying_the_rest_ends_the_same():
    a = app_of()
    log = np.zeros((60, 2), np.uint8)
    cs, kfs = a.replay_keyframes(log, 4, 16)
    for f, blob in kfs:
        seek = app_of()
        seek.world.ring.add(f)
        seek._set_restored_resources(f, seek._parse_resources(blob, blob.index(b"|") + 1, "checkpoint"))
        seek.world.frame = f
        assert seek.replay(log[f:], 4) == [x for x in cs if x[0] >= f]
        assert host_state(seek) == host_state(a)


def test_refusals_change_nothing_and_non_finite_commits():
    app = app_of()
    app.replay(np.zeros((13, 2), np.uint8), 5)
    before = host_state(app)
    app.world.frame += 1                           # the App's resources out of step with its world
    with pytest.raises(BgrError) as e:
        app.replay(np.zeros((4, 2), np.uint8), 1)
    assert e.value.status == capi.BGR_ERR_STATE
    app.world.frame -= 1
    for status in (capi.BGR_ERR_STATE, capi.BGR_ERR_INVALID_ARGUMENT, capi.BGR_ERR_CAPACITY):
        app.world.refuse = status
        for call in (lambda: app.replay(np.zeros((4, 2), np.uint8), 1),
                     lambda: app.replay_keyframes(np.zeros((4, 2), np.uint8), 1, 2),
                     lambda: app.replay_trace(np.zeros((4, 2), np.uint8), 1, 2, [(0, 0, 8)], 0, 1)):
            with pytest.raises(BgrError) as e:
                call()
            assert e.value.status == status and host_state(app) == before
    app.world.refuse, app.world.non_finite = None, True
    with pytest.raises(BgrError) as e:
        app.replay(np.zeros((4, 2), np.uint8), 1)
    assert e.value.status == capi.BGR_ERR_NON_FINITE
    assert app._res_frame == app.world.frame == 17 and struct.unpack("<I", app.resources["FrameCount"])[0] == 17
    hosted = app_of()
    hosted.rollback_component_with_clone("Sprite")
    with pytest.raises(BgrError, match="host-side component tables") as e:
        hosted.replay(np.zeros((4, 2), np.uint8), 1)
    assert e.value.status == capi.BGR_ERR_UNSUPPORTED and hosted.world.frame == 0


def test_an_absent_checksummed_resource_fails_before_anything_runs():
    app = App(FrameEngine())
    app.rollback_resource_with_copy("Wallet").checksum_resource_with_hash("Wallet")
    app.finish()
    with pytest.raises(KeyError):
        app.replay(np.zeros((3, 2), np.uint8), 1)
    assert app.world.frame == 0 and app._res_frame == 0


def test_batches_equal_each_apps_own_replay_and_commit_before_raising():
    apps = [app_of() for _ in range(5)]
    twins = [app_of() for _ in range(5)]
    batch = FrameBatch([a.world for a in apps])
    rng = np.random.default_rng(1)
    for rnd in range(9):
        subset = [int(i) for i in rng.choice(5, int(rng.integers(1, 6)), replace=False)]
        logs = {i: np.zeros((int(rng.integers(0, 40)), 2), np.uint8) for i in subset}
        if rnd % 3 == 0:
            got = replay_batch([(apps[i], logs[i], 1 + i) for i in subset], batch)
            want = [twins[i].replay(logs[i], 1 + i) for i in subset]
        elif rnd % 3 == 1:
            got = replay_keyframes_batch([(apps[i], logs[i], 1 + i, 3) for i in subset], batch)
            want = [twins[i].replay_keyframes(logs[i], 1 + i, 3) for i in subset]
        else:
            got = replay_trace_batch([(apps[i], logs[i], 1 + i, 2, 0, 1) for i in subset], batch, [(0, 0, 8)])
            want = [twins[i].replay_trace(logs[i], 1 + i, 2, [(0, 0, 8)], 0, 1) for i in subset]
            got = [(cs, s, r.tobytes()) for cs, s, r in got]
            want = [(cs, s, r.tobytes()) for cs, s, r in want]
        assert got == want
        assert [host_state(a) for a in apps] == [host_state(t) for t in twins]
    before = [host_state(a) for a in apps]
    with pytest.raises(BgrError):
        replay_batch([(apps[0], np.zeros((3, 2), np.uint8), 1), (apps[0], np.zeros((3, 2), np.uint8), 1)], batch)
    assert [host_state(a) for a in apps] == before
    apps[3].world.non_finite = True
    with pytest.raises(BgrError, match="world 3") as e:
        replay_batch([(a, np.zeros((6, 2), np.uint8), 2) for a in apps], batch)
    assert e.value.status == capi.BGR_ERR_NON_FINITE
    assert all(a._res_frame == a.world.frame == b[1] + 6 for a, b in zip(apps, before))
