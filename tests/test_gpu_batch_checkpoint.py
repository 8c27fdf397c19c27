"""Batched checkpoints (bgr_batch_checkpoint_save / bgr_batch_checkpoint_restore, EngineBatch.checkpoint / .restore):
the blobs of a batched save equal each member's own bgr_checkpoint_save byte for byte, a batched restore leaves each
listed member as its own bgr_checkpoint_restore leaves a twin (then both tick identically), a refused call changes no
world, and one call's launches do not grow with the number of worlds.  Members differ in rows, order_base, depth,
BGR_CFG_DESYNC_CAPTURE, BGR_CFG_GROWABLE and retained frames.  Every test runs with the batch specialised and not
(BGR_TUNE_JIT=0): the checkpoint kernels do not depend on it."""
import ctypes as C
import struct

import numpy as np
import pytest

import checkpoint_codec as cc
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine, EngineBatch
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request

from test_gpu_batch import presence_world
from test_gpu_generic_spawn import spawn_world
from test_gpu_replay import FIN, live, log_for

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]
ROWS = [1, 127, 700, 2000, 129, 40]


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


def box_member(n, depth, stream=None, flags=0, order_base=0, seed=0, fps=60, retain=0):
    """box_game's Velocity / Transform with move_cube_system (retain: keep 3 confirmed frames every `retain`)."""
    w = Engine(max_entities=n + 8, max_depth=depth, flags=flags, order_base=order_base, stream=stream, fps=fps)
    vel = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    tf = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
    w.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
    w.checksum_component(tf, 0, 12, FIN)
    w.checksum_component(vel, 0, 12)
    if retain:
        w.retain_confirmed(retain, 3)
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(seed)
    t = np.zeros((n, 10), np.float32)
    t[:, 0:3] = rng.uniform(-2, 2, (n, 3)); t[:, 6] = 1.0; t[:, 7:10] = 1.0
    w.write_component(tf, 0, t)
    w.write_component(vel, 0, rng.uniform(-1, 1, (n, 3)).astype(np.float32))
    return w


def odd_member(n, depth, stream=None, seed=0, order_base=0):
    """A 5-byte column (3 bytes of its second word past the element) and an optional u32 counter."""
    e = Engine(max_entities=n + 8, max_depth=depth, stream=stream, order_base=order_base)
    a = e.rollback_component("Odd", 5, capi.BGR_STRATEGY_COPY)
    b = e.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)
    e.checksum_component(a, 0, 5)
    e.add_system(capi.BGR_SYS_U32_ADD, [b], [0, 1])
    e.build()
    e.spawn(n)
    rng = np.random.default_rng(seed)
    e.write_component(a, 0, rng.integers(0, 256, (n, 5), dtype=np.uint8))
    e.write_component(b, 0, rng.integers(0, 99, n, dtype=np.uint32))
    return e


def member_kw(i):
    """What members of one batch may differ in: depth, desync capture, retained frames, order_base."""
    return dict(depth=4 + i % 3, flags=capi.BGR_CFG_DESYNC_CAPTURE if i % 2 else 0, retain=4 if i % 3 == 0 else 0,
                order_base=(1 << 32) - 700 if i % 4 == 3 else 0)


MAKERS = {
    "box": lambda i, s: box_member(ROWS[i % 6], stream=s, seed=i, **member_kw(i)),
    "presence": lambda i, s: presence_world(ROWS[i % 6] + 1300, 4 + i % 3, stream=s, seed=i, order_base=member_kw(i)["order_base"]),
    "spawning_fixed": lambda i, s: spawn_world(ROWS[i % 6], 4 + i % 3, stream=s, seed=i),
    "spawning_growable": lambda i, s: spawn_world(ROWS[i % 6], 4 + i % 3, stream=s, seed=i, flags=capi.BGR_CFG_GROWABLE,
                                                  cap=ROWS[i % 6] + 64),
}


def pair(make, stream, n):
    """Members on the batch stream and twins on their own streams, built alike."""
    return [make(i, stream) for i in range(n)], [make(i, None) for i in range(n)]


def drive(e, frames, seed, spawn=False):
    """P2P vectors of Save(f), Advance that confirm every frame before the current one (retained frames fill up)."""
    log = log_for(frames, 2, seed, spawn_every=4 if spawn else 0)
    out = []
    for row in log:
        f = e.rollback_frame_count()
        info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))
        out += e.handle_requests(info, [Request(SAVE, f), Request(ADVANCE, 0, [int(v) for v in row])])
    return out


def vectors(f, rng, spawn):
    """A P2P tick or a SyncTest-like rollback of one frame, from frame f."""
    a = [int(v) for v in rng.integers(0, 16, 2)]
    if spawn and rng.random() < 0.3:
        a[0] |= capi.BGR_INPUT_SPAWN
    if rng.random() < 0.4:
        return [Request(SAVE, f), Request(ADVANCE, 0, a), Request(LOAD, f), Request(ADVANCE, 0, a), Request(SAVE, f + 1)]
    return [Request(SAVE, f), Request(ADVANCE, 0, a)]


def state(e):
    f = e.rollback_frame_count()
    d = e.frame_digest(f)
    world = live(e) if e.row_count() else (f, 0, e.active_count())
    return world, e.snapshot_frames(), e.retained_frames(), None if d is None else (d[0].root, d[0].active)


def tick_pair(batch, members, twins, worlds, n_ticks, seed, spawn):
    rng = np.random.default_rng(seed)
    for t in range(n_ticks):
        calls = []
        for w in worlds:
            f = members[w].rollback_frame_count()
            reqs = vectors(f, rng, spawn)
            calls.append((w, (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1)), reqs))
        res = batch.handle_requests(calls)
        for (w, info, reqs), (status, cs) in zip(calls, res):
            assert status == capi.BGR_OK
            assert cs == twins[w].handle_requests(info, reqs), f"world {w} tick {t}"


def save_raw(batch, worlds, frames, cap=None, query=False):
    n = len(worlds)
    w = (C.c_uint32 * n)(*worlds)
    fr = (C.c_int32 * n)(*frames)
    index = (capi.bgr_keyframe * n)()
    size = C.c_size_t()
    status = (C.c_int32 * n)()
    buf = None if query else np.full(max(1, cap), 0xFF, np.uint8)   # padding the call leaves alone would show
    rc = batch._lib.bgr_batch_checkpoint_save(batch._h, w, n, fr, None if query else buf.ctypes.data, 0 if query else cap,
                                              index, C.byref(size), status)
    return rc, [(index[i].frame, index[i].offset, index[i].bytes) for i in range(n)], size.value, list(status), buf


@pytest.mark.parametrize("name", list(MAKERS))
def test_batched_save_equals_each_members_checkpoint(stream, name):
    spawn = name.startswith("spawning")
    members, twins = pair(MAKERS[name], stream, 6)
    batch = EngineBatch(members)
    for i, (m, t) in enumerate(zip(members, twins)):
        assert drive(m, 9 + i, seed=i, spawn=spawn) == drive(t, 9 + i, seed=i, spawn=spawn)
    # the newest queued frames (world 3: a frame no world holds), then the oldest retained or queued ones
    rounds = [[(w, m.snapshot_frames()[-1]) for w, m in enumerate(members) if w != 3] + [(3, 10 ** 6)],
              [(w, (m.retained_frames() or m.snapshot_frames())[0]) for w, m in enumerate(members)][::-1]]
    assert any(m.retained_frames() for m in members) or not name == "box"
    for rnd in rounds:
        got = batch.checkpoint(rnd)
        assert got == [members[w].checkpoint(f) for w, f in rnd]
        assert got == [twins[w].checkpoint(f) for w, f in rnd]
        for (w, f), blob in zip(rnd, got):
            assert (blob is None) == (f == 10 ** 6)
    # the query runs nothing and bounds every blob; a short dst_cap is refused with the exact total
    rnd = rounds[0]
    worlds, frames = [w for w, _ in rnd], [f for _, f in rnd]
    launches = [m.launch_count() for m in members]
    rc, bound, total_bound, _, _ = save_raw(batch, worlds, frames, query=True)
    assert rc == capi.BGR_OK and [m.launch_count() for m in members] == launches
    blobs = batch.checkpoint(rnd)
    for (_, off, b), blob in zip(bound, blobs):
        assert off % 8 == 0 and (blob is None and b == 0 or len(blob) <= b)
    rc, index, total, _, buf = save_raw(batch, worlds, frames, cap=total_bound)
    assert rc == capi.BGR_OK
    padding = np.ones(total, bool)
    for (f, off, b), blob in zip(index, blobs):
        assert off % 8 == 0 and bytes(buf[off:off + b]) == (blob or b"")
        padding[off:off + b] = False
    assert total == (index[-1][1] + index[-1][2] + 7) // 8 * 8 and total <= total_bound
    assert not buf[:total][padding].any(), "the padding between and after the blobs is zero"
    rc, index2, total2, _, buf = save_raw(batch, worlds, frames, cap=total - 1)
    assert rc == capi.BGR_ERR_CAPACITY and total2 == total and (buf == 0xFF).all()


def test_batched_save_with_submits_in_flight_and_a_zero_row_world(stream):
    members = [box_member(0 if i == 2 else 300 + 100 * i, 4, stream=stream, seed=i) for i in range(4)]
    twins = [box_member(0 if i == 2 else 300 + 100 * i, 4, seed=i) for i in range(4)]
    batch = EngineBatch(members)
    for m, t in zip(members, twins):
        assert drive(m, 5, seed=1) == drive(t, 5, seed=1)
    f = members[1].rollback_frame_count()
    info = (capi.BGR_SESSION_P2P, 7, 0, f - 1)
    reqs = [Request(SAVE, f), Request(ADVANCE, 0, [3, 4])]
    members[1].submit_requests(info, reqs)
    got = batch.checkpoint([(1, f), (2, 4), (0, 4)])
    expect_cs = twins[1].handle_requests(info, reqs)
    assert members[1].collect() == expect_cs   # the result stayed queued
    assert got == [twins[1].checkpoint(f), twins[2].checkpoint(4), twins[0].checkpoint(4)]
    assert cc.unpack_header(got[1])["rows"] == 0
    batch.restore([(2, got[1]), (0, got[2])])
    twins[2].restore(got[1])
    twins[0].restore(got[2])
    for w in (0, 2):
        assert state(members[w]) == state(twins[w])


@pytest.mark.parametrize("name", list(MAKERS))
def test_batched_restore_equals_each_members_restore(stream, name):
    spawn = name.startswith("spawning")
    members, twins = pair(MAKERS[name], stream, 6)
    batch = EngineBatch(members)
    # the blobs: each world's own frame from a third engine of its kind that ran a different match
    srcs = [MAKERS[name](i, None) for i in range(6)]
    blobs = []
    for i, s in enumerate(srcs):
        drive(s, 14 + 3 * i, seed=50 + i, spawn=spawn)
        blobs.append(s.checkpoint(s.snapshot_frames()[-1 - i % 2]))
    for i, (m, t) in enumerate(zip(members, twins)):
        assert drive(m, 6, seed=i, spawn=spawn) == drive(t, 6, seed=i, spawn=spawn)
    # box and presence: world 3 has order_base 2^32 - 700, the others 0.  It is listed first, then after worlds of 0
    for rnd, listed in enumerate(([3, 0, 2, 5], [4, 1, 3])):
        unlisted_before = {w: state(members[w]) for w in range(6) if w not in listed}
        batch.restore([(w, blobs[w]) for w in listed])
        for w in listed:
            twins[w].restore(blobs[w])
            assert state(members[w]) == state(twins[w]), f"world {w}"
            assert members[w].checkpoint(members[w].rollback_frame_count()) == blobs[w]
        for w, before in unlisted_before.items():
            assert state(members[w]) == before, f"unlisted world {w}"
        tick_pair(batch, members, twins, list(range(6)), 15, seed=7 + rnd, spawn=spawn)
        for w in range(6):
            assert state(members[w]) == state(twins[w]), f"world {w}"


def test_cross_restores_and_growth(stream):
    ms = [box_member(300, 4, stream=stream, seed=0), box_member(900, 4, stream=stream, seed=1),
          box_member(300, 4, stream=stream, seed=2, order_base=1000), box_member(300, 4, stream=stream, seed=3, fps=30)]
    batch = EngineBatch(ms)
    for m in ms:
        drive(m, 4, seed=2)
    twin = box_member(300, 4, seed=0)
    drive(twin, 4, seed=2)
    blob0 = ms[0].checkpoint(3)
    batch.restore([(1, blob0), (0, blob0)])   # one blob for two worlds, one of them its writer
    twin.restore(blob0)
    assert live(ms[1])[1:] == live(twin)[1:] and live(ms[0]) == live(twin)
    for bad in (2, 3):   # another order_base, another fps
        before = [state(m) for m in ms]
        with pytest.raises(BgrError) as ei:
            batch.restore([(0, blob0), (bad, blob0)])
        assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and str(ei.value).startswith(f"world {bad}: ")
        assert [state(m) for m in ms] == before
    # a growable member grows to a larger blob; a fixed one refuses it
    g = [spawn_world(50, 4, stream=stream, seed=i, flags=capi.BGR_CFG_GROWABLE, cap=64) for i in range(2)]
    g.append(spawn_world(50, 4, stream=stream, seed=2, cap=64))
    big = spawn_world(50, 4, seed=0, cap=2000)
    drive(big, 30, seed=3, spawn=True)
    blob = big.checkpoint(big.snapshot_frames()[-1])
    assert cc.unpack_header(blob)["rows"] > 64
    gb = EngineBatch(g)
    before = [state(m) for m in g]
    with pytest.raises(BgrError) as ei:
        gb.restore([(0, blob), (2, blob)])
    assert ei.value.status == capi.BGR_ERR_CAPACITY and str(ei.value).startswith("world 2: ")
    assert [state(m) for m in g] == before
    gb.restore([(1, blob), (0, blob)])
    for m in g[:2]:
        assert m.capacity()[0] >= cc.unpack_header(blob)["rows"]
        assert m.checkpoint(m.rollback_frame_count()) == blob


def _corrupt_cases(blob, words):
    h = cc.unpack_header(blob)
    pre = 104 + 8 * (h["n_blocks"] + 1)
    _, planes, mask = cc.decode(blob, words)
    fields = {k: h[k] for k in ("layout", "frame", "rows", "n_columns", "fps", "active", "elapsed_ns", "rng", "digest_root")}
    r = int(np.nonzero(mask[0] & 1)[0][0])
    flipped = planes.copy()
    flipped[0, 0, r] ^= 1 << 9
    kind = bytearray(blob)
    kind[pre] = 3
    offs = bytearray(blob)
    struct.pack_into("<Q", offs, 104 + 8, struct.unpack_from("<Q", blob, 104 + 8)[0] + 4)
    return [("bad magic", b"XXXX" + blob[4:], capi.BGR_ERR_INVALID_ARGUMENT),
            ("truncated", blob[:-4], capi.BGR_ERR_INVALID_ARGUMENT),
            ("bad offsets", bytes(offs), capi.BGR_ERR_INVALID_ARGUMENT),
            ("digest mismatch", cc.encode(flipped, mask, **fields), capi.BGR_ERR_INVALID_ARGUMENT),
            ("bad kind byte", bytes(kind), capi.BGR_ERR_INVALID_ARGUMENT)], planes, mask, fields


def test_refusals_are_atomic(stream):
    ms = [odd_member(1000, 4, stream=stream, seed=i, order_base=(1 << 32) - 700 if i == 3 else 0) for i in range(4)]
    batch = EngineBatch(ms)
    for m in ms:
        drive(m, 3, seed=1)
    blob, blob3 = ms[0].checkpoint(2), ms[3].checkpoint(2)   # world 3 has another order_base than the others
    cases, planes, mask, fields = _corrupt_cases(blob, 3)
    stray = planes.copy()
    stray[1, 1, 700 - 512] |= np.uint32(1 << 31)   # row 700 exists and holds Odd: a bit past its fifth byte
    cases.append(("stray bits", cc.encode(stray, mask, **fields), capi.BGR_ERR_INVALID_ARGUMENT))
    for name, bad, status in cases:
        before = [state(m) for m in ms]
        with pytest.raises(BgrError) as ei:
            batch.restore([(3, blob3), (0, blob), (2, bad), (1, blob)])
        assert ei.value.status == status, name
        assert str(ei.value).startswith("world 2: "), (name, str(ei.value))
        assert [state(m) for m in ms] == before, name
    ms[3].submit_requests((capi.BGR_SESSION_NONE, 0, 0, 0), [Request(ADVANCE, 0, [1])])
    before = [state(m) for m in ms[:3]]
    with pytest.raises(BgrError) as ei:
        batch.restore([(0, blob), (3, blob3), (1, blob)])
    assert ei.value.status == capi.BGR_ERR_STATE and str(ei.value).startswith("world 3: ")
    ms[3].collect()
    assert [state(m) for m in ms[:3]] == before
    for bad, prefix in (([(0, blob), (1, blob), (0, blob)], "world 0: "), ([(1, blob), (9, blob)], "world 9: ")):
        before = [state(m) for m in ms]
        with pytest.raises(BgrError) as ei:
            batch.restore(bad)
        assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and str(ei.value).startswith(prefix)
        assert [state(m) for m in ms] == before
    for bad, prefix in (([(0, 2), (0, 2)], "world 0: "), ([(5, 2)], "world 5: ")):
        with pytest.raises(BgrError) as ei:
            batch.checkpoint(bad)
        assert str(ei.value).startswith(prefix)
    batch.restore([(3, blob3), (0, blob), (2, blob)])   # the valid blobs of the refused calls restore
    assert [ms[w].checkpoint(2) for w in (3, 0, 2)] == [blob3, blob, blob]


def test_seek_by_batched_restore_then_batched_replay(stream):
    n, kk = 5, 20
    members = [box_member(ROWS[i] + 200, 4, stream=stream, seed=i) for i in range(n)]
    full = [box_member(ROWS[i] + 200, 4, seed=i) for i in range(n)]
    batch = EngineBatch(members)
    logs = [log_for(90 + 7 * i, 2, seed=i) for i in range(n)]
    res = batch.replay_keyframes([(i, logs[i], 10, kk) for i in range(n)])
    targets = [33, 47, 60, 71, 89]
    calls, rest = [], []
    for i, (status, _, kfs) in enumerate(res):
        assert status == capi.BGR_OK
        f, blob = [kf for kf in kfs if kf[0] <= targets[i]][-1]
        calls.append((i, blob))
        rest.append((i, logs[i][f:], 10))
    batch.restore(calls)
    got = batch.replay(rest)
    for i in range(n):
        whole = full[i].replay(logs[i], 10)
        f0 = cc.unpack_header(calls[i][1])["frame"]
        assert got[i][0] == capi.BGR_OK
        assert got[i][1] == [c for c in whole if c[0] >= f0], f"world {i}"
        assert live(members[i]) == live(full[i]), f"world {i}"


@pytest.mark.parametrize("call", ["save", "restore"])
def test_launch_count_does_not_grow_with_the_worlds(stream, call):
    counts = []
    for n in (2, 9):
        ms = [box_member(ROWS[i % 6] + 100, 4, stream=stream, seed=i) for i in range(n)]
        batch = EngineBatch(ms)
        for m in ms:
            drive(m, 3, seed=1)
        blobs = batch.checkpoint([(w, 2) for w in range(n)])
        before = ms[0].launch_count()
        if call == "save":
            batch.checkpoint([(w, 1) for w in range(n)])
        else:
            batch.restore(list(enumerate(blobs)))
        counts.append(ms[0].launch_count() - before)
    assert counts[0] == counts[1] == (4 if call == "save" else 3)
