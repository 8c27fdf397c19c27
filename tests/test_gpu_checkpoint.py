"""World checkpoints on the H100: the GPU encoder's blob equals the numpy encoder (checkpoint_codec.py) applied to the
frame's exported tiles, byte for byte; an engine restored from it continues the source match bit for bit on every kernel
and capacity; a change feed and a pending deferred live image survive a restore; every malformed blob and every refused
call leaves the engine unchanged."""
import contextlib
import os

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, SESSION_P2P, P2PTraceSession, Request
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
import checkpoint_codec as cc
from change_feed_model import FeedModel, world_of
from test_checkpoint_codec import malformed_cases

pytestmark = pytest.mark.gpu
OPT = capi.BGR_STRATEGY_OPTIONAL
BLOB_HEADER = 80   # bgr_frame_blob_header
P2P_INFO = (SESSION_P2P, 8, 0, -1)


@contextlib.contextmanager
def _env(values):
    old = {k: os.environ.get(k) for k in values}
    os.environ.update(values)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def particles_engine(n, spawn=True, flags=0, cap=None, retain=(4, 3), env=None):
    with _env(env or {}):
        eng = Engine(max_entities=cap or n + 4096, max_depth=9, flags=flags)
    cols = register_particles(eng, spawn_rate=5 if spawn else 0, rng_seed=77)
    if retain:
        eng.retain_confirmed(*retain)
    eng.build()
    return eng, cols


def presence_engine(n, flags=0, env=None):
    with _env(env or {}):
        eng = Engine(max_entities=n + 64, max_depth=9, flags=flags)
    score = eng.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = eng.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = eng.rollback_component("Tag", 12)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        eng.checksum_component(c, 0, ln)
    eng.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    eng.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    eng.retain_confirmed(4, 3)
    eng.build()
    eng.spawn(n)
    rng = np.random.default_rng(5)
    eng.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    eng.write_component(health, 0, rng.integers(3, 60, n, dtype=np.uint32))
    eng.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in range(3, n, 37):
        eng.remove_component(score, r)
    for r in range(5, n, 53):
        eng.remove_component(health, r)
    return eng


def drive(eng, ticks, seed=1, spawn_every=0):
    """A P2P trace with rollbacks; the spawn input every ``spawn_every`` ticks (0: never)."""
    sess = P2PTraceSession(2, 8, seed=seed, p_clean=0.3)
    out = []
    for t in range(ticks):
        for h in range(sess.num_players()):
            sess.add_local_input(h, capi.BGR_INPUT_SPAWN if spawn_every and t % spawn_every == h else 0)
        res = eng.handle_requests(sess.info(), sess.advance_frame())
        for f, c in res:
            sess.save_cell(f, c)
        out.append(res)
    return out


def reference_blob(eng, frame, absent):
    """The numpy encoder applied to every exported block of ``frame``, canonicalised."""
    h, _ = eng.frame_digest(frame)
    exp = eng.export_blocks(frame, range(h.n_blocks))
    words = len(absent)
    tb = cc.BLOCK * (4 * words + 1)
    img = np.frombuffer(exp, np.uint8)[BLOB_HEADER:].reshape(-1, 8 + tb)[:, 8:] if h.n_blocks else np.zeros((0, tb), np.uint8)
    planes, mask = cc.tiles_from_image(np.ascontiguousarray(img), words)
    planes, mask = cc.canonical(planes, mask, h.rows, absent)
    return cc.encode(planes, mask, layout=h.layout, frame=frame, rows=h.rows, n_columns=h.n_columns, fps=60,
                     active=h.active, elapsed_ns=h.elapsed_ns, rng=tuple(h.rng), digest_root=h.root)


PARTICLE_ABSENT = cc.plane_absent([40, 12, 8], [False] * 3)
PRESENCE_ABSENT = cc.plane_absent([4, 4, 12], [True, True, False])


def _check_identity(eng, absent, frames):
    for f in frames:
        blob = eng.checkpoint(f)
        assert blob == reference_blob(eng, f, absent), f"frame {f}"
        assert eng.checkpoint(f) == blob   # twice in a row
        h = cc.unpack_header(blob)
        assert h["frame"] == f and h["payload_bytes"] == len(blob) - 104 - 8 * (h["n_blocks"] + 1)


@pytest.mark.parametrize("world", ["stress_1400", "presence", "spawning"])
def test_blob_equals_the_numpy_encoder(world):
    if world == "presence":
        eng, absent = presence_engine(1400), PRESENCE_ABSENT
        drive(eng, 40)
    else:
        eng, cols = particles_engine(1400, spawn=world == "spawning")
        populate(eng, cols, *synth_particles(1400, 3, 5, 60, z_fraction=0.2))
        absent = PARTICLE_ABSENT
        drive(eng, 60, spawn_every=3 if world == "spawning" else 0)
    queued, retained = eng.snapshot_frames(), eng.retained_frames()
    assert queued and retained
    if world != "stress_1400":
        assert eng.active_count() < eng.row_count()   # despawned rows are zeroed in the blob
    _check_identity(eng, absent, [queued[0], queued[-1], retained[0]])
    assert eng.checkpoint(10**6) is None


def test_blob_equals_the_numpy_encoder_at_1m_rows():
    n = 1 << 20
    eng, cols = particles_engine(n, spawn=False, retain=None)
    populate(eng, cols, *synth_particles(n, 3, 400, 800))
    drive(eng, 6)
    f = eng.snapshot_frames()[0]
    _check_identity(eng, PARTICLE_ABSENT, [f])
    # ten of fifteen word planes and the mask plane CONST in every tile, translation x/y, velocity x/y, ttl.lo RAW
    assert len(eng.checkpoint(f)) == 104 + 8 * 2049 + 2048 * 10300


# ---- continuation ----
def script(f, n_vectors, seed):
    """Request vectors from frame f on: ticks [ADVANCE, SAVE] and rollbacks to frames >= f, spawn inputs included."""
    rng = np.random.default_rng(seed)
    cur, out = f, [[Request(LOAD, f)] + tick(rng)]
    cur += 1
    for _ in range(n_vectors - 1):
        if rng.random() < 0.35 and cur > f:
            g = int(rng.integers(max(f, cur - 5), cur + 1))
            vec = [Request(LOAD, g)]
            for _ in range(cur - g + 1):
                vec += tick(rng)
            out.append(vec)
        else:
            out.append(tick(rng))
        cur += 1
    return out


def tick(rng):
    ins = [int(capi.BGR_INPUT_SPAWN if rng.random() < 0.3 else 0), int(rng.integers(0, 4))]
    return [Request(ADVANCE, 0, ins, [0, 0]), Request(SAVE, 0)]


def observe(eng, n_cols):
    rows = eng.row_count()
    # the elements rows hold: an absent optional column's stored bytes are not part of the world (the canonical form
    # zeroes them)
    live = [eng.read_component(c, 0, rows)[eng.has_component(c, 0, rows).astype(bool)].tobytes() for c in range(n_cols)]
    digests = {}
    for f in eng.snapshot_frames():
        h, w = eng.frame_digest(f)
        digests[f] = (h.root, h.rows, h.active, h.elapsed_ns, tuple(h.rng), w.tobytes())
    return rows, eng.active_count(), eng.rollback_frame_count(), live, eng.snapshot_frames(), digests


def run_script(eng, vecs):
    return [eng.handle_requests(P2P_INFO, v) for v in vecs]


CONTINUATIONS = {
    "same": dict(),
    "bigger": dict(cap=20000),
    "growable_small": dict(cap=512, flags=capi.BGR_CFG_GROWABLE),
    "capture": dict(flags=capi.BGR_CFG_DESYNC_CAPTURE),
    # the generic program has no spawn_particles: these two run the presence world
    "interpreter": dict(env={"BGR_TUNE_JIT": "0"}),
    "nvrtc": dict(env={"BGR_TUNE_JIT": "2"}),
    "stepwise_tma": dict(flags=capi.BGR_CFG_FORCE_STEPWISE, env={"BGR_TUNE_TMA": "1"}),
    "stepwise_flat": dict(flags=capi.BGR_CFG_FORCE_STEPWISE, env={"BGR_TUNE_TMA": "0"}),
}


@pytest.mark.parametrize("name", list(CONTINUATIONS))
def test_restored_engine_continues_the_match(name):
    n = 3000
    kw = CONTINUATIONS[name]
    if name in ("interpreter", "nvrtc"):
        a = presence_engine(1400)
        drive(a, 40, seed=4)
        b = presence_engine(1400, env=kw["env"])
    else:
        a, cols = particles_engine(n)
        populate(a, cols, *synth_particles(n, 9, 5, 80, z_fraction=0.2))
        drive(a, 50, seed=4, spawn_every=4)
        b, _ = particles_engine(n, retain=None, **kw)
    f = a.snapshot_frames()[0]
    blob = a.checkpoint(f)
    b.restore(blob)
    assert b.snapshot_frames() == [f] and b.rollback_frame_count() == f and b.row_count() == cc.unpack_header(blob)["rows"]
    assert b.checkpoint(f) == blob
    if name == "capture":
        assert b.peek_first(f, 0, 0, 4) is not None
    vecs = script(f, 24, seed=len(name))
    ra, rb = run_script(a, vecs), run_script(b, vecs)
    assert ra == rb
    assert observe(a, 3) == observe(b, 3)
    if name == "growable_small":
        assert b.capacity()[0] >= a.row_count()
    if name in ("interpreter", "nvrtc"):
        assert b.last_kernel().kind == ("generic_interpreter" if name == "interpreter" else "generic_nvrtc")


def test_restore_with_a_feed_open_and_a_deferred_live_image():
    n = 2000
    a, cols = particles_engine(n)
    populate(a, cols, *synth_particles(n, 1, 5, 80))
    drive(a, 30, seed=2, spawn_every=5)
    f = a.snapshot_frames()[0]
    blob = a.checkpoint(f)
    b, bcols = particles_engine(n)
    populate(b, bcols, *synth_particles(n, 6, 5, 80))
    fields = [(0, 0, 12), (2, 0, 8)]
    feed = b.feed_create(fields)
    buf = b.feed_alloc(feed, 1 << 14)
    model = FeedModel(fields, b.capacity()[0])
    drive(b, 7, seed=3)
    recs, info = b.feed_wait(b.feed_begin(feed, buf, 1 << 14))
    mrecs, minfo = model.report(world_of(b, [0, 2]), 1 << 14)
    assert info == minfo and recs.tobytes() == mrecs.tobytes()
    drive(b, 3, seed=5)
    assert b.last_kernel().deferred_live   # a deferred live image is pending
    b.restore(blob)
    recs, info = b.feed_wait(b.feed_begin(feed, buf, 1 << 14))
    mrecs, minfo = model.report(world_of(b, [0, 2]), 1 << 14)
    assert info == minfo and recs.tobytes() == mrecs.tobytes()
    assert info.n_records > 0
    vecs = script(f, 20, seed=8)
    assert run_script(a, vecs) == run_script(b, vecs)
    assert observe(a, 3) == observe(b, 3)


# ---- refusals ----
def _refused(b, blob, status):
    with pytest.raises(BgrError) as ei:
        b.restore(blob)
    assert ei.value.status == status, str(ei.value)


def test_refusals_leave_the_engine_unchanged():
    n = 1400
    a, cols = particles_engine(n)
    populate(a, cols, *synth_particles(n, 2, 5, 80, z_fraction=0.2))
    drive(a, 20, seed=6, spawn_every=3)
    f = a.snapshot_frames()[0]
    blob = a.checkpoint(f)

    def fresh():
        e, c = particles_engine(n)
        populate(e, c, *synth_particles(n, 8, 5, 80, z_fraction=0.2))
        drive(e, 9, seed=7)
        return e
    b, twin = fresh(), fresh()
    cases = malformed_cases(blob, 15)
    hdr = cc.unpack_header(blob)
    # a flipped payload bit in a live row: a well-formed blob whose content the header's digest does not describe
    _, planes, mask = cc.decode(blob, 15)
    r = int(np.nonzero(mask[0] & 1)[0][0])
    planes[0, 0, r] ^= 1 << 9
    fields = {k: hdr[k] for k in ("layout", "frame", "rows", "n_columns", "fps", "active", "elapsed_ns", "rng", "digest_root")}
    cases.append(("flipped payload bit", cc.encode(planes, mask, **fields)))
    for field, at, fmt, val in (("layout", 8, "<Q", hdr["layout"] ^ 1), ("fps", 36, "<I", 30), ("words", 24, "<I", 16),
                                ("active", 40, "<Q", hdr["active"] + 1)):
        cases.append((field, cc.pack_header({**hdr, field: val}) + blob[104:]))
    for name, bad in cases:
        _refused(b, bad, capi.BGR_ERR_INVALID_ARGUMENT)
    # a presence bit of a column this registration does not have, on an existing row: the decoder refuses the block
    mask2 = mask.copy()
    mask2[0, r] |= 0x80
    with pytest.raises(BgrError) as ei:
        b.restore(cc.encode(planes, mask2, **fields))
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and "mask byte" in str(ei.value)
    small, sc = particles_engine(256, cap=512, retain=None)
    with pytest.raises(BgrError) as ei:
        small.restore(blob)
    assert ei.value.status == capi.BGR_ERR_CAPACITY
    b.submit_requests(P2P_INFO, [Request(ADVANCE, 0, [0, 0], [0, 0])])
    twin.submit_requests(P2P_INFO, [Request(ADVANCE, 0, [0, 0], [0, 0])])
    _refused(b, blob, capi.BGR_ERR_STATE)
    assert b.collect() == twin.collect()
    vecs = [[Request(ADVANCE, 0, [16, 0], [0, 0]), Request(SAVE, 0)] for _ in range(4)]
    assert run_script(b, vecs) == run_script(twin, vecs)
    assert observe(b, 3) == observe(twin, 3)
    sharded = Engine(max_entities=2048, max_depth=9, flags=capi.BGR_CFG_SHARDED)
    register_particles(sharded)
    sharded.build()
    for call in (lambda: sharded.restore(blob), lambda: sharded.checkpoint(0)):
        with pytest.raises(BgrError) as ei:
            call()
        assert ei.value.status == capi.BGR_ERR_UNSUPPORTED


def test_zero_rows_roundtrip():
    a, _ = particles_engine(0, spawn=False, retain=None)
    a.handle_requests(P2P_INFO, [Request(SAVE, 0)])
    blob = a.checkpoint(0)
    assert len(blob) == 104 + 8
    b, _ = particles_engine(0, spawn=False, retain=None)
    b.restore(blob)
    assert b.row_count() == 0 and b.snapshot_frames() == [0]


# ---- the App: resources travel behind the engine blob ----
def _frame_count_app(sess, mismatches, host_column=False):
    """A SyncTest App with a Score column (+3 per frame), a checksummed FrameCount resource (+1 per frame) and retained
    confirmed frames."""
    import struct
    from bevy_ggrs_b200.plugin import (App, GgrsPlugin, GgrsSchedule, LocalInputs, ReadInputs, ResourceSystem, Session,
                                       Startup, SyncTestMismatch, System)

    def bump(res):
        res["FrameCount"] = bytearray(struct.pack("<I", struct.unpack("<I", res["FrameCount"])[0] + 1))
    app = App(Engine(max_entities=64, max_depth=9))
    app.insert_resource(Session.SyncTest(sess)).add_plugins(GgrsPlugin())
    score = app.rollback_component_with_copy("Score", 4)
    app.checksum_component_with_hash(score)
    app.rollback_resource_with_copy("FrameCount", bytes(4)).checksum_resource_with_hash("FrameCount")
    if host_column:
        app.rollback_component_with_clone("Sprite")
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_U32_ADD, [score], [0, 3]))
    app.add_systems(GgrsSchedule, ResourceSystem(bump))
    app.add_systems(ReadInputs, lambda a: a.insert_resource(LocalInputs({h: 0 for h in a.local_players.handles})))
    app.add_systems(Startup, lambda a: a.world.write_component(score, a.world.spawn(10), np.arange(10, dtype=np.uint32)))
    app.add_observer(SyncTestMismatch, mismatches.append)
    app.retain_confirmed(4, 2)
    return app


def test_app_checkpoint_carries_its_resources_into_a_second_app():
    import copy
    from bevy_ggrs_b200.plugin import Session
    from bevy_ggrs_b200.session import SyncTestSession
    d = 3
    sa, mis = SyncTestSession(1, d, 9), []
    a = _frame_count_app(sa, mis)
    for _ in range(30):
        a.step()
    f = sa.current_frame - d   # the frame the next tick loads: the restored ring holds it alone
    blob = a.checkpoint(f)
    assert blob == a.checkpoint(f)
    assert a.retained_frames()
    with pytest.raises(BgrError) as ei:   # the engine retains the frame, the App no longer has its resources
        a.checkpoint(a.retained_frames()[0])
    assert ei.value.status == capi.BGR_ERR_NO_SNAPSHOT
    b = _frame_count_app(SyncTestSession(1, d, 9), mis)
    b.step()
    before = (b.world.snapshot_frames(), dict(b.resources))
    for bad in (blob[:-1], blob + b"\0", blob[:-8] + b"\x08" + blob[-7:], blob[:-12] + b"\x02" + blob[-11:]):
        with pytest.raises(BgrError) as ei:
            b.restore_checkpoint(bad)
        assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    assert (b.world.snapshot_frames(), dict(b.resources)) == before
    b.restore_checkpoint(blob)
    b.insert_resource(Session.SyncTest(copy.deepcopy(sa)))
    assert b.world.snapshot_frames() == [f] and b.resources["FrameCount"] == (a.resources["FrameCount"][0] - d).to_bytes(4, "little")
    for _ in range(20):
        a.step()
        b.step()
        assert a.last_checksums == b.last_checksums
    assert not mis and a.resources == b.resources
    c = _frame_count_app(SyncTestSession(1, d, 9), [], host_column=True)
    c.step()
    for call in (lambda: c.checkpoint(c.world.snapshot_frames()[0]), lambda: c.restore_checkpoint(blob)):
        with pytest.raises(BgrError) as ei:
            call()
        assert ei.value.status == capi.BGR_ERR_UNSUPPORTED
