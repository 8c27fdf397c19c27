"""-m gpu: the change feed (bgr_feed_*) against the numpy model of change_feed_model.py, fed with the oracle's live
world.  Every case runs the engine and the oracle side by side, asks for a report after every tick (or every few) and
applies it to a host replica: the records must be byte for byte the model's (exactly the rows whose state or tracked
bytes differ from the last report, ascending), and the replica must equal the oracle's live world.  The same calls with
and without a feed must give the same checksums and snapshots: the feed only reads the live image."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, SAVE, P2PTraceSession, Request, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from change_feed_model import FeedModel, Replica, host_edits, world_of
from oracle_backend import OracleWorld
from schema_util import random_schema

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
BIG = 1 << 30


def _particles(w, n, mode, spawn_rate=0):
    """The particles bundle: MODE 0 (one column without the finite assertion), 1 (the example's registration, with
    spawn_particles when spawn_rate > 0) or 2 (Velocity and Ttl optional)."""
    if mode == 2:
        t = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
        v = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY | OPT)
        l = w.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY | OPT)
        w.checksum_component(v, 0, 12, FIN)
        w.checksum_component(t, 0, 12, FIN)
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        w.build()
        cols = (t, v, l)
    else:
        ck = None if mode == 1 else (lambda w_, t_, v_: (w_.checksum_component(v_, 0, 12, 0), w_.checksum_component(t_, 0, 12, FIN)))
        cols = register_particles(w, spawn_rate=spawn_rate, spawn_ttl=40, checksums=ck)
        w.build()
    populate(w, cols, *synth_particles(n, 17, 4, 60, z_fraction=0.2))
    if mode == 2:
        for r in range(0, n, 13):
            w.remove_component(cols[1 + (r // 13) % 2], r)
    return cols


def _scores(w, n):
    """A world the bundle does not cover: Score (optional, +1 per frame), Health (optional, despawns at 0), Tag."""
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = w.rollback_component("Tag", 12, capi.BGR_STRATEGY_COPY)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        w.checksum_component(c, 0, ln)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(5)
    w.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    w.write_component(health, 0, rng.integers(3, 40, n, dtype=np.uint32))
    w.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in range(0, n, 17):
        w.remove_component(score, r)
    return (score, health, tag)


# variant -> (environment, engine flags, builder, kernel kind, fields(cols), (optional column, value column, bytes))
P_FIELDS = lambda c: [(c[0], 0, 12), (c[1], 0, 8), (c[2], 0, 8)]     # translation, velocity.xy, ttl
S_FIELDS = lambda c: [(c[0], 0, 4), (c[2], 4, 8), (c[1], 0, 4)]      # score, a part of tag, health
VARIANTS = {
    "bundle_mode0": ({}, 0, lambda w, n: _particles(w, n, 0), "bundle", P_FIELDS, None),
    "bundle_mode1_spawn": ({}, 0, lambda w, n: _particles(w, n, 1, spawn_rate=7), "bundle", P_FIELDS, None),
    "bundle_mode2": ({}, 0, lambda w, n: _particles(w, n, 2), "bundle", P_FIELDS, (1, 0, 40)),
    "bundle_eager": ({"BGR_TUNE_DEFER_LIVE": "0"}, 0, lambda w, n: _particles(w, n, 2), "bundle", P_FIELDS, (1, 0, 40)),
    "interpreter": ({"BGR_TUNE_JIT": "0"}, 0, _scores, "generic_interpreter", S_FIELDS, (0, 2, 12)),
    "nvrtc_tile": ({"BGR_TUNE_JIT": "2", "BGR_TUNE_JIT_ITEM": "512"}, 0, _scores, "generic_nvrtc", S_FIELDS, (0, 2, 12)),
    "nvrtc_quarter": ({"BGR_TUNE_JIT": "2", "BGR_TUNE_JIT_ITEM": "128"}, 0, _scores, "generic_nvrtc", S_FIELDS, (0, 2, 12)),
    "nvrtc_eager": ({"BGR_TUNE_JIT": "2", "BGR_TUNE_DEFER_LIVE": "0"}, 0, _scores, "generic_nvrtc", S_FIELDS, (0, 2, 12)),
    "stepwise_tma": ({}, capi.BGR_CFG_FORCE_STEPWISE, _scores, "stepwise_tma", S_FIELDS, (0, 2, 12)),
    "stepwise_flat": ({"BGR_TUNE_TMA": "0"}, capi.BGR_CFG_FORCE_STEPWISE, _scores, "stepwise_flat", S_FIELDS, (0, 2, 12)),
    "capture": ({}, capi.BGR_CFG_DESYNC_CAPTURE, lambda w, n: _particles(w, n, 2), "bundle", P_FIELDS, (1, 0, 40)),
    "retention": ({}, -1, _scores, None, S_FIELDS, (0, 2, 12)),
}


def _make(monkeypatch, variant, n, depth=8, extra=4096):
    env, flags, build, _, fields, _ = VARIANTS[variant]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = Engine(max_entities=n + extra, max_depth=depth, flags=max(flags, 0))
    if flags == -1:
        eng.retain_confirmed(4, 3)
    cols = build(eng, n)
    orc = OracleWorld()
    build(orc, n)
    return eng, orc, cols, fields(cols)


class Mirror:
    """One feed of `eng` with its model (fed from the oracle's world) and replica."""

    def __init__(self, eng, fields, cap=BIG):
        self.eng, self.fields = eng, fields
        self.feed = eng.feed_create(fields)
        self.cap = eng.max_entities if cap == BIG else cap
        self.buf = eng.feed_alloc(self.feed, self.cap)
        self.model = FeedModel(fields, eng.max_entities)
        self.replica = Replica(len(fields), [ln for _, _, ln in fields], eng.max_entities)
        self.stream = []

    def begin(self):
        return self.eng.feed_begin(self.feed, self.buf, self.cap)

    def finish(self, ticket, world):
        recs, info = self.eng.feed_wait(ticket)
        want, winfo = self.model.report(world, self.cap)
        assert info == winfo
        assert recs.tobytes() == want.tobytes()
        self.replica.apply(recs)
        if info.pending == 0:  # a capped report leaves rows for the next one
            assert self.replica.matches(self.model, world)
        self.stream.append(recs.tobytes())
        return recs, info

    def report(self, orc_world):
        return self.finish(self.begin(), orc_world)


def _session(kind, seed):
    return SyncTestSession(2, 3, 8, input_delay=2) if kind == "synctest" else P2PTraceSession(2, 8, 2, seed=seed, p_clean=0.4)


def _run(eng, orc, cols, fields, edit, session, ticks, spawn_input=False, reference=None):
    """Ticks of `session` on engine and oracle with a report after each; host edits every third tick.  `reference`,
    an engine built the same way without a feed, must produce the same checksums."""
    m = Mirror(eng, fields)
    sess = _session(session, 11)
    rng = np.random.default_rng(3)
    for t in range(ticks):
        for h in range(2):
            sess.add_local_input(h, capi.BGR_INPUT_SPAWN if (spawn_input and (t + h) % 4 == 0) else (t * 7 + h) & 0xF)
        reqs = sess.advance_frame()
        out = eng.handle_requests(sess.info(), reqs)
        assert out == orc.handle_requests(sess.info(), reqs)
        if reference is not None:
            assert out == reference.handle_requests(sess.info(), reqs)
        for f, c in out:  # host edits between ticks are not re-simulated: a SyncTest compares nothing here
            sess.save_cell(f, c if session == "p2p" else 0)
        if edit and t % 3 == 1:
            host_edits([w for w in (eng, orc, reference) if w is not None], rng, *edit[:2], edit[2])
        m.report(world_of(orc, [c for c, _, _ in fields]))
    return m


@pytest.mark.parametrize("session", ["synctest", "p2p"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_replica_equals_the_oracle_after_every_tick(monkeypatch, variant, session):
    n = 1500
    eng, orc, cols, fields = _make(monkeypatch, variant, n)
    ref = Engine(max_entities=eng.max_entities, max_depth=8, flags=max(VARIANTS[variant][1], 0))
    if VARIANTS[variant][1] == -1:
        ref.retain_confirmed(4, 3)
    VARIANTS[variant][2](ref, n)
    edit = VARIANTS[variant][5]
    edit = (cols[edit[0]], cols[edit[1]], edit[2]) if edit else None
    m = _run(eng, orc, cols, fields, edit, session, 24, spawn_input=variant == "bundle_mode1_spawn", reference=ref)
    kind = VARIANTS[variant][3]
    if kind:
        assert eng.last_kernel().kind == kind
    for c in cols:  # the feed changed no image: snapshots equal the engine's without a feed
        for f in eng.snapshot_frames():
            a, b = eng.peek(f, c, 0, eng.row_count()), ref.peek(f, c, 0, ref.row_count())
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert sum(len(s) for s in m.stream) > 0


def test_multi_wave_bundle_with_spawns_despawns_and_rollbacks(monkeypatch):
    """250k rows: the stamped multi-wave bundle grid; P2P rollbacks resurrect ttl-despawned rows and un-spawn
    spawned ones."""
    n = 250_000
    eng, orc = Engine(max_entities=n + 20_000, max_depth=8), OracleWorld()
    for w in (eng, orc):
        cols = register_particles(w, spawn_rate=64, spawn_ttl=30)
        w.build()
        populate(w, cols, *synth_particles(n, 5, 2, 12))
    fields = [(cols[0], 0, 12), (cols[2], 0, 8)]
    m = _run(eng, orc, cols, fields, None, "p2p", 16, spawn_input=True)
    assert eng.last_kernel().kind == "bundle" and eng.row_count() > n
    states = [np.frombuffer(s, m.model.dtype)["state"] for s in m.stream[1:]]
    assert any((s == 0).any() for s in states) and any((s == 7).any() for s in states)


@pytest.mark.parametrize("seed", range(4))
def test_random_schemas(monkeypatch, seed):
    rng = np.random.default_rng(100 + seed)
    sch = random_schema(rng, words=int(rng.integers(2, 24)))
    n = int(rng.integers(1, 1400))
    eng, orc = Engine(max_entities=n + 64, max_depth=8), OracleWorld()
    for w in (eng, orc):
        cols = sch.register(w)
        w.build()
        w.spawn(n)
    for c, v in zip(cols, sch.values(rng, n)):
        eng.write_component(c, 0, v)
        orc.write_component(c, 0, v)
    fields = []
    for c, s in enumerate(sch.sizes):
        if s >= 4 and len(fields) < 8:
            ln = 4 * int(rng.integers(1, s // 4 + 1))
            fields.append((cols[c], 4 * int(rng.integers(0, s // 4 - ln // 4 + 1)), ln))
    opt = [c for c, o in zip(cols, sch.optional) if o]
    for r in range(0, n, 7):
        for c in opt[:2]:
            eng.remove_component(c, r)
            orc.remove_component(c, r)
    _run(eng, orc, cols, fields, None, "p2p", 12)


@pytest.mark.parametrize("words", [24, 25, 49, 50, 256])
@pytest.mark.parametrize("n", [511, 512, 513, 1023, 1025])
def test_wide_rows_and_populations_around_tiles(words, n):
    eng, orc = Engine(max_entities=n + 8, max_depth=4), OracleWorld()
    for w in (eng, orc):
        big = w.rollback_component("Big", 4 * (words - 1), capi.BGR_STRATEGY_COPY)
        cnt = w.rollback_component("Cnt", 4, capi.BGR_STRATEGY_COPY | OPT)
        w.add_system(capi.BGR_SYS_U32_ADD, [cnt], [0, 1])
        w.build()
        w.spawn(n)
    rng = np.random.default_rng(n + words)
    v = rng.integers(0, 256, (n, 4 * (words - 1)), dtype=np.uint8)
    for w in (eng, orc):
        w.write_component(big, 0, v)
        for r in range(0, n, 5):
            w.remove_component(cnt, r)
    fields = [(big, 4 * (words - 2), 4), (cnt, 0, 4), (big, 0, min(64, 4 * (words - 1)))]
    m = _run(eng, orc, (big, cnt), fields, None, "synctest", 5)
    assert len(np.frombuffer(m.stream[0], m.model.dtype)) == n


@pytest.mark.parametrize("cap", [0, 1, 17, 31, 32, 33, 511, 512, 513, 1000, 1500, 1501, 5000])
def test_cap_edges_concatenate_to_one_uncapped_report(cap):
    n = 1500
    eng, orc = Engine(max_entities=n, max_depth=4), OracleWorld()
    for w in (eng, orc):
        cols = register_particles(w)
        w.build()
        populate(w, cols, *synth_particles(n, 3, 2, 9))
    fields = [(cols[0], 0, 12)]
    whole = Mirror(eng, fields)  # the uncapped feed
    capped = Mirror(eng, fields, cap=max(cap, 1))
    capped.cap = cap
    for f in range(3):
        for w in (eng, orc):
            w.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, f, [0])])
        world = world_of(orc, [cols[0]])
        full, _ = whole.report(world)
        parts, rounds = [], 0
        while True:
            recs, info = capped.report(world)
            parts.append(recs)
            rounds += 1
            assert info.n_records == min(cap, info.n_records + info.pending)
            if info.pending == 0 or cap == 0:
                break
        if cap == 0:
            assert info.pending == len(full) or f > 0
            continue
        assert np.concatenate(parts).tobytes() == full.tobytes()
        assert rounds == max(1, -(-len(full) // cap))


def test_reports_between_queued_submits_see_the_world_the_submits_before_them_left():
    n = 3000
    eng, orc = Engine(max_entities=n, max_depth=8), OracleWorld()
    for w in (eng, orc):
        cols = register_particles(w)
        w.build()
        populate(w, cols, *synth_particles(n, 9, 3, 40))
    fields = [(cols[0], 0, 12), (cols[1], 0, 12), (cols[2], 0, 8)]
    m = Mirror(eng, fields)
    tick = lambda f: [Request(SAVE, f), Request(ADVANCE, f, [0, 0])]
    tickets, worlds = [], []
    for f in range(4):
        eng.submit_requests(NOSESS, tick(f))
        orc.handle_requests(NOSESS, tick(f))
        worlds.append(world_of(orc, [c for c, _, _ in fields]))
        if f % 2 == 1:  # one report per feed in flight: wait for the previous one first
            tickets.append(m.begin())
            with pytest.raises(BgrError) as ei:
                m.begin()
            assert ei.value.status == capi.BGR_ERR_STATE
            m.finish(tickets[-1], worlds[-1])
    second = Mirror(eng, fields[:1])
    t2 = second.begin()
    for f in range(4, 8):  # later ticks run while the copy is in flight and must not leak into it
        eng.submit_requests(NOSESS, tick(f))
        orc.handle_requests(NOSESS, tick(f))
    second.finish(t2, worlds[-1])
    for _ in range(8):
        eng.collect()
    m.report(world_of(orc, [c for c, _, _ in fields]))


def test_feeds_are_independent_reset_and_late_feeds_list_every_row_and_refusals():
    n = 1200
    eng, orc = Engine(max_entities=n + 100, max_depth=8), OracleWorld()
    with pytest.raises(BgrError) as ei:
        eng.feed_create([(0, 0, 4)])
    assert ei.value.status == capi.BGR_ERR_STATE
    for w in (eng, orc):
        cols = _scores(w, n)
    world = lambda: world_of(orc, list(cols))
    a = Mirror(eng, [(cols[0], 0, 4), (cols[2], 0, 12)])
    b = Mirror(eng, [(cols[2], 4, 4), (cols[1], 0, 4)])
    e0 = Mirror(eng, [])  # existence only
    for f in range(6):
        for w in (eng, orc):
            w.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, f, [0])])
        for m in (a, b, e0) if f % 2 else (a, e0):
            m.report(world())
    late = Mirror(eng, [(cols[1], 0, 4)])
    recs, info = late.report(world())
    alive = orc.read_alive(0, orc.row_count()).astype(bool)
    assert np.array_equal(recs["row"], np.nonzero(alive)[0])  # every existing row
    eng.feed_reset(a.feed)
    a.model.reset()
    recs, _ = a.report(world())
    assert np.array_equal(recs["row"], np.nonzero(alive)[0])
    # refusals
    for fields, status in (([(cols[2], 2, 4)], capi.BGR_ERR_INVALID_ARGUMENT), ([(cols[2], 8, 8)], capi.BGR_ERR_INVALID_ARGUMENT),
                           ([(cols[2], 0, 0)], capi.BGR_ERR_INVALID_ARGUMENT), ([(99, 0, 4)], capi.BGR_ERR_INVALID_ARGUMENT),
                           ([(cols[2], 0, 4)] * 9, capi.BGR_ERR_CAPACITY)):
        with pytest.raises(BgrError) as ei:
            eng.feed_create(fields)
        assert ei.value.status == status, fields
    for _ in range(4):
        eng.feed_create([(cols[2], 0, 4)])
    with pytest.raises(BgrError) as ei:
        eng.feed_create([(cols[2], 0, 4)])
    assert ei.value.status == capi.BGR_ERR_CAPACITY
    t = a.begin()
    a.finish(t, world())
    for bad in (t, t + 1, 12345):
        with pytest.raises(BgrError) as ei:
            eng.feed_wait(bad)
        assert ei.value.status == capi.BGR_ERR_STATE
    eng.close()


def test_begin_before_build_and_pageable_host_memory_are_refused():
    import ctypes as C
    eng = Engine(max_entities=64)
    c = eng.rollback_component("A", 4)
    t = C.c_uint32()
    assert eng._lib.bgr_feed_begin(eng._h, 0, None, 0, C.byref(t)) == capi.BGR_ERR_STATE
    eng.build()
    f = eng.feed_create([(c, 0, 4)])
    buf = np.zeros(64 * 12, np.uint8)
    assert eng._lib.bgr_feed_begin(eng._h, f, buf.ctypes.data, 64, C.byref(t)) == capi.BGR_ERR_INVALID_ARGUMENT
    eng.close()


def _minimal_world(n):
    eng, orc = Engine(max_entities=n, max_depth=9), OracleWorld()
    for w in (eng, orc):
        pos = w.rollback_component("Pos", 12, capi.BGR_STRATEGY_COPY)
        cnt = w.rollback_component("Cnt", 4, capi.BGR_STRATEGY_COPY)
        w.checksum_component(pos, 0, 12)
        w.add_system(capi.BGR_SYS_U32_ADD, [cnt], [0, 1])
        w.build()
        w.spawn(n)
    v = np.random.default_rng(1).integers(0, 256, (n, 12), dtype=np.uint8)
    eng.write_component(pos, 0, v)
    orc.write_component(pos, 0, v)
    return eng, orc, pos, cnt


def test_untouched_field_reports_nothing_after_the_first_report_at_1m_rows():
    n = 1 << 20
    eng, _, pos, cnt = _minimal_world(n)
    feed = eng.feed_create([(pos, 0, 12)])
    buf = eng.feed_alloc(feed, n)
    recs, info = eng.feed_wait(eng.feed_begin(feed, buf, n))
    assert info.n_records == n and info.rows == n and info.record_bytes == 20
    assert np.array_equal(recs["row"], np.arange(n)) and (recs["state"] == 3).all()
    assert recs["f0"].tobytes() == eng.read_component(pos, 0, n).tobytes()
    buf[:] = 0xAB
    for f in range(5):
        eng.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, f, [0])])
        recs, info = eng.feed_wait(eng.feed_begin(feed, buf, n))
        assert info.n_records == 0 and info.pending == 0
    assert (buf == 0xAB).all()  # no record byte crossed PCIe
    # the written field: every row, every tick
    f2 = eng.feed_create([(cnt, 0, 4)])
    b2 = eng.feed_alloc(f2, n)
    eng.feed_wait(eng.feed_begin(f2, b2, n))
    eng.handle_requests(NOSESS, [Request(SAVE, 5), Request(ADVANCE, 5, [0])])
    recs, info = eng.feed_wait(eng.feed_begin(f2, b2, n))
    assert info.n_records == n and (recs["f0"].view(np.uint32)[:, 0] == 6).all()
    eng.close()


def test_two_engines_give_byte_identical_record_streams():
    streams = []
    for _ in range(2):
        eng, orc = Engine(max_entities=40_000, max_depth=8), OracleWorld()
        for w in (eng, orc):
            cols = register_particles(w, spawn_rate=32, spawn_ttl=20)
            w.build()
            populate(w, cols, *synth_particles(30_000, 8, 2, 15))
        m = _run(eng, orc, cols, [(cols[0], 0, 12), (cols[2], 0, 8)], None, "p2p", 10, spawn_input=True)
        streams.append(b"".join(m.stream))
        eng.close()
    assert streams[0] == streams[1] and len(streams[0]) > 0
