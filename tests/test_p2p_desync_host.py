"""P2P desync reports without a GPU: the ring's retention of confirmed frames (bgr_ring_set_retention, the same SlotRing
class the engine runs) and bgr_digest_mismatch, the one place the digest format is interpreted."""
import ctypes as C
import random

import numpy as np
import pytest

import test_ring_kats as kats
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import digest_mismatch
from ring_adapters import EngineRing
from test_desync_capture import REFERENCE_KATS


class RetainingRing(EngineRing):
    """bgr_ring_* of a ring that retains confirmed frames; the payload per slot stands for the HBM image."""

    def __init__(self, depth=None, n_slots=64, interval=3, count=4, capture=False):
        self.lib = capi.load_library()
        self.cap = n_slots
        self.h = C.c_void_p((self.lib.bgr_ring_create_capture if capture else self.lib.bgr_ring_create)(n_slots))
        assert self.lib.bgr_ring_set_retention(self.h, interval, count) == 0
        self.payload = {}
        if depth is not None:
            self.set_depth(depth)

    def retained(self):
        buf, n = (C.c_int32 * 64)(), C.c_uint32()
        self.lib.bgr_ring_retained(self.h, buf, 64, C.byref(n))
        return [buf[i] for i in range(n.value)]

    def slots_in_use(self):
        n = C.c_uint32()
        self.lib.bgr_ring_slots_in_use(self.h, C.byref(n))
        return n.value


class PlainRing(EngineRing):
    def __init__(self, n_slots):
        self.lib = capi.load_library()
        self.cap = n_slots
        self.h = C.c_void_p(self.lib.bgr_ring_create(n_slots))
        self.payload = {}


@pytest.mark.parametrize("name", REFERENCE_KATS)
@pytest.mark.parametrize("interval", [1, 2, 5])
def test_reference_ring_kats_hold_on_a_retaining_ring(name, interval):
    getattr(kats, name)(lambda depth: RetainingRing(depth, interval=interval))


class RetentionModel:
    """The retention rules restated on a frame-only queue (oldest first)."""

    def __init__(self, interval, count):
        self.q, self.retained, self.interval, self.count, self.depth = [], [], interval, count, 60

    def _leave_old_end(self):
        f = self.q.pop(0)
        if f >= 0 and f % self.interval == 0:
            self.retained.append(f)
            del self.retained[:-self.count]

    def push(self, f):
        if f in self.retained:
            self.retained.remove(f)
        while self.q and not self.q[-1] < f:
            self.q.pop()                       # new end: not final
        while self.q and len(self.q) + 1 > self.depth:
            self._leave_old_end()
        if self.depth:
            self.q.append(f)

    def confirm(self, c):
        while self.q and self.q[0] < c:
            self._leave_old_end()

    def rollback(self, f):
        while self.q and self.q[-1] != f:
            self.q.pop()

    def reset(self):
        self.retained = []


def _p2p_trace(rng, ticks, max_depth, queued):
    """The ring calls compile_requests makes for a P2P session: per Save sync_depth, confirm, push; a rollback loads a
    queued frame (``queued()``, oldest first) and re-saves the frames after it."""
    frame, confirmed = 0, -1
    for _ in range(ticks):
        depth = rng.randint(1, max_depth)
        q = queued()
        if q and rng.random() < 0.3:
            target = rng.choice(q)
            yield ("rollback", target)
            for f in range(target, frame):
                yield ("save", f, depth, confirmed)
        yield ("save", frame, depth, confirmed)
        frame += 1
        confirmed = max(confirmed, frame - rng.randint(1, depth + 1))


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("interval,count", [(1, 1), (3, 2), (10, 4), (4, 7)])
def test_random_p2p_traces_keep_the_plain_queue_and_retain_by_the_rules(seed, interval, count):
    rng = random.Random(seed * 1000 + interval * 10 + count)
    max_depth = rng.randint(1, 8)
    plain, ring, model = PlainRing(max_depth), RetainingRing(n_slots=max_depth + count, interval=interval, count=count), \
        RetentionModel(interval, count)
    n_push = 0
    for op in _p2p_trace(rng, 120, max_depth, lambda: list(model.q)):
        if op[0] == "rollback":
            for r in (plain, ring):
                r.rollback(op[1])
            model.rollback(op[1])
            assert plain.get() == ring.get()
            continue
        _, f, depth, confirmed = op
        for r in (plain, ring):
            r.set_depth(depth)
            r.confirm(confirmed)
        model.depth = depth
        model.confirm(confirmed)
        plain.push(f, (f, n_push))
        ring.push(f, (f, n_push))
        model.push(f)
        n_push += 1
        for g in range(f - 12, f + 2):
            assert plain.peek(g) == ring.peek(g), (g, op)
        assert ring.retained() == model.retained[::-1], op
        assert ring.slots_in_use() <= max_depth + count
        if rng.random() < 0.02:
            assert capi.load_library().bgr_ring_set_retention(ring.h, interval, count) == 0  # releases every retained frame
            model.reset()
            assert ring.retained() == []


def test_retained_slots_are_not_reused_and_a_repush_releases_the_stale_copy():
    ring = RetainingRing(depth=2, n_slots=4, interval=2, count=2)
    ring.push(0, "a")
    ring.push(1, "b")
    ring.push(2, "c")            # depth 2: frame 0 leaves from the old end and is retained
    assert ring.retained() == [0]
    ring.rollback(1)             # frame 2 dropped from the new end: not retained
    ring.push(2, "c2")
    ring.push(3, "d")            # frame 1 evicted: not a multiple of 2
    ring.push(4, "e")            # frame 2 retained
    assert ring.retained() == [2, 0]
    ring.confirm(4)              # frame 3 confirmed: not a multiple of 2
    ring.push(5, "f")
    ring.push(6, "g")            # frame 4 retained; frame 0 released (count 2)
    assert ring.retained() == [4, 2]
    ring.push(2, "again")        # a new save of frame 2 releases the stale retained copy
    assert ring.retained() == [4]
    assert ring.slots_in_use() <= 4


def test_retention_on_a_capture_ring_keeps_the_capture_queue():
    ring = RetainingRing(depth=3, n_slots=10, interval=1, count=4, capture=True)
    for f in range(12):
        ring.push(f, f)
        ring.confirm(f - 2)
    assert ring.retained() == [8, 7, 6, 5]
    assert [ring.peek(f) for f in range(9, 12)] == [9, 10, 11]


# ---- bgr_digest_mismatch ----
def _digest(frame=30, rows=1200, n_columns=3, layout=0xABCDEF, seed=1, rng_state=(1, 2, 3, 4), elapsed=500):
    h = capi.bgr_frame_digest_header()
    h.layout, h.frame, h.rows, h.n_columns, h.elapsed_ns = layout, frame, rows, n_columns, elapsed
    h.n_blocks = (rows + capi.BGR_DIGEST_BLOCK_ROWS - 1) // capi.BGR_DIGEST_BLOCK_ROWS
    for i, v in enumerate(rng_state):
        h.rng[i] = v
    words = np.random.default_rng(seed).integers(0, 2**63, size=(h.n_blocks, n_columns + 1), dtype=np.uint64)
    return h, words


def test_digest_mismatch_lists_exactly_the_differing_blocks():
    a = _digest(rows=5000)
    assert digest_mismatch(a, a) == ([], 0)
    b = (a[0], a[1].copy())
    b[1][3, 1] ^= 1
    b[1][7, 3] ^= 1 << 40
    assert digest_mismatch(a, b) == ([3, 7], 0)
    assert digest_mismatch(b, a) == ([3, 7], 0)


def test_digest_mismatch_blocks_past_the_shorter_side_and_host_state():
    a = _digest(rows=1200)                       # 3 blocks
    b = _digest(rows=2100, rng_state=(9, 2, 3, 4), elapsed=600)   # 5 blocks
    b[1][:3] = a[1]
    assert digest_mismatch(a, b) == ([3, 4], 3)
    c = _digest(rows=1100)                       # same block count, different rows: the mask words say it
    c[1][:] = a[1]
    c[1][2, 3] ^= 5
    assert digest_mismatch(a, c) == ([2], 0)


@pytest.mark.parametrize("field,value,text", [("layout", 1, "layout"), ("frame", 31, "frames"),
                                              ("n_columns", 2, "column counts")])
def test_digest_mismatch_refuses_incomparable_digests(field, value, text):
    a = _digest()
    h = capi.bgr_frame_digest_header.from_buffer_copy(a[0])
    setattr(h, field, value)
    with pytest.raises(capi.BgrError) as ei:
        digest_mismatch(a, (h, a[1]))
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and text in str(ei.value)


def test_digest_and_blob_headers_have_the_c_layout():
    assert C.sizeof(capi.bgr_frame_digest_header) == 80
    assert capi.bgr_frame_digest_header.root.offset == 72
    assert C.sizeof(capi.bgr_frame_blob_header) == 80
    assert capi.bgr_frame_blob_header.rng.offset == 48


# ---- the oracle's restatement of the digest (tests/oracle_p2p.py), checked against the oracle's own checksums ----
def test_oracle_digest_folds_to_the_oracle_checksum_and_retains_by_the_rules():
    """Without a GPU: the restated digest words of every queued and retained frame fold (bgr_fold_partials) to the
    checksum the oracle returned for that frame, so the restatement the GPU tests compare against is itself right."""
    from bevy_ggrs_b200.session import P2PTraceSession
    from oracle_p2p import RetainOracleWorld
    n = 1100
    w = RetainOracleWorld(max_entities=n + 8, max_depth=8)
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | capi.BGR_STRATEGY_OPTIONAL)
    tag = w.rollback_component("Tag", 12)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        w.checksum_component(c, 0, ln)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.retain_confirmed(4, 3)
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(2)
    w.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    w.write_component(health, 0, rng.integers(5, 60, n, dtype=np.uint32))
    w.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in range(3, n, 41):
        w.remove_component(score, r)
    sess, latest = P2PTraceSession(2, 8, seed=3, p_clean=0.3), {}
    for _ in range(40):
        for h in range(2):
            sess.add_local_input(h, 0)
        reqs = sess.advance_frame()
        for f, c in w.handle_requests(sess.info(), reqs):
            latest[f] = c
    assert len(w.retained_frames()) == 3 and all(f % 4 == 0 for f in w.retained_frames())
    lib = capi.load_library()
    for f in w.snapshot_frames() + w.retained_frames():
        rows, active, words = w.frame_digest(f)
        p = capi.bgr_partial()
        p.frame, p.n_columns, p.active, p.total = f, 3, active, rows
        x = np.bitwise_xor.reduce(words, axis=0)
        p.xor_[0], p.xor_[1], p.xor_[2] = int(x[0]), int(x[1]), int(x[2])
        cs = capi.bgr_checksum()
        assert lib.bgr_fold_partials(C.byref(p), C.byref(cs)) == 0
        assert cs.lo == latest[f], f


@pytest.mark.parametrize("seed,args,order_base", [
    (0, dict(sizes=[1, 2, 3, 5, 7, 8, 12, 40], n_opt=7), 0),
    (1, dict(words=24), (1 << 32) + 5),
    (2, dict(words=50, n_opt=3), 17),
    (3, dict(sizes=[1024, 3], n_opt=1), 0),
])
def test_oracle_digest_folds_on_random_schemas(seed, args, order_base):
    """The restated digest on schema_util's random registrations (sub-word tails, up to seven optional columns, an
    order_base above 2^32): for columns checksummed over their whole element, the words fold to the oracle's checksum."""
    from bevy_ggrs_b200.session import P2PTraceSession
    from oracle_p2p import RetainOracleWorld
    from schema_util import random_schema
    rng = np.random.default_rng(seed)
    spec = random_schema(rng, ranges=("none", "whole"), **args)
    n = int(rng.integers(500, 1100))
    w = RetainOracleWorld(max_entities=n + 8, max_depth=8, order_base=order_base)
    spec.register(w)
    w.retain_confirmed(3, 3)
    w.build()
    w.spawn(n)
    for i, d in enumerate(spec.values(rng, n)):
        w.write_component(i, 0, d)
    for i in (i for i, o in enumerate(spec.optional) if o):
        for r in rng.choice(n, 9, replace=False):
            w.remove_component(i, int(r))
    sess, latest = P2PTraceSession(2, 8, seed=seed, p_clean=0.3), {}
    for t in range(24):
        if t % 6 == 5:
            alive = np.flatnonzero(w.read_alive(0, n))
            w.despawn(int(alive[len(alive) // 2]))
        for h in range(2):
            sess.add_local_input(h, 0)
        for f, c in w.handle_requests(sess.info(), sess.advance_frame()):
            latest[f] = c
    assert len(w.retained_frames()) == 3
    lib = capi.load_library()
    frames = w.snapshot_frames() + w.retained_frames()
    assert any(w.frame_digest(f)[1] < w.frame_digest(f)[0] for f in frames)   # despawned rows are in the frames
    for f in frames:
        rows, active, words = w.frame_digest(f)
        p = capi.bgr_partial()
        p.frame, p.n_columns, p.active, p.total = f, len(spec.cks), active, rows
        x = np.bitwise_xor.reduce(words, axis=0)
        for k, (i, _, _) in enumerate(spec.cks):
            p.xor_[k] = int(x[i])
        cs = capi.bgr_checksum()
        assert lib.bgr_fold_partials(C.byref(p), C.byref(cs)) == 0
        assert cs.lo == latest[f], f


def test_two_world_diff_reports_the_local_only_rows_as_existence_records():
    """A frame with more blocks locally than on the peer: the local blocks at or past the peer's block count are
    diffed without the peer exporting them (it cannot), so every existing row there is an existence record."""
    from bevy_ggrs_b200.desync import NO_INDEX
    from bevy_ggrs_b200.session import SAVE, SESSION_NONE, Request
    from oracle_p2p import RetainOracleWorld, two_world_diff

    def world(rows):
        w = RetainOracleWorld(max_entities=1100, max_depth=4)
        w.rollback_component("A", 6)
        w.rollback_component("B", 4, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)
        w.checksum_component(0, 2, 4)
        w.set_depth(2)
        w.spawn(rows)
        w.write_component(0, 0, np.arange(rows * 6, dtype=np.uint32).astype(np.uint8).reshape(rows, 6))
        w.remove_component(1, 3)
        return w
    big, small = world(1030), world(512)          # 3 blocks against 1
    big.despawn(1029)
    big.remove_component(1, 600)
    for w in (big, small):
        w.handle_requests((SESSION_NONE, 0, 0, 0), [Request(SAVE, 0)])
    for blocks in ([0], []):
        rep = two_world_diff(big, small, 0, blocks, 10_000)
        local_only = [r for r in range(512, 1029)]
        assert rep.existence_differing == rep.rows_differing == len(local_only)
        assert list(rep.records["row"]) == local_only
        assert set(rep.records["column"]) == {NO_INDEX} and set(rep.records["word"]) == {NO_INDEX}
        assert set(rep.records["latest"]) == {0} and set(rep.records["first"]) == {1, 1 | 2}   # row 600: B absent
        assert rep.columns[1].presence == 0
    # the other direction diffs only what the blob carries: the peer's rows past 512 are in blocks 1 and 2
    assert two_world_diff(small, big, 0, [0], 10_000).rows_differing == 0
    rep = two_world_diff(small, big, 0, [1, 2], 10_000)
    assert rep.existence_differing == len(local_only) and set(rep.records["first"]) == {0}
