"""-m gpu: batched host edits (bgr_batch_apply_edits, EngineBatch.apply_edits).

Members of one batch differ in rows, growth, optional columns and spawning (the ``spawning`` and ``presence``
registrations of test_gpu_batch_feed.py).  Each has a twin engine on its own stream that gets the same records through
bgr_apply_edits, and an oracle that gets them as single calls.  After every batched call over a random subset in random
order, each listed member's live world (every column, alive bytes, row and active counts) equals its twin's and its
oracle's, the next batched tick's checksums agree, and unlisted members are byte for byte as before.  Also: rows spawned
earlier in the same entry, bands across segment and tile boundaries, empty entries, growth inside the call, refusals
that change nothing, a call queued behind a busy stream with un-collected submits, the staging ring, launch counts at 1,
16 and 256 worlds, and the server loop (batched edits, batched tick, batched feed).  Every test runs on the interpreter
under BGR_TUNE_JIT=0 (a batch that is not specialised) and on both item sizes of the generated kernel (the
generic_kernel fixture); the random interleavings (a Fleet with batched edits as one more action) run on the same three."""
import ctypes as C
import time

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import EDIT_DTYPE, Engine, EngineBatch
from interleave_driver import SEGMENT, TILE, Fleet
from oracle_backend import OracleWorld
from test_gpu_batch_feed import MARGIN, REGISTRATIONS, ROWS, batched_tick, stream  # noqa: F401  (stream: a fixture)
from test_gpu_batch_oracle import fleet_configs, fleet_engines
from test_gpu_host_edits import DESPAWN, INSERT, REMOVE, SLEEP_CYCLES, SPAWN, WRITE, Batch, EditInterleaving

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
GROW = capi.BGR_CFG_GROWABLE
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
DEFER_BITS = capi.BGR_KERNEL_DEFERRED_LIVE | capi.BGR_KERNEL_FROM_DEFERRED
OPTIONAL = {"spawning": [1], "presence": [0, 2]}   # the registrations' optional columns, as indices into their fields


class Member:
    """A batch member (on the batch stream; every third one growable from 64 rows above its population), its twin on
    its own stream and its oracle, with the registration's columns."""

    def __init__(self, reg, i, stream, margin=MARGIN):
        n = ROWS[i % len(ROWS)]
        self.grow = i % 3 == 2
        self.cap0 = n + 64 if self.grow else n + margin
        self.eng = Engine(max_entities=self.cap0, max_depth=9, flags=GROW if self.grow else 0, stream=stream)
        self.twin = Engine(max_entities=n + margin, max_depth=9)
        self.orc = OracleWorld(max_entities=n + margin, max_depth=9)
        for w in (self.eng, self.twin, self.orc):
            self.fields = REGISTRATIONS[reg](w, n, i)
            w.set_depth(8)
        self.cols = sorted({c for c, _, _ in self.fields})
        self.optional = [self.fields[k][0] for k in OPTIONAL[reg]]
        self.limit = n + margin - 400   # rows edits may spawn up to: the ticks spawn too (spawning)

    def close(self):
        for w in (self.eng, self.twin, self.orc):
            w.close()


def fleet(reg, stream, k=6, margin=MARGIN):
    members = [Member(reg, i, stream, margin) for i in range(k)]
    return members, EngineBatch([m.eng for m in members])


def image(x, cols):
    """The live world of an engine: row count, active count, alive bytes and every column of every row."""
    n = x.row_count()
    return (n, x.active_count(), x.read_alive(0, n).tobytes(), tuple(x.read_component(c, 0, n).tobytes() for c in cols),
            tuple(x.has_component(c, 0, n).tobytes() for c in cols))


def live_view(x, cols):
    """What the oracle holds too: row count, active count, alive bytes, the presence of live rows and the columns of
    the live rows that hold them."""
    n = x.row_count()
    alive = x.read_alive(0, n).astype(bool)
    has = [x.has_component(c, 0, n).astype(bool) & alive for c in cols]
    return (n, x.active_count(), alive.tobytes(), tuple(h.tobytes() for h in has),
            tuple(x.read_component(c, 0, n)[h].tobytes() for c, h in zip(cols, has)))


def draw_edits(m, rng, tally):
    """A random batch for member m, drawn against its oracle: bands across 64-row segment and 512-row tile boundaries,
    field writes, overlapping writes, inserts / removes of its optional columns, despawns, and spawns followed by writes
    to the rows just spawned.  Returns the Batch and the single calls the oracle gets (only those on live rows for
    presence changes and despawns: the oracle holds no dead rows)."""
    orc, cols = m.orc, m.cols
    rows = orc.row_count()
    alive = set(int(r) for r in np.flatnonzero(orc.read_alive(0, rows))) if rows else set()
    sizes = {c: orc.elem_bytes[c] for c in cols}
    optional = m.optional
    b, calls = Batch(), []

    def finite(count, ln):   # bytes of finite f32 values: the f32 systems assert finite values at checksum frames
        return rng.uniform(-5, 5, (count, ln // 4)).astype(np.float32).view(np.uint8)

    def write(c, first, count, off, ln):
        vals = finite(count, ln)
        b.add(WRITE, c, first, count, off, ln, vals.tobytes())
        calls.append(("write", (c, first, count, off, vals)))

    for _ in range(int(rng.integers(1, 12))):
        what = str(rng.choice(["band", "band", "field", "overlap", "presence", "despawn", "spawn"]))
        if what == "spawn" and rows + 200 < m.limit:
            edge = (rows // SEGMENT + 1) * SEGMENT if rng.random() < 0.6 else (rows // TILE + 1) * TILE
            k = max(1, min(200, edge - rows + int(rng.integers(0, 40))))
            b.add(SPAWN, count=k)
            calls.append(("spawn", (k,)))
            first, rows = rows, rows + k
            alive.update(range(first, rows))
            for c in cols:
                write(c, first, k, 0, sizes[c])
            tally["spawn_then_write"] += 1
        elif what in ("band", "field", "overlap") and rows:
            c = int(rng.choice(cols))
            off, ln = (0, sizes[c]) if what == "band" or sizes[c] == 4 else (4, sizes[c] - 4)
            if what == "overlap":   # a row written twice in one entry: the later record wins
                first, count = int(rng.integers(0, rows)), 1
                write(c, first, count, off, ln)
            else:
                edge = min(rows - 1, int(rng.choice([SEGMENT, TILE])) * int(rng.integers(1, max(2, rows // SEGMENT))))
                first = max(0, edge - int(rng.integers(1, 80)))
                count = min(rows - first, int(rng.integers(1, 120)))
                tally["boundary_bands"] += first < edge <= first + count - 1
            write(c, first, count, off, ln)
        elif what == "presence" and optional and rows:
            c, r = int(rng.choice(optional)), int(rng.integers(0, rows))
            if rng.random() < 0.5:
                v = finite(1, sizes[c])[0]
                b.add(INSERT, c, r, value=v.tobytes())
                if r in alive:
                    calls.append(("insert_component", (c, r, v)))
            else:
                b.add(REMOVE, c, r)
                if r in alive:
                    calls.append(("remove_component", (c, r)))
            tally["presence"] += 1
        elif what == "despawn" and rows:
            r = int(rng.integers(0, rows))
            b.add(DESPAWN, row=r)
            if r in alive:
                calls.append(("despawn", (r,)))
            alive.discard(r)
    return b, calls


def apply_single(x, calls):
    for name, args in calls:
        if name == "write":
            c, first, count, off, vals = args
            cur = x.read_component(c, first, count).copy()
            cur[:, off:off + vals.shape[1]] = vals
            x.write_component(c, first, cur)
        else:
            getattr(x, name)(*args)


def batched_edits(batch, members, rng, listed, tally, empty=()):
    """One batched call over `listed` (members in `empty` get no edits): every listed member equals its twin (which
    got the same records through bgr_apply_edits) and its oracle; unlisted members are unchanged."""
    others = {i: image(m.eng, m.cols) for i, m in enumerate(members) if i not in listed}
    entries = []
    for i in listed:
        m = members[i]
        if i in empty:
            entries.append((i, np.zeros(0, EDIT_DTYPE), b""))
            continue
        b, calls = draw_edits(m, rng, tally)
        entries.append((i, b.array(), bytes(b.values)))
        m.twin.apply_edits(b.array(), bytes(b.values))
        apply_single(m.orc, calls)
    batch.apply_edits(entries)
    for i in listed:
        m = members[i]
        got = image(m.eng, m.cols)
        assert got == image(m.twin, m.cols), f"world {i}: differs from its twin"
        assert live_view(m.eng, m.cols) == live_view(m.orc, m.cols), f"world {i}: differs from its oracle"
    for i, before in others.items():
        assert image(members[i].eng, members[i].cols) == before, f"world {i}: unlisted, but changed"
    tally["calls"] += 1
    tally["entries"] += len(listed)


def kernels_agree(members, listed):
    """The listed members deferred their live image exactly when their twins did (both were read after the edits)."""
    for i in listed:
        m = members[i]
        assert m.eng.last_kernel().raw & DEFER_BITS == m.twin.last_kernel().raw & DEFER_BITS, f"world {i}: deferral"


# ------------------------------------------------------------------------------------------ batched = twin = oracle
@pytest.mark.usefixtures("generic_kernel")
@pytest.mark.parametrize("reg", sorted(REGISTRATIONS))
def test_batched_edits_equal_single_edits_and_the_oracle(stream, reg):
    members, batch = fleet(reg, stream)
    rng = np.random.default_rng(sum(map(ord, reg)) + 7)
    tally = {k: 0 for k in ("calls", "entries", "spawn_then_write", "boundary_bands", "presence")}
    try:
        for t in range(24):
            batched_tick(batch, members, rng)
            order = [int(x) for x in rng.permutation(len(members))]
            listed = order[:int(rng.integers(1, len(members) + 1))]
            batched_edits(batch, members, rng, listed, tally)
            batched_tick(batch, members, rng)   # the next tick's checksums: the twin's and the oracle's
            kernels_agree(members, listed)
        grown = any(m.eng.capacity()[0] > m.cap0 for m in members if m.grow)
    finally:
        batch.close()
        for m in members:
            m.close()
    print(f"\n[batched edits] {reg}: {tally} grown={grown}")
    assert tally["spawn_then_write"] and tally["boundary_bands"], tally
    if reg == "spawning":
        assert grown, "no growable member grew inside a batched call"


# ------------------------------------------------------------------------------------------ empty entries
@pytest.mark.usefixtures("generic_kernel")
def test_an_empty_entry_leaves_a_deferred_live_image_deferred(stream):
    """An entry with no edits materialises nothing, as bgr_apply_edits with n == 0 returns at once; a listed world with
    edits and a deferred live image gets its own materialisation."""
    members, batch = fleet("presence", stream)
    rng = np.random.default_rng(11)
    tally = {k: 0 for k in ("calls", "entries", "spawn_then_write", "boundary_bands", "presence")}
    try:
        batched_tick(batch, members, rng)
        deferred = [i for i, m in enumerate(members) if m.eng.last_kernel().deferred_live]
        before = [m.eng.launch_count() for m in members]
        batch.apply_edits([(i, np.zeros(0, EDIT_DTYPE), b"") for i in range(len(members))])
        assert [m.eng.launch_count() for m in members] == before, "an empty call launched"
        if deferred:   # world `deferred[0]` is still deferred: with edits, it materialises once, on its own count
            d = deferred[0]
            first = (d + 1) % len(members)
            b0 = [m.eng.launch_count() for m in members]
            batched_edits(batch, members, rng, [first, d], tally, empty=(first,))
            grew = [m.eng.launch_count() - x for m, x in zip(members, b0)]
            assert grew[d] >= 1 and all(g == 0 for i, g in enumerate(grew) if i not in (first, d)), grew
        batched_tick(batch, members, rng)
    finally:
        batch.close()
        for m in members:
            m.close()


# ------------------------------------------------------------------------------------------ growth and refusals
def _raw_call(batch, entries):
    """bgr_batch_apply_edits through ctypes: (status, status_out, last error)."""
    lib = capi.load_library()
    keep = [(np.ascontiguousarray(x, EDIT_DTYPE), np.frombuffer(v, np.uint8)) for _, x, v in entries]
    arr = (capi.bgr_batch_edits * max(1, len(entries)))(*[
        capi.bgr_batch_edits(w, len(x), x.ctypes.data if len(x) else None, v.ctypes.data if v.size else None, v.size)
        for (w, _, _), (x, v) in zip(entries, keep)])
    status = (C.c_int32 * max(1, len(entries)))()
    rc = lib.bgr_batch_apply_edits(batch._h, arr, len(entries), status)
    return rc, list(status)[:len(entries)], lib.bgr_last_error().decode()


@pytest.mark.usefixtures("generic_kernel")
def test_refusals_change_nothing_and_growth(stream):
    """Every refusal class marks its entry, names its world with the single call's text, and changes no image, row
    count, capacity or launch count on any member; a growable member then grows inside a call."""
    members, batch = fleet("spawning", stream, margin=4096)
    rng = np.random.default_rng(5)
    tally = {k: 0 for k in ("calls", "entries", "spawn_then_write", "boundary_bands", "presence")}
    try:
        batched_tick(batch, members, rng)

        def ok(i):
            b = Batch()
            b.add(WRITE, members[0].cols[0], 0, 1, 0, 4, b"\1\2\3\4")   # one registration: one column index
            return (i, b.array(), bytes(b.values))

        def spawn(i, k):
            b = Batch()
            b.add(SPAWN, count=k)
            return (i, b.array(), b"")

        bad = Batch()
        for _ in range(3):
            bad.add(WRITE, members[0].cols[0], 0, 1, 0, 4, b"\0\0\0\0")
        bad.add(DESPAWN, row=members[0].eng.row_count() + 5)
        fixed = 0   # member 0: fixed capacity; member 2: growable
        cases = [
            ([ok(1), ok(6)], 1, capi.BGR_ERR_INVALID_ARGUMENT, "world 6: no such world in a batch of 6"),
            ([ok(1), ok(3), ok(1)], 2, capi.BGR_ERR_INVALID_ARGUMENT, "world 1: listed twice in one call"),
            ([ok(4), ok(1), (0, bad.array(), bytes(bad.values))], 2, capi.BGR_ERR_INVALID_ARGUMENT,
             "world 0: edit 3: row out of range"),
            ([spawn(2, 10_000), spawn(fixed, members[fixed].cap0)], 1, capi.BGR_ERR_CAPACITY,
             "world 0: spawn exceeds max_entities"),
            ([ok(1), spawn(2, 1 << 31)], 1, capi.BGR_ERR_CAPACITY, "world 2: "),
        ]
        for entries, at, status, text in cases:   # (reads launch kernels too: launch counts are taken around the call)
            before = [(image(m.eng, m.cols), m.eng.capacity()[0]) for m in members]
            launches = [m.eng.launch_count() for m in members]
            rc, st, err = _raw_call(batch, entries)
            assert [m.eng.launch_count() for m in members] == launches, f"{text}: a refused call launched"
            assert rc == status and st[at] == status and all(s == 0 for j, s in enumerate(st) if j != at), (text, rc, st)
            assert err.startswith(text), (text, err)
            after = [(image(m.eng, m.cols), m.eng.capacity()[0]) for m in members]
            assert after == before, f"{text}: a refused call changed a member"
            with pytest.raises(BgrError) as ex:
                batch.apply_edits(entries)
            assert ex.value.status == status
        # growth inside the call: member 2 (growable, 64 rows of headroom) spawns past its capacity and writes one of
        # the new rows, next to another member's write
        m2 = members[2]
        cap = m2.eng.capacity()[0]
        k = cap - m2.eng.row_count() + 100
        b = Batch()
        b.add(SPAWN, count=k)
        b.add(WRITE, m2.cols[0], cap + 50, 1, 0, 4, b"\7\7\7\7")
        entries = [ok(1), (2, b.array(), bytes(b.values))]
        for i, x, v in entries:
            members[i].twin.apply_edits(x, v)
        apply_single(members[1].orc, [("write", (members[1].cols[0], 0, 1, 0, np.frombuffer(b"\1\2\3\4", np.uint8).reshape(1, 4)))])
        apply_single(m2.orc, [("spawn", (k,)), ("write", (m2.cols[0], cap + 50, 1, 0, np.full((1, 4), 7, np.uint8)))])
        batch.apply_edits(entries)
        assert m2.eng.capacity()[0] > cap, "the growable member did not grow inside the call"
        for i in (1, 2):
            m = members[i]
            assert image(m.eng, m.cols) == image(m.twin, m.cols), f"world {i}: differs from its twin after growth"
            assert live_view(m.eng, m.cols) == live_view(m.orc, m.cols), f"world {i}: differs from its oracle"
        batched_tick(batch, members, rng)
    finally:
        batch.close()
        for m in members:
            m.close()


# ------------------------------------------------------------------------------------------ queued
@pytest.mark.usefixtures("generic_kernel")
def test_the_call_is_queued_behind_a_busy_stream(stream):
    """The call returns while the shared stream runs a 100 ms kernel, behind a member's un-collected submits, which
    keep their results; five calls in a row go through the staging ring."""
    import torch
    from test_gpu_batch_feed import vector
    members, batch = fleet("presence", stream)
    rng = np.random.default_rng(17)
    tally = {k: 0 for k in ("calls", "entries", "spawn_then_write", "boundary_bands", "presence")}
    s = torch.cuda.ExternalStream(stream)
    try:
        batched_tick(batch, members, rng)
        for rep in range(5):
            q = rep % len(members)
            m = members[q]
            reqs = vector(m, rng)
            expect = m.orc.handle_requests(NOSESS, reqs)
            m.eng.submit_requests(NOSESS, reqs)
            assert m.twin.handle_requests(NOSESS, reqs) == expect
            listed = [int(x) for x in rng.permutation(len(members))]
            entries = []
            for i in listed:
                b, calls = draw_edits(members[i], rng, tally)
                entries.append((i, b.array(), bytes(b.values)))
                members[i].twin.apply_edits(b.array(), bytes(b.values))
                apply_single(members[i].orc, calls)
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP_CYCLES)
            t0 = time.perf_counter()
            batch.apply_edits(entries)
            dt = time.perf_counter() - t0
            busy = not s.query()
            assert dt < 0.03, f"the batched call took {dt * 1e3:.1f} ms behind a 100 ms kernel"
            assert busy, "the shared stream finished before the call returned: the call waited"
            assert m.eng.collect() == expect
            for i in listed:
                assert image(members[i].eng, members[i].cols) == image(members[i].twin, members[i].cols), (rep, i)
        batched_tick(batch, members, rng)
    finally:
        batch.close()
        for m in members:
            m.close()


# ------------------------------------------------------------------------------------------ launches
@pytest.mark.usefixtures("generic_kernel")
@pytest.mark.parametrize("k", [1, 16, 256])
def test_launches_do_not_grow_with_the_number_of_worlds(stream, k):
    """After a call that materialised every deferred live image, a call whose entries spawn and write is two launches
    on the first listed world's engine and none on the others'."""
    engines = []
    try:
        for i in range(k):
            e = Engine(max_entities=1024, max_depth=4, stream=stream)
            REGISTRATIONS["presence"](e, 64 + i % 5, i)
            engines.append(e)
        batch = EngineBatch(engines)
        rng = np.random.default_rng(k)
        order = [int(x) for x in rng.permutation(k)]

        def entries():
            out = []
            for i in order:
                b = Batch()
                b.add(SPAWN, count=3)
                b.add(WRITE, 0, int(rng.integers(0, 60)), 2, 0, 4, rng.integers(0, 256, 8, dtype=np.uint8).tobytes())
                out.append((i, b.array(), bytes(b.values)))
            return out

        batch.handle_requests([(i, NOSESS, []) for i in range(k)])
        batch.apply_edits(entries())   # materialises what is deferred
        before = [e.launch_count() for e in engines]
        batch.apply_edits(entries())
        grew = [e.launch_count() - b for e, b in zip(engines, before)]
        assert grew == [2 if i == order[0] else 0 for i in range(k)], grew
        assert all(e.row_count() == 64 + i % 5 + 6 for i, e in enumerate(engines))
        batch.close()
    finally:
        for e in engines:
            e.close()


# ------------------------------------------------------------------------------------------ server loop
@pytest.mark.usefixtures("generic_kernel")
def test_server_loop_batched_edits_tick_and_feed(stream):
    """Batched edits, then a batched tick, then a batched feed report: every entry's records equal its twin's single
    report after the same edits and tick, so the edited rows show up."""
    members, batch = fleet("presence", stream)
    rng = np.random.default_rng(23)
    tally = {k: 0 for k in ("calls", "entries", "spawn_then_write", "boundary_bands", "presence")}
    feeds = [(m.eng.feed_create(m.fields), m.twin.feed_create(m.fields)) for m in members]
    try:
        for t in range(6):
            listed = [int(x) for x in rng.permutation(len(members))]
            batched_edits(batch, members, rng, listed, tally)
            batched_tick(batch, members, rng)
            calls = [(i, feeds[i][0], 100_000) for i in listed]
            res = batch.feed_wait(batch.feed_begin(calls, batch.feed_alloc(calls)))
            for (i, _, cap), (recs, info) in zip(calls, res):
                tw, tf = members[i].twin, feeds[i][1]
                trecs, tinfo = tw.feed_wait(tw.feed_begin(tf, tw.feed_alloc(tf, cap), cap))
                assert tuple(info) == tuple(tinfo) and recs.tobytes() == trecs.tobytes(), f"tick {t}: world {i}"
                assert info.n_records > 0 or t > 0
    finally:
        batch.close()
        for m in members:
            m.close()


# ------------------------------------------------------------------------------------------ random interleavings
class EditFleet(Fleet):
    """A Fleet with batched edits as one more action: a random subset of the members, in random order, each draws an
    edit batch with ``EditInterleaving.act_edit_batch`` (its twin and oracle get the records as single calls there),
    and the member's engine gets all of them in one bgr_batch_apply_edits, also while a member has submits in
    flight (that member may be listed)."""

    def one_step(self) -> None:
        if self.rng.random() < 0.2:
            return self.act_batch_edits()
        return super().one_step()

    def act_between(self, exclude: int) -> None:
        if self.rng.random() < 0.4:
            return self.act_batch_edits(queued=exclude)
        return super().act_between(exclude)

    def act_batch_edits(self, queued=None) -> None:
        rng = self.rng
        avail = [i for i, m in enumerate(self.members) if m.cfg.order_base == 0]   # the generator spawns
        if not avail:
            return self.note("(no member with order_base 0)")
        worlds = [avail[int(j)] for j in rng.permutation(len(avail))[:int(rng.integers(1, len(avail) + 1))]]
        entries = []
        for i in worlds:
            m = self.members[i]
            held, eng = [], m.eng

            class Capture:   # stands in for the member's engine while the generator draws: keeps the records
                def __getattr__(_, name):
                    return getattr(eng, name)

                def apply_edits(_, edits, values=b""):
                    held.append((np.array(edits, copy=True), bytes(values)))

            m.eng = Capture()
            try:
                EditInterleaving.act_edit_batch(m)
            finally:
                m.eng = eng
            entries.append((i,) + held[0])
            m.tally["batched_edit_entries"] += 1
        self.note(f"batched apply_edits over {worlds}" + (f" (w{queued} has submits in flight)" if queued is not None else ""))
        self.batch.apply_edits(entries)
        for i in worlds:
            self.members[i].note_growth()
        self.tally["batch_edits"] += 1
        self.tally["batch_edits_queued"] += queued is not None and queued in worlds


FLEETS = {"interpreter": "fallback", "jit": "jit_whole_rows4", "jit_quarter_tiles": "jit_quarter"}


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("kernel", sorted(FLEETS))
def test_random_interleavings_with_batched_edits(monkeypatch, stream, kernel):
    for k in ("BGR_TUNE_JIT", "BGR_TUNE_JIT_ITEM", "BGR_TUNE_JIT_ROWS"):
        monkeypatch.delenv(k, raising=False)
    fcfg = fleet_configs()[FLEETS[kernel]]
    total = {}
    for seed in range(4):
        fl = EditFleet(fcfg, seed, fleet_engines(stream), EngineBatch)
        for m in fl.members:   # the generator's helpers (_field, _write); its edit batches in their host writes too
            if m.cfg.order_base == 0:
                m.__class__ = EditInterleaving
        try:
            t = fl.run()
        finally:
            fl.close()
        for key, v in t.items():
            total[key] = total.get(key, 0) + v
    print(f"\n[batched edit interleavings] {kernel}: " + ", ".join(f"{k}={v}" for k, v in sorted(total.items()) if "edit" in k))
    for key, least in {"batch_edits": 10, "batched_edit_entries": 20}.items():
        assert total.get(key, 0) >= least, (key, total.get(key, 0))
