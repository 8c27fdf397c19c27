"""-m gpu: host edits (bgr_apply_edits): a batch of row writes, presence changes, spawns and despawns in one queued launch.

  - random interleavings (tests/interleave_driver.py) on every kernel configuration, where the engine receives random
    edit batches through ``apply_edits`` and the twin and the oracle the same records as single calls, in order;
  - refusals: an invalid batch changes nothing and launches nothing;
  - the call is queued: it returns while the engine stream is busy, and un-collected submits keep their results;
  - precision on the bundle with content stamps: an edit of a stable plane costs the stores of the (segment, plane)
    pairs it touched, and a write confined to active planes leaves the passive planes elided."""
import time
from collections import Counter

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import EDIT_DTYPE, Engine
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from interleave_driver import NOSESS, SEGMENT, TILE, UNITS_PER_SEGMENT, Config, Interleaving, replay_filter
from test_gpu_interleavings import CONFIG_NAMES, FLAG_SETS, configs, new_engine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
OPT = capi.BGR_STRATEGY_OPTIONAL
WRITE, INSERT, REMOVE, DESPAWN, SPAWN = (capi.BGR_EDIT_WRITE, capi.BGR_EDIT_INSERT, capi.BGR_EDIT_REMOVE,
                                         capi.BGR_EDIT_DESPAWN, capi.BGR_EDIT_SPAWN)
SLEEP_CYCLES = 200_000_000   # about 100 ms at the H100's 1.98 GHz boost clock
KIND_NAMES = {WRITE: "write", INSERT: "insert", REMOVE: "remove", DESPAWN: "despawn", SPAWN: "spawn"}


class Batch:
    """Edit records and their value bytes, built in order."""

    def __init__(self):
        self.recs, self.values = [], bytearray()

    def add(self, kind, column=0, row=0, count=0, byte_offset=0, byte_len=0, value=b""):
        self.recs.append((kind, column, row, count, byte_offset, byte_len, len(self.values), 0))
        self.values += bytes(value)

    def array(self):
        return np.array(self.recs, dtype=EDIT_DTYPE)


class EditInterleaving(Interleaving):
    """The driver's interleavings, where half the host writes are edit batches."""

    def act_host_write(self) -> None:
        if self.rng.random() < 0.5:
            return self.act_edit_batch()
        return super().act_host_write()

    def _field(self, c):
        """A field of column c: 4-byte aligned, its length a multiple of 4 or ending at the element's end."""
        size = self.world.sizes[c]
        off = 4 * int(self.rng.integers(0, -(-size // 4)))
        ends = [e for e in range(off + 4, size + 1, 4)] + [size]
        return off, int(self.rng.choice(sorted(set(e for e in ends if e > off)))) - off

    def act_edit_batch(self) -> None:
        w, rng = self.world, self.rng
        rows = self.orc.row_count()
        alive = set(int(r) for r in np.flatnonzero(self.orc.read_alive(0, rows))) if rows else set()
        optional = [i for i, o in enumerate(w.optional) if o]
        batch, calls = Batch(), []   # calls: single calls in record order, (kind, args, oracle_too)
        hot = int(rng.integers(0, rows)) if rows else 0   # overlapping records land on this row
        for _ in range(int(rng.integers(1, 25))):
            what = str(rng.choice(["band", "band", "field", "overlap", "presence", "despawn", "spawn"]))
            if what == "spawn" and self.room() - (rows - self.orc.row_count()) > 300:
                edge = (rows // SEGMENT + 1) * SEGMENT if rng.random() < 0.6 else (rows // TILE + 1) * TILE
                k = max(1, min(200, edge - rows + int(rng.integers(0, 40))))
                batch.add(SPAWN, count=k)
                calls.append(("spawn", (k,), True))
                self.tally["edit_records_spawn"] += 1
                first, rows = rows, rows + k
                alive.update(range(first, rows))
                for c in range(len(w.sizes)):   # writes to the rows spawned just before
                    self._write(batch, calls, c, first, k, 0, w.sizes[c])
                self.tally["edit_spawn_writes"] += 1
            elif what in ("band", "field", "overlap") and rows:
                if what == "field" and w.bundle:   # Transform.translation only: rotation and scale are passive planes
                    c, off, ln = 0, 0, 12
                    self.tally["edit_translation_writes"] += 1
                else:
                    c = int(rng.integers(0, len(w.sizes)))
                    off, ln = self._field(c) if rng.random() < 0.7 else (0, w.sizes[c])
                if what == "overlap":
                    first, count = hot, 1
                    self.tally["edit_overlaps"] += 1
                else:   # a band across a 64-row segment or a 512-row tile boundary
                    edge = min(rows - 1, int(rng.choice([SEGMENT, TILE])) * int(rng.integers(1, max(2, rows // SEGMENT))))
                    first = max(0, edge - int(rng.integers(1, 80)))
                    count = min(rows - first, int(rng.integers(1, 120)))
                self._write(batch, calls, c, first, count, off, ln)
            elif what == "presence" and optional and rows:
                c = int(rng.choice(optional))
                r = hot if rng.random() < 0.3 else int(rng.integers(0, rows))
                live = r in alive
                if rng.random() < 0.5:
                    v = self.values(c, 1)[0]
                    batch.add(INSERT, c, r, value=v.tobytes())
                    calls.append(("insert_component", (c, r, v), live))
                    self.tally["edit_records_insert"] += 1
                else:
                    batch.add(REMOVE, c, r)
                    calls.append(("remove_component", (c, r), live))
                    self.tally["edit_records_remove"] += 1
                self.tally["edit_presence_on_dead_rows"] += not live
            elif what == "despawn" and rows:
                r = hot if rng.random() < 0.3 else int(rng.integers(0, rows))
                batch.add(DESPAWN, row=r)
                calls.append(("despawn", (r,), r in alive))
                alive.discard(r)
                self.tally["edit_records_despawn"] += 1
        self.note(f"apply_edits: {len(batch.recs)} records "
                  f"{dict(Counter(KIND_NAMES[k[0]] for k in batch.recs))}{' (vectors in flight)' if self.pending else ''}")
        self._touch()
        self.eng.apply_edits(batch.array(), bytes(batch.values))
        for x in (self.twin, self.orc):
            for name, args, oracle_too in calls:
                if x is self.orc and not oracle_too:
                    continue   # the oracle holds no dead rows: presence records and despawns of them change nothing
                if name == "write":
                    c, first, count, off, vals = args
                    cur = x.read_component(c, first, count).copy()
                    cur[:, off:off + vals.shape[1]] = vals
                    x.write_component(c, first, cur)
                else:
                    getattr(x, name)(*args)
        self.max_rows = max(self.max_rows, self.orc.row_count())
        self.tally["edit_batches"] += 1
        self.tally["edit_records_write"] += sum(r[0] == WRITE for r in batch.recs)
        if self.pending:
            self.tally["edit_batches_in_flight"] += 1
        self.note_growth()

    def _write(self, batch, calls, c, first, count, off, ln):
        vals = np.ascontiguousarray(self.values(c, count)[:, off:off + ln])
        batch.add(WRITE, c, first, count, off, ln, vals.tobytes())
        calls.append(("write", (c, first, count, off, vals), True))


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_random_edit_batches_match_the_single_calls(name):
    cfg0 = {c.name: c for c in configs()}[name]
    total = Counter()
    ran = 0
    for seed, (flags, retain) in enumerate(FLAG_SETS[:5]):
        r = replay_filter()
        if r is not None and r != (name, seed):
            continue
        cfg = Config(**{**cfg0.__dict__, "flags": flags, "retain": retain})
        drv = EditInterleaving(cfg, 100 + seed, new_engine(name))
        try:
            t = drv.run()
        finally:
            drv.close()
        ran += 1
        total.update(t)
        if cfg.stamped:
            assert t["stamp_rollovers"] == 1 and t["rollover_verified"] == 1, f"{name} seed {seed}: {t}"
    if not ran:
        pytest.skip("not the configuration BGR_INTERLEAVE_REPLAY selects")
    print(f"\n[edit interleavings] {name}: " + ", ".join(f"{k}={v}" for k, v in sorted(total.items()) if k.startswith("edit")))
    if ran < 5:
        return
    minimums = {"edit_batches": 8, "edit_batches_in_flight": 1, "edit_records_write": 20, "edit_records_despawn": 3,
                "edit_records_spawn": 2, "edit_spawn_writes": 2, "edit_overlaps": 3, "growth_steps": 1}
    if name.startswith("bundle"):
        minimums["edit_translation_writes"] = 3
    if name == "bundle_mode2_stamped":
        minimums.update({"edit_records_insert": 2, "edit_records_remove": 2, "edit_presence_on_dead_rows": 1})
    missing = {k: (total[k], v) for k, v in minimums.items() if total[k] < v}
    assert not missing, f"{name}: tally below its minimum (reached, minimum): {missing}"


# ---------------------------------------------------------------------------------------------------------------------
def _mode2(n, max_entities, flags=0, env=None, monkeypatch=None):
    """The particles world with optional Velocity and Ttl (the bundle's MODE 2)."""
    e = Engine(max_entities=max_entities, max_depth=9, flags=flags)
    t = e.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
    v = e.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY | OPT)
    l = e.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY | OPT)
    e.checksum_component(v, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
    e.checksum_component(t, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
    e.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
    e.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
    e.build()
    populate(e, (t, v, l), *synth_particles(n, 3, 50, 90))
    return e


def _live(e):
    n = e.row_count()
    return [e.read_alive(0, n)] + [e.read_component(c, 0, n) for c in range(3)] + [e.has_component(c, 0, n) for c in (1, 2)]


def _counter_world(monkeypatch, kernel, n):
    """Score (u32, +1 per frame) and an optional Tag (12 B): a registration without the bundle, so without a stamp
    table; `kernel` picks the interpreter or the stepwise path."""
    with monkeypatch.context() as m:
        m.setenv("BGR_TUNE_JIT", "0")
        e = Engine(max_entities=n + 4096, max_depth=9, flags=capi.BGR_CFG_FORCE_STEPWISE if kernel == "stepwise" else 0)
    s = e.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY)
    t = e.rollback_component("Tag", 12, capi.BGR_STRATEGY_CLONE | OPT)
    e.checksum_component(s, 0, 4)
    e.checksum_component(t, 0, 12)
    e.add_system(capi.BGR_SYS_U32_ADD, [s], [0, 1])
    e.build()
    e.spawn(n)
    e.write_component(s, 0, np.arange(n, dtype=np.uint32))
    e.write_component(t, 0, np.arange(3 * n, dtype=np.uint32).reshape(n, 3))
    return e


@pytest.mark.parametrize("kernel", ["interpreter", "stepwise"])
def test_batches_with_an_empty_patch(monkeypatch, kernel):
    """Without a stamp table a spawn-only batch folds into no store, no mask update and no stamp, and neither does a
    write of zero rows: such batches, the first of each staging buffer included, do what bgr_spawn does."""
    n = 1500
    e, twin = _counter_world(monkeypatch, kernel, n), _counter_world(monkeypatch, kernel, n)
    for i in range(6):
        b = Batch()
        if i == 1:
            b.add(WRITE, 0, 7, 0, 0, 4)
        else:
            b.add(SPAWN, count=3 + i)
            twin.spawn(3 + i)
        before = e.launch_count()
        e.apply_edits(b.array(), bytes(b.values))
        # k_apply_edits, and k_spawn_rows when the batch spawns
        assert e.launch_count() - before == (1 if i == 1 else 2)
        assert e.row_count() == twin.row_count()
    rows = e.row_count()
    assert np.array_equal(e.read_alive(0, rows), twin.read_alive(0, rows))
    for c in (0, 1):
        assert np.array_equal(e.read_component(c, 0, rows), twin.read_component(c, 0, rows))
        assert np.array_equal(e.has_component(c, 0, rows), twin.has_component(c, 0, rows))
    f = e.rollback_frame_count()
    reqs = [Request(SAVE, f), Request(ADVANCE, 0, [0])]
    assert e.handle_requests(NOSESS, reqs) == twin.handle_requests(NOSESS, reqs)
    e.close(); twin.close()


def test_invalid_batches_change_nothing():
    n = 3000
    e = _mode2(n, n + 64)
    v = np.zeros(12, np.uint8).tobytes()
    bad = {   # each batch starts with valid records: nothing of them may run either
        "unknown kind": [(WRITE, 1, 5, 1, 0, 4, 0, 0), (9, 0, 0, 0, 0, 0, 0, 0)],
        "unknown column": [(WRITE, 3, 5, 1, 0, 4, 0, 0)],
        "insert into a required column": [(INSERT, 0, 5, 0, 0, 0, 0, 0)],
        "remove of a required column": [(REMOVE, 0, 5, 0, 0, 0, 0, 0)],
        "misaligned field": [(WRITE, 1, 5, 1, 2, 4, 0, 0)],
        "field length neither whole words nor to the end": [(WRITE, 0, 5, 1, 0, 6, 0, 0)],
        "field past the element": [(WRITE, 1, 5, 1, 8, 8, 0, 0)],
        "empty field": [(WRITE, 1, 5, 1, 0, 0, 0, 0)],
        "rows past the row count": [(WRITE, 1, n - 1, 2, 0, 4, 0, 0)],
        "row spawned by a later record": [(WRITE, 1, n, 1, 0, 4, 0, 0), (SPAWN, 0, 0, 1, 0, 0, 0, 0)],
        "values past values_bytes": [(WRITE, 1, 5, 4, 0, 4, 0, 0)],
        "insert value past values_bytes": [(INSERT, 1, 5, 0, 0, 0, 4, 0)],
        "despawn past the row count": [(SPAWN, 0, 0, 2, 0, 0, 0, 0), (DESPAWN, 0, n + 2, 0, 0, 0, 0, 0)],
        "remove past the row count": [(REMOVE, 1, n, 0, 0, 0, 0, 0)],
        "spawn past max_entities": [(DESPAWN, 0, 1, 0, 0, 0, 0, 0), (SPAWN, 0, 0, 65, 0, 0, 0, 0)],
    }
    for what, recs in bad.items():
        live = _live(e)   # the reads launch kernels of their own: counted before the call
        before = (e.launch_count(), e.row_count())
        with pytest.raises(BgrError) as ei:
            e.apply_edits(np.array(recs, EDIT_DTYPE), v)
        expect = capi.BGR_ERR_CAPACITY if what == "spawn past max_entities" else capi.BGR_ERR_INVALID_ARGUMENT
        assert ei.value.status == expect, (what, str(ei.value))
        assert (e.launch_count(), e.row_count()) == before, what
        assert all(np.array_equal(a, b) for a, b in zip(_live(e), live)), what
    # the same records made valid: rows spawned earlier in the batch are addressable; n == 0 launches nothing
    lc = e.launch_count()
    e.apply_edits(np.zeros(0, EDIT_DTYPE))
    assert e.launch_count() == lc
    e.apply_edits(np.array([(SPAWN, 0, 0, 1, 0, 0, 0, 0), (WRITE, 1, n, 1, 0, 12, 0, 0)], EDIT_DTYPE),
                  np.arange(3, dtype=np.float32).tobytes())
    assert e.launch_count() == lc + 2 and e.row_count() == n + 1   # k_spawn_rows + k_apply_edits
    assert np.array_equal(e.read_component(1, n, 1).view(np.float32)[0], np.arange(3, dtype=np.float32))
    e.close()


def test_apply_edits_is_queued_behind_a_busy_stream():
    import torch
    n = 5000
    e, twin = _mode2(n, n + 256), _mode2(n, n + 256)
    stream = torch.cuda.ExternalStream(e.stream())
    f0 = e.rollback_frame_count()

    def tick(f):
        return NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, [0])]

    def batch(rng):
        b = Batch()
        for r in rng.integers(0, n, 20):
            b.add(WRITE, 1, int(r), 1, 0, 4, rng.uniform(-5, 5, 1).astype(np.float32).tobytes())
        b.add(REMOVE, 2, int(rng.integers(0, n)))
        b.add(DESPAWN, 0, int(rng.integers(0, n)))
        b.add(SPAWN, 0, 0, 3)
        return b

    def single(x, b):
        for kind, c, row, count, off, ln, vo, _ in b.recs:
            if kind == WRITE:
                cur = x.read_component(c, row, 1).copy()
                cur[0, off:off + ln] = np.frombuffer(bytes(b.values[vo:vo + ln]), np.uint8)
                x.write_component(c, row, cur)
            elif kind == REMOVE:
                x.remove_component(c, row)
            elif kind == DESPAWN:
                x.despawn(row)
            else:
                x.spawn(count)

    rng = np.random.default_rng(5)
    warm = batch(rng)   # the first batch allocates the staging buffers
    e.apply_edits(warm.array(), bytes(warm.values))
    single(twin, warm)
    for pending in (0, 2):
        f = e.rollback_frame_count()
        expect = [twin.handle_requests(*tick(f + i)) for i in range(pending)]
        for i in range(pending):
            e.submit_requests(*tick(f + i))
        b = batch(rng)
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SLEEP_CYCLES)
        t0 = time.perf_counter()
        e.apply_edits(b.array(), bytes(b.values))
        dt = time.perf_counter() - t0
        busy = not stream.query()
        assert dt < 0.03, f"apply_edits took {dt * 1e3:.1f} ms behind a 100 ms kernel"
        assert busy, "the engine stream finished before apply_edits returned: the call waited"
        got = [e.collect() for _ in range(pending)]
        assert got == expect
        single(twin, b)
        f = e.rollback_frame_count()
        assert twin.rollback_frame_count() == f
        assert e.handle_requests(*tick(f)) == twin.handle_requests(*tick(f))
        for a, c in zip(_live(e), _live(twin)):
            assert np.array_equal(a, c)
    assert e.rollback_frame_count() > f0
    e.close(); twin.close()


def test_edits_store_only_the_planes_they_touch(monkeypatch):
    """Several waves, [Save(f), Advance] ticks in steady state: the launch trace's word [3] counts the 64-byte
    active-plane units each vector stored."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = max(262_144, 3 * sms * TILE + 4096) + 77
    monkeypatch.setenv("BGR_TUNE_PASSIVE_EARLY", "0")
    e = Engine(max_entities=n, max_depth=9)
    cols = register_particles(e)
    t_col, v_col, _ = cols
    e.build()
    populate(e, cols, *synth_particles(n, 9, 100_000, 200_000, z_fraction=0.2))
    e.set_depth(8)
    e.trace_enable(256)
    segs = -(-n // TILE) * (TILE // SEGMENT)
    launched = [0]

    def tick():
        f = e.rollback_frame_count()
        e.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, [0])])
        launched[0] += 1
        k = e.last_kernel()
        assert k.kind == "bundle" and k.stable_planes
        return int(e.trace_read(256)[launched[0] - 1, 3]), k

    def edit(c, rows, off, ln):
        vals = e.read_component(c, rows[0], len(rows))[:, off:off + ln].copy()
        vals.view(np.float32)[:] += np.float32(1.5)
        b = Batch()
        b.add(WRITE, c, rows[0], len(rows), off, ln, vals.tobytes())
        e.apply_edits(b.array(), bytes(b.values))

    for _ in range(20):
        tick()
    e.read_alive(0, 1)   # the baseline tick writes the live image eagerly, as a tick after an edit does
    base, k = tick()
    assert not k.passive_planes
    seg = 100
    rows = list(range(seg * SEGMENT + 3, seg * SEGMENT + 40))
    edit(v_col, rows, 0, 4)   # Velocity.x: no system changes it
    after, k = tick()
    # one (segment, plane) pair, stored into the Save's slot and into the live image: 4 units each
    assert 0 < after - base <= 2 * 4, (base, after)
    assert not k.passive_planes
    for _ in range(3):
        tick()
    edit(t_col, rows, 0, 12)   # Transform.translation only
    _, k = tick()
    assert not k.passive_planes
    edit(t_col, rows, 0, 40)   # the whole Transform: rotation and scale are passive planes
    _, k = tick()
    assert k.passive_planes
    for _ in range(12):
        tick()
    vals = e.read_component(v_col, rows[0], len(rows)).copy()
    vals.view(np.float32)[:, 0] -= np.float32(1.5)
    e.write_component(v_col, rows[0], vals)   # the same change through the single call
    single, k = tick()
    assert k.passive_planes
    assert single >= UNITS_PER_SEGMENT * segs, (single, UNITS_PER_SEGMENT * segs)
    e.close()
