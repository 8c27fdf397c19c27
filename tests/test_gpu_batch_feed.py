"""-m gpu: batched change-feed reports (bgr_batch_feed_begin / bgr_batch_feed_wait, EngineBatch.feed_begin / .feed_wait).

Members of one batch differ in rows, growth, optional columns and spawning (BGR_SYS_PARTICLES_SPAWN).  Each has a twin
engine on its own stream and an oracle.  After every batched tick a random subset of the members reports, in random
order, with caps of 0, below the rows that differ and above them: each entry's records and info must equal, byte for
byte, the twin's bgr_feed_begin of the same feed and cap, and the FeedModel of change_feed_model.py on the oracle's live
world, and a Replica fed the records must equal the oracle's world whenever nothing is pending.  Batched and single
reports of one feed alternate, feed_reset falls in between, a member reports with submits in flight, refusals change
nothing, and one call's launches do not grow with the number of worlds.  Every test runs on the interpreter and on
both item sizes of the generated kernel (the generic_kernel fixture); the random interleavings (a Fleet with batched
reports as one more action) run on the same three."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine, EngineBatch
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from change_feed_model import FeedModel, Replica, world_of
from interleave_driver import Fleet
from oracle_backend import OracleWorld
from test_gpu_batch_oracle import fleet_configs, fleet_engines
from test_gpu_generic_spawn import whole_transform

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
OPT = capi.BGR_STRATEGY_OPTIONAL
GROW = capi.BGR_CFG_GROWABLE
SPAWN = capi.BGR_INPUT_SPAWN
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
ROWS = [1, 700, 2000, 129, 40, 513]
MARGIN = 1024   # rows a sequence may add


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ registrations
def spawning(w, n, i):
    """The particles columns with spawn_particles (rate and seed per member, ttl 9: rows die and are not reclaimed) and
    an optional Score (+1 per frame) that spawned rows carry; one row in seven without it."""
    cols = register_particles(w, spawn_rate=5 + 3 * i, spawn_ttl=9, rng_seed=0xC0FFEE + i, checksums=whole_transform)
    s = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    w.checksum_component(s, 0, 4)
    w.add_system(capi.BGR_SYS_U32_ADD, [s], [0, 1])
    w.build()
    populate(w, cols, *synth_particles(n, i, 2, 30, 0.2))
    for r in range(0, n, 7):
        w.remove_component(s, r)
    return [(cols[0], 0, 12), (s, 0, 4), (cols[1], 4, 8)]   # translation, score, velocity.yz


def presence(w, n, i):
    """Score (optional, +1 per frame), Health (optional, despawns at 0), Tag: presence changes and despawns."""
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = w.rollback_component("Tag", 12, capi.BGR_STRATEGY_COPY)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        w.checksum_component(c, 0, ln)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(i)
    w.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    w.write_component(health, 0, rng.integers(2, 30, n, dtype=np.uint32))
    w.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in rng.choice(n, n // 5, replace=False):
        w.remove_component((score, health)[int(r) % 2], int(r))
    return [(score, 0, 4), (tag, 4, 8), (health, 0, 4)]


REGISTRATIONS = {"spawning": spawning, "presence": presence}


class Member:
    """A batch member (on the batch stream; every third one growable from 64 rows above its population), its twin on
    its own stream, its oracle, and one feed on the member and the twin with the model and replica of that feed."""

    def __init__(self, reg, i, stream):
        n = ROWS[i % len(ROWS)]
        self.grow = i % 3 == 2
        self.cap0 = n + 64 if self.grow else n + MARGIN
        self.eng = Engine(max_entities=self.cap0, max_depth=9, flags=GROW if self.grow else 0, stream=stream)
        self.twin = Engine(max_entities=n + MARGIN, max_depth=9)
        self.orc = OracleWorld(max_entities=n + MARGIN, max_depth=9)
        for w in (self.eng, self.twin, self.orc):
            self.fields = REGISTRATIONS[reg](w, n, i)
            w.set_depth(8)
        self.feed, self.tfeed = self.eng.feed_create(self.fields), self.twin.feed_create(self.fields)
        self.model = FeedModel(self.fields, n + MARGIN)
        self.replica = Replica(len(self.fields), [ln for _, _, ln in self.fields], n + MARGIN)

    def world(self):
        return world_of(self.orc, [c for c, _, _ in self.fields])

    def reset(self):
        self.eng.feed_reset(self.feed)
        self.twin.feed_reset(self.tfeed)
        self.model.reset()
        self.replica = Replica(len(self.fields), [ln for _, _, ln in self.fields], len(self.model.state))

    def draw_cap(self, rng, world):
        n = len(self.model.differing(world))
        return int(rng.choice([0, max(0, n - 1 - int(rng.integers(0, max(1, n)))), n + 5])), n

    def check(self, recs, info, world, cap, tally, what):
        """One report of this member's feed at `cap`: the twin's single report and the model's."""
        buf = self.twin.feed_alloc(self.tfeed, cap)
        trecs, tinfo = self.twin.feed_wait(self.twin.feed_begin(self.tfeed, buf, cap))
        want, winfo = self.model.report(world, cap)
        assert tuple(info) == tuple(winfo) == tuple(tinfo), f"{what}: info {info}, twin {tinfo}, model {winfo}"
        assert recs.tobytes() == trecs.tobytes(), f"{what}: records differ from the twin's"
        assert recs.tobytes() == want.tobytes(), f"{what}: records differ from the model's"
        self.replica.apply(recs)
        if winfo.pending == 0:
            assert self.replica.matches(self.model, world), f"{what}: the replica does not match the oracle's world"
        rows = self.orc.row_count()
        tally["unspawned"] += int(np.count_nonzero((recs["state"] == 0) & (recs["row"] >= rows)))
        tally["past_old_capacity"] += int(np.count_nonzero(recs["row"] >= self.cap0)) if self.grow else 0
        tally["capped"] += winfo.pending > 0
        tally["cap0"] += cap == 0

    def close(self):
        for w in (self.eng, self.twin, self.orc):
            w.close()


def fleet(reg, stream, k=6):
    members = [Member(reg, i, stream) for i in range(k)]
    return members, EngineBatch([m.eng for m in members])


def inputs(rng, spawn):
    a = [int(v) for v in rng.integers(0, 16, 2)]
    if spawn:
        a[0] |= SPAWN
    return a


def vector(m, rng):
    """A plain tick (spawning one time in two) or a rollback of 1..3 frames re-simulated without spawns, which
    un-spawns the rows the rolled-back frames spawned."""
    f, held = m.orc.rollback_frame_count(), [g for g in m.orc.snapshot_frames() if 0 < m.orc.rollback_frame_count() - g <= 3]
    if held and rng.random() < 0.35:
        g = int(rng.choice(held))
        reqs, k = [Request(LOAD, g)], g
        while k < f:
            if k > g:
                reqs.append(Request(SAVE, k))
            reqs.append(Request(ADVANCE, 0, inputs(rng, False)))
            k += 1
        return reqs + [Request(SAVE, f), Request(ADVANCE, 0, inputs(rng, rng.random() < 0.5))]
    return [Request(SAVE, f), Request(ADVANCE, 0, inputs(rng, rng.random() < 0.5))]


def batched_tick(batch, members, rng, skip=()):
    calls = [(i, NOSESS, vector(m, rng)) for i, m in enumerate(members) if i not in skip]
    expect = [members[i].orc.handle_requests(info, reqs) for i, info, reqs in calls]
    for (i, info, reqs), (status, cs), ex in zip(calls, batch.handle_requests(calls), expect):
        m = members[i]
        assert status == capi.BGR_OK and cs == ex, f"world {i}: batched checksums {cs} != oracle {ex}"
        assert m.twin.handle_requests(info, reqs) == ex, f"world {i}: twin"
        assert m.eng.snapshot_frames() == m.orc.snapshot_frames() == m.twin.snapshot_frames(), f"world {i}: snapshots"


def batched_report(batch, members, rng, listed, tally, what):
    calls, worlds = [], []
    for i in listed:
        world = members[i].world()
        cap, _ = members[i].draw_cap(rng, world)
        calls.append((i, members[i].feed, cap))
        worlds.append(world)
    buf = batch.feed_alloc(calls)
    res = batch.feed_wait(batch.feed_begin(calls, buf))
    assert len(res) == len(calls)
    for (i, _, cap), world, (recs, info) in zip(calls, worlds, res):
        members[i].check(recs, info, world, cap, tally, f"{what}: world {i} cap {cap}")
    tally["batched_entries"] += len(calls)


def single_report(m, rng, tally, what):
    world = m.world()
    cap, _ = m.draw_cap(rng, world)
    buf = m.eng.feed_alloc(m.feed, cap)
    recs, info = m.eng.feed_wait(m.eng.feed_begin(m.feed, buf, cap))
    m.check(recs, info, world, cap, tally, f"{what}: single report cap {cap}")
    tally["single"] += 1


# ------------------------------------------------------------------------------------------ batched = single = model
@pytest.mark.usefixtures("generic_kernel")
@pytest.mark.parametrize("reg", sorted(REGISTRATIONS))
def test_batched_reports_equal_single_reports_and_the_model(stream, reg):
    """Random subsets in random order after every batched tick, alternating with single reports of the same feeds and
    feed_reset, one member with an un-collected submit at begin time every fifth tick."""
    members, batch = fleet(reg, stream)
    rng = np.random.default_rng(sum(map(ord, reg)))
    tally = {k: 0 for k in ("unspawned", "past_old_capacity", "capped", "cap0", "batched_entries", "single", "queued")}
    try:
        for t in range(36):
            queued = int(rng.integers(0, len(members))) if t % 5 == 4 else None
            batched_tick(batch, members, rng, skip=() if queued is None else (queued,))
            if queued is not None:   # its vector in flight on the shared stream while the batched report begins
                m = members[queued]
                reqs = vector(m, rng)
                expect = m.orc.handle_requests(NOSESS, reqs)
                m.eng.submit_requests(NOSESS, reqs)
                assert m.twin.handle_requests(NOSESS, reqs) == expect
            order = [int(x) for x in rng.permutation(len(members))]
            listed = order[:int(rng.integers(1, len(members) + 1))]
            if queued is not None and queued not in listed:
                listed.append(queued)
            for i in order:
                if rng.random() < 0.08:
                    members[i].reset()
            if rng.random() < 0.25:   # single reports of some of the listed feeds first: both kinds advance one state
                for i in listed[: int(rng.integers(1, len(listed) + 1))]:
                    single_report(members[i], rng, tally, f"tick {t}")
            batched_report(batch, members, rng, listed, tally, f"tick {t}")
            if queued is not None:
                assert members[queued].eng.collect() == expect
                tally["queued"] += 1
        for i, m in enumerate(members):   # every feed in step with the model at the end
            batched_report(batch, members, rng, [i], tally, "end")
            assert m.eng.row_count() == m.orc.row_count()
        grown = any(m.eng.capacity()[0] > m.cap0 for m in members if m.grow)
    finally:
        batch.close()
        for m in members:
            m.close()
    print(f"\n[batched feed] {reg}: {tally}")
    assert tally["capped"] and tally["cap0"] and tally["single"] and tally["queued"], tally
    if reg == "spawning":
        assert tally["unspawned"] and tally["past_old_capacity"] and grown, tally


# ------------------------------------------------------------------------------------------ launches
@pytest.mark.usefixtures("generic_kernel")
def test_launches_do_not_grow_with_the_number_of_worlds(stream):
    """After a report that materialised every deferred live image, a batched report is four launches on the first
    listed world's engine and none on the others', whether it lists one world or six."""
    members, batch = fleet("spawning", stream)
    rng = np.random.default_rng(3)
    tally = {k: 0 for k in ("unspawned", "past_old_capacity", "capped", "cap0", "batched_entries")}
    try:
        for k in (1, 3, 6):
            batched_tick(batch, members, rng)
            listed = [int(x) for x in rng.permutation(len(members))[:k]]
            batched_report(batch, members, rng, listed, tally, f"{k} worlds, materialising")
            before = [m.eng.launch_count() for m in members]
            calls = [(i, members[i].feed, ROWS[i] + MARGIN) for i in listed]
            worlds = [members[i].world() for i in listed]
            buf = batch.feed_alloc(calls)
            res = batch.feed_wait(batch.feed_begin(calls, buf))
            grew = [m.eng.launch_count() - b for m, b in zip(members, before)]
            assert grew == [4 if i == listed[0] else 0 for i in range(len(members))], (k, listed, grew)
            for (i, _, cap), world, (recs, info) in zip(calls, worlds, res):
                members[i].check(recs, info, world, cap, tally, f"{k} worlds")
    finally:
        batch.close()
        for m in members:
            m.close()


# ------------------------------------------------------------------------------------------ refusals
def _refused(batch, members, calls, buf, status, text):
    before = [m.eng.launch_count() for m in members]
    with pytest.raises(BgrError) as ex:
        batch.feed_begin(calls, buf)
    assert ex.value.status == status, (calls, ex.value)
    assert str(ex.value).startswith(text), (calls, str(ex.value))
    assert [m.eng.launch_count() for m in members] == before, "a refused report launched"


@pytest.mark.usefixtures("generic_kernel")
def test_refusals_change_nothing(stream):
    """Every refusal leaves every feed's next report equal to the model's (no feed busy, no reported state moved), and
    members not listed untouched."""
    members, batch = fleet("presence", stream)
    rng = np.random.default_rng(5)
    tally = {k: 0 for k in ("unspawned", "past_old_capacity", "capped", "cap0", "batched_entries")}
    other = [m.eng.feed_create(m.fields[:1]) for m in members]   # another field list, another record size
    try:
        batched_tick(batch, members, rng)
        ok = [(i, members[i].feed, 50) for i in (4, 1, 3)]
        buf = batch.feed_alloc([(4, members[4].feed, 200)])   # room for every call below, the refused ones included
        inv, state = capi.BGR_ERR_INVALID_ARGUMENT, capi.BGR_ERR_STATE
        _refused(batch, members, ok + [(6, 0, 5)], buf, inv, "world 6: no such world in a batch of 6")
        _refused(batch, members, ok + [(1, members[1].feed, 5)], buf, inv, "world 1: listed twice in one call")
        _refused(batch, members, ok + [(0, 7, 5)], buf, inv, "world 0: unknown feed")
        _refused(batch, members, ok + [(0, other[0], 5)], buf, inv, "world 0: its feed's fields differ")
        _refused(batch, members, ok, np.zeros(4096, np.uint8), inv, "host_dst must come from bgr_host_alloc")
        # a single report of member 3's feed in flight
        m3 = members[3]
        sbuf = m3.eng.feed_alloc(m3.feed, 10)
        world3 = m3.world()
        t3 = m3.eng.feed_begin(m3.feed, sbuf, 10)
        _refused(batch, members, ok, buf, state, "world 3: a report of this feed is in flight")
        recs, info = m3.eng.feed_wait(t3)
        m3.check(recs, info, world3, 10, tally, "the single report a batched one was refused behind")
        # a batched report in flight refuses a second begin and single begins of its feeds
        worlds = [members[i].world() for i, _, _ in ok]
        t = batch.feed_begin(ok, buf)
        _refused(batch, members, [(0, members[0].feed, 5)], batch.feed_alloc([(0, members[0].feed, 5)]), state,
                 "a batched feed report of this batch is in flight")
        with pytest.raises(BgrError) as ex:
            members[4].eng.feed_begin(members[4].feed, members[4].eng.feed_alloc(members[4].feed, 5), 5)
        assert ex.value.status == state
        with pytest.raises(BgrError) as ex:
            batch.feed_wait(t + 1)
        assert ex.value.status == state
        for (i, _, cap), world, (recs, info) in zip(ok, worlds, batch.feed_wait(t)):
            members[i].check(recs, info, world, cap, tally, f"after the refusals: world {i}")
        with pytest.raises(BgrError) as ex:
            batch.feed_wait(t)
        assert ex.value.status == state
        # unlisted members untouched: every feed's next report is the model's
        batched_tick(batch, members, rng)
        batched_report(batch, members, rng, list(range(len(members))), tally, "every member after the refusals")
        batched_report(batch, members, rng, [], tally, "an empty call")
    finally:
        batch.close()
        for m in members:
            m.close()


# ------------------------------------------------------------------------------------------ buffers and destroy
@pytest.mark.usefixtures("generic_kernel")
def test_buffers_and_a_report_never_waited(stream):
    """EngineBatch.feed_begin refuses a buffer too small for sum(cap) records before the library runs anything; a call
    whose caps are all 0 takes no buffer; destroying a batch whose report was never waited frees its feeds, whose
    next reports continue from the state that report left."""
    members, batch = fleet("presence", stream)
    rng = np.random.default_rng(9)
    tally = {k: 0 for k in ("unspawned", "past_old_capacity", "capped", "cap0", "batched_entries")}
    other = None
    try:
        batched_tick(batch, members, rng)
        calls = [(2, members[2].feed, 40), (0, members[0].feed, 40)]
        small = batch.feed_alloc(calls[:1])
        before = [m.eng.launch_count() for m in members]
        with pytest.raises(AssertionError):
            batch.feed_begin(calls, small)
        assert [m.eng.launch_count() for m in members] == before
        worlds = [members[i].world() for i, _, _ in calls]
        zero = [(i, f, 0) for i, f, _ in calls]
        for (i, _, _), world, (recs, info) in zip(zero, worlds, batch.feed_wait(batch.feed_begin(zero, None))):
            members[i].check(recs, info, world, 0, tally, f"caps 0, no buffer: world {i}")
        # a second batch over the same engines begins a report and is destroyed without a wait
        other = EngineBatch([m.eng for m in members])
        listed = [3, 1, 5]
        worlds = [members[i].world() for i in listed]
        other.feed_begin([(i, members[i].feed, 7) for i in listed], other.feed_alloc([(i, members[i].feed, 7) for i in listed]))
        other.close()
        other = None
        for i, world in zip(listed, worlds):   # what the discarded report reported, on the model and the twin's feed
            members[i].model.report(world, 7)
            members[i].twin.feed_wait(members[i].twin.feed_begin(members[i].tfeed, members[i].twin.feed_alloc(members[i].tfeed, 7), 7))
            members[i].replica = Replica(len(members[i].fields), [ln for _, _, ln in members[i].fields], len(members[i].model.state))
        batched_tick(batch, members, rng)
        for i in listed:
            single_report(members[i], rng, {**tally, "single": 0}, f"after the unwaited report: world {i}")
        batched_report(batch, members, rng, list(range(len(members))), tally, "every member after the unwaited report")
    finally:
        if other is not None:
            other.close()
        batch.close()
        for m in members:
            m.close()


# ------------------------------------------------------------------------------------------ random interleavings
class FeedFleet(Fleet):
    """A Fleet with batched reports as one more action: a random subset of the members, in random order, reports one
    feed (the same feed index on each: one field list per call), also from between a member's queued submits, where
    that member may be listed with its vectors in flight.  Each entry is held to the member's feed model and replica as
    ``Interleaving.act_feed_report`` holds a single report."""

    def one_step(self) -> None:
        if self.rng.random() < 0.2:
            return self.act_batch_feed()
        return super().one_step()

    def act_between(self, exclude: int) -> None:
        if self.rng.random() < 0.5:
            return self.act_batch_feed(queued=exclude)
        return super().act_between(exclude)

    def act_batch_feed(self, queued=None) -> None:
        rng = self.rng
        avail = [i for i, m in enumerate(self.members) if m.feeds]
        if not avail:
            return self.note("(no feed)")
        k_feed = int(rng.integers(0, len(self.members[avail[0]].feeds)))
        worlds = [avail[int(j)] for j in rng.permutation(len(avail))[:int(rng.integers(1, len(avail) + 1))]]
        calls, seen = [], []
        for i in worlds:
            m = self.members[i]
            fe, _, model, _ = m.feeds[k_feed]
            world = world_of(m.orc, [f[0] for f in model.fields])
            n_diff = len(model.differing(world))
            cap = int(rng.choice([0, max(0, n_diff - 1 - int(rng.integers(0, max(1, n_diff)))), n_diff + 5]))
            m._touch()
            calls.append((i, fe, cap))
            seen.append((world, n_diff))
        self.note(f"batched feed report {k_feed} over {[(i, cap) for i, _, cap in calls]}"
                  + (f" (w{queued} has submits in flight)" if queued is not None else ""))
        res = self.batch.feed_wait(self.batch.feed_begin(calls, self.batch.feed_alloc(calls)))
        self.check(len(res) == len(calls), f"{len(res)} results for {len(calls)} entries")
        for (i, _, cap), (world, n_diff), (recs, info) in zip(calls, seen, res):
            m = self.members[i]
            _, _, model, replica = m.feeds[k_feed]
            expect, einfo = model.report(world, cap)
            m.check(tuple(info) == tuple(einfo), f"batched feed info {info} != model {einfo}")
            m.check(recs.tobytes() == expect.tobytes(), f"batched feed records differ from the model's "
                                                        f"(rows {recs['row'][:8].tolist()} vs {expect['row'][:8].tolist()})")
            replica.apply(recs)
            if einfo.pending == 0:
                m.check(replica.matches(model, world), "the replica does not match the model after a complete report")
            m.tally["feed_reports"] += 1
            m.tally["feed_reports_batched"] += 1
            m.tally["feed_cap_hit"] += cap < n_diff
            if i == queued:
                m.tally["feed_reports_batched_queued"] += 1
        self.tally["batch_feeds"] += 1


FLEETS = {"interpreter": "fallback", "jit": "jit_whole_rows4", "jit_quarter_tiles": "jit_quarter"}


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("kernel", sorted(FLEETS))
def test_random_interleavings_with_batched_reports(monkeypatch, stream, kernel):
    for k in ("BGR_TUNE_JIT", "BGR_TUNE_JIT_ITEM", "BGR_TUNE_JIT_ROWS"):
        monkeypatch.delenv(k, raising=False)
    fcfg = fleet_configs()[FLEETS[kernel]]
    total = {}
    for seed in range(6):
        fl = FeedFleet(fcfg, seed, fleet_engines(stream), EngineBatch)
        try:
            t = fl.run()
        finally:
            fl.close()
        for key, v in t.items():
            total[key] = total.get(key, 0) + v
    print(f"\n[batched feed interleavings] {kernel}: " + ", ".join(f"{k}={v}" for k, v in sorted(total.items()) if "feed" in k))
    for key, least in {"batch_feeds": 10, "feed_reports_batched": 20, "feed_reports_batched_queued": 1, "feed_cap_hit": 5}.items():
        assert total.get(key, 0) >= least, (key, total.get(key, 0))
