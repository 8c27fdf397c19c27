"""-m gpu: world batches (EngineBatch, bgr_batch_handle_requests, k_generic_jit_batch) held to the oracle.

- Random interleavings (interleave_driver.Fleet): fleets of members with one random registration, differing in rows,
  data, flags, fps and order_base (one above 2^32, one whose RollbackOrdered range crosses 2^32 inside a tile), under
  the default kernel selection (solo vectors of small worlds run the interpreter, batched ones the generated kernel),
  forced instances of the generated kernel, the sequential fallback, the widest registration the generated kernel
  takes, and a multi-wave member among tiny ones.
- Shape parity on all nine (item rows, rows per thread) instances of the batch kernel: members of 0 rows and on either
  side of tile and work-item boundaries, per-member fps and order_base, every session kind; and a 25-word registration,
  which the batch runs sequentially.
- The default selection's hand-over: one member alternating solo vectors (interpreter) and batched ones (generated
  kernel) through rollbacks to slots the other kernel wrote, deferred live images planned by one and consumed by the
  other, and growth past 16 384 rows, after which its solo vectors run its own generated kernel.
- The C contract through ctypes: sessions == NULL, empty vectors, checksums_cap below the total, and one call over
  1 000 worlds.

Replay one interleaving configuration and seed: BGR_INTERLEAVE_REPLAY=<configuration>:<seed>."""
import contextlib
import ctypes as C
import os
import time
from collections import Counter

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine, EngineBatch
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request
from interleave_driver import Config, Fleet, FleetConfig, World, replay_filter
from oracle_backend import OracleWorld
from schema_util import random_schema
from test_gpu_batch import driver

pytestmark = [pytest.mark.gpu]
OPT = capi.BGR_STRATEGY_OPTIONAL
CAPTURE, GROW = capi.BGR_CFG_DESYNC_CAPTURE, capi.BGR_CFG_GROWABLE
ABOVE = (1 << 32) + 12345   # an order_base above 2^32
CROSS = (1 << 32) - 700     # rows 700.. of tile 1 cross 2^32
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
TUNE_VARS = ("BGR_TUNE_JIT", "BGR_TUNE_JIT_ITEM", "BGR_TUNE_JIT_ROWS")


@pytest.fixture
def batch_env(monkeypatch):
    """Sets the generated kernel's selection variables to exactly ``values`` (the others unset: their defaults)."""
    def set_env(values):
        for k in TUNE_VARS:
            monkeypatch.delenv(k, raising=False)
        for k, v in values.items():
            monkeypatch.setenv(k, v)
    set_env({})
    return set_env


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


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


def _sms() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------ random interleavings
def registration(sizes=None, rows=(1000, 2500), big_member=None):
    """A random registration the generated kernel takes (whole-word columns and checksummed ranges), or one of the
    given element sizes with every checksummed range whole; members of ``rows`` rows, member 0 of ``big_member``."""
    def draw(rng):
        if sizes is None:
            sz = [int(x) for x in rng.choice([4, 8, 12, 16, 40], int(rng.integers(2, 5)))]
            while sum(sz) > 96:   # at most 24 words
                sz.pop()
            s = random_schema(rng, sizes=sz, ranges=("none", "whole"))
        else:
            s = random_schema(rng, sizes=sizes, ranges=("whole",))
        strategies = [(capi.BGR_STRATEGY_COPY | OPT) if o else capi.BGR_STRATEGY_CLONE for o in s.optional]
        feed = [(c, 0, min(8, sz)) for c, sz in enumerate(s.sizes) if sz % 4 == 0][:3]

        def make(rng, member):
            n = big_member if big_member and member == 0 else int(rng.integers(*rows))
            removes = [(c, int(r)) for c, o in enumerate(s.optional) if o for r in rng.choice(n, min(n, 9), replace=False)]
            return World(s.sizes, strategies, [(c, off, ln, 0) for c, off, ln in s.cks], s.systems, s.values(rng, n),
                         removes, feed_fields=feed)
        return make
    return draw


def _member(**kw):
    return Config("", None, **kw)


# flags 0, desync capture, growth, retention, growth with capture; fps 30 / 60 / 144; order_base 0, above 2^32 and
# crossing it (growth and spawns are refused with order_base != 0)
MEMBERS = [_member(), _member(flags=CAPTURE, fps=30), _member(flags=GROW, fps=144, grow_margin=3000),
           _member(retain=(2, 4), order_base=ABOVE), _member(flags=GROW | CAPTURE, grow_margin=3000),
           _member(flags=CAPTURE, fps=144, order_base=CROSS)]
SEEDS = list(range(6))


def fleet_configs():
    one_wave = 3 * _sms() * 512
    jit2 = {"BGR_TUNE_JIT": "2"}
    return {
        "default_env": FleetConfig("default_env", registration(), MEMBERS, steps=110),
        "jit_quarter": FleetConfig("jit_quarter", registration(), MEMBERS, env=jit2),
        "jit_whole_rows4": FleetConfig("jit_whole_rows4", registration(), MEMBERS, env={**jit2, "BGR_TUNE_JIT_ITEM": "512"}),
        "item256_rows1": FleetConfig("item256_rows1", registration(), MEMBERS,
                                     env={**jit2, "BGR_TUNE_JIT_ITEM": "256", "BGR_TUNE_JIT_ROWS": "1"}),
        "fallback": FleetConfig("fallback", registration(), MEMBERS, env={"BGR_TUNE_JIT": "0"}),
        # 24 words, a 16-word checksummed range: the generated kernel's limits
        "wide": FleetConfig("wide", registration(sizes=[64, 16, 8, 8]), MEMBERS, env=jit2),
        "multi_wave": FleetConfig("multi_wave", registration(rows=(1, 400), big_member=one_wave + 300),
                                  [_member(), _member(flags=CAPTURE, fps=30), _member(order_base=CROSS),
                                   _member(flags=GROW, grow_margin=3000)], steps=50),
    }


FLEETS = ["default_env", "jit_quarter", "jit_whole_rows4", "item256_rows1", "fallback", "wide", "multi_wave"]


def fleet_engines(stream):
    def make(member, role, max_entities, flags, env, fps=60, order_base=0):
        with _env(env):   # read once, at bgr_engine_create
            return Engine(max_entities=max_entities, max_depth=9, fps=fps, flags=flags, order_base=order_base,
                          stream=stream if role == "engine" else None)
    return make


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", FLEETS)
def test_random_batched_interleavings_match_the_oracle(batch_env, stream, name):
    fcfg = fleet_configs()[name]
    total, ran, t0 = Counter(), 0, time.perf_counter()
    for seed in SEEDS:
        r = replay_filter()
        if r is not None and r != (name, seed):
            continue
        fl = Fleet(fcfg, seed, fleet_engines(stream), EngineBatch)
        try:
            assert fl.specialised == (name != "fallback")
            t = fl.run()
            if name == "default_env":
                # every member ran both ways; small worlds run their solo vectors on the interpreter and batched ones on
                # the generated kernel (a growable member's first growth maps past 16 384 rows: its own generated kernel)
                for i, m in enumerate(fl.members):
                    solo = m.tally["solo_generic_interpreter"] + m.tally["solo_generic_nvrtc"]
                    assert solo > 0 and m.tally["batched_generic_nvrtc"] > 0, f"seed {seed} member {i}: {dict(m.tally)}"
                    if not m.growable:
                        assert m.tally["solo_generic_nvrtc"] == 0, f"seed {seed} member {i}: {dict(m.tally)}"
            if name == "multi_wave":
                assert fl.members[0].orc.row_count() >= 3 * _sms() * 512
        finally:
            fl.close()
        ran += 1
        total.update(t)
    if not ran:
        pytest.skip("not the configuration BGR_INTERLEAVE_REPLAY selects")
    print(f"\n[batch interleavings] {name}: {time.perf_counter() - t0:.1f} s, "
          + ", ".join(f"{k}={v}" for k, v in sorted(total.items())))
    if ran < len(SEEDS):
        return   # a replay: the tally minimums are over every seed
    minimums = {"batched_calls": 30, "batched_worlds": 60, "batch_refusals": 1, "batch_with_queued_member": 1,
                "solo_after_batched": 5, "batched_after_solo": 5, "vectors_queued": 5, "invalid_rollbacks": 1,
                "band_writes": 3, "despawns": 1, "peeks": 3, "live_reads": 2, "feed_reports": 2}
    if name != "multi_wave":
        minimums.update({"growth_steps": 1, "spawns": 1, "capture_reads": 1, "retained_released": 1})
    if name != "fallback":
        minimums.update({"batched_generic_nvrtc": 60, "materialisations": 1, "from_deferred": 1})
    else:
        minimums.update({"batched_generic_interpreter": 60})
    if name == "default_env":
        minimums.update({"solo_generic_interpreter": 10})
    missing = {k: (total[k], v) for k, v in minimums.items() if total[k] < v}
    assert not missing, f"{name}: tally below its minimum (reached, minimum): {missing}"


# ------------------------------------------------------------------------------------------ shared helpers
def schema(words25=False):
    """A fixed registration: 11 words, or 25 (one word more than the generated kernel takes); two optional columns,
    every range whole, U32_ADD / U32_SATSUB_DESPAWN systems."""
    rng = np.random.default_rng(0xBA7C)
    return random_schema(rng, sizes=[40, 40, 12, 8] if words25 else [12, 4, 16, 8, 4], ranges=("whole",), n_opt=2)


def populate(s, w, n, seed, ring=None):
    """Registers ``s`` on an engine or oracle world, builds it and spawns n rows of seeded data."""
    s.register(w)
    w.build()
    if ring:
        w.set_depth(ring)
    if n == 0:
        return
    rng = np.random.default_rng(seed)
    w.spawn(n)
    for c, d in enumerate(s.values(rng, n)):
        w.write_component(c, 0, d)
    for c, o in enumerate(s.optional):
        if o:
            for r in rng.choice(n, max(1, n // 7), replace=False):
                w.remove_component(c, int(r))


def pair(s, n, depth, seed, stream, fps=60, order_base=0, flags=0, ring=None):
    """A batch member on ``stream`` and its oracle; ``ring``: their snapshot depth (set_depth), for vectors without a
    session, which confirm nothing (the oldest frame makes room only below max_depth)."""
    e = Engine(max_entities=n + 8, max_depth=depth, fps=fps, order_base=order_base, flags=flags, stream=stream)
    o = OracleWorld(max_entities=n + 8, max_depth=depth, fps=fps, order_base=order_base)
    for w in (e, o):
        populate(s, w, n, seed, ring)
    return e, o


def assert_matches_oracle(e, o, what, rows_of=None):
    """Counters, alive rows, presence and present bytes, live and in every held frame (``rows_of(frame)``: its rows,
    if they differ from the live row count)."""
    assert e.rollback_frame_count() == o.rollback_frame_count(), what
    assert e.snapshot_frames() == o.snapshot_frames(), what
    n = o.row_count()
    assert e.row_count() == n, what
    if n == 0:
        return
    assert np.array_equal(e.read_alive(0, n).astype(bool), o.read_alive(0, n).astype(bool)), f"{what}: alive rows"
    for c in range(len(e.elem_bytes)):
        vo, ho = o.read_component_alive(c, 0, n)
        he = e.has_component(c, 0, n).astype(bool)
        assert np.array_equal(he, ho.astype(bool)), f"{what}: presence of column {c}"
        assert np.array_equal(e.read_component(c, 0, n)[he], vo[he]), f"{what}: live bytes of column {c}"
        for f in o.snapshot_frames():
            k = rows_of(f) if rows_of else n
            pe, po = e.peek(f, c, 0, k), o.peek(f, c, 0, k)
            pres = po[1].astype(bool)
            assert np.array_equal(pe[1].astype(bool), pres), f"{what}: presence of column {c} in frame {f}"
            assert np.array_equal(pe[0][pres], po[0][pres]), f"{what}: column {c} of frame {f}"


def assert_bytes_equal(e, t, what, rows_of=None):
    """Every byte below the row count, dead rows and absent components included, live and in every held frame."""
    n = e.row_count()
    assert t.row_count() == n and e.snapshot_frames() == t.snapshot_frames(), what
    assert np.array_equal(e.read_alive(0, n), t.read_alive(0, n)), f"{what}: alive bytes"
    for c in range(len(e.elem_bytes)):
        assert np.array_equal(e.read_component(c, 0, n), t.read_component(c, 0, n)), f"{what}: live column {c}"
        assert np.array_equal(e.has_component(c, 0, n), t.has_component(c, 0, n)), f"{what}: live presence {c}"
        for f in e.snapshot_frames():
            k = rows_of(f) if rows_of else n
            pe, pt = e.peek(f, c, 0, k), t.peek(f, c, 0, k)
            assert np.array_equal(pe[0], pt[0]) and np.array_equal(pe[1], pt[1]), f"{what}: column {c} of frame {f}"


# ------------------------------------------------------------------------------------------ shape parity
PARITY_ROWS = [0, 1, 511, 512, 513, 1023, 1024, 1025]
FPS = [30, 60, 144]
BASES = [0, ABOVE, CROSS]
INSTANCES = [(item, rows) for item in (128, 256, 512) for rows in (1, 2, 4)]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("item,rows", INSTANCES + [(0, 0)], ids=[f"item{i}_rows{r}" for i, r in INSTANCES] + ["words25"])
def test_shape_parity_with_the_oracle(batch_env, stream, item, rows):
    """Every instance of the batch kernel against the oracle on members of 0, 1 and 511..1025 rows, per-member fps and
    order_base, every session kind.  (0, 0): a 25-word registration, which the batch runs one world after another."""
    batch_env({"BGR_TUNE_JIT": "2"} if item == 0 else
              {"BGR_TUNE_JIT": "2", "BGR_TUNE_JIT_ITEM": str(item), "BGR_TUNE_JIT_ROWS": str(rows)})
    s = schema(words25=item == 0)
    assert (s.words == 25) == (item == 0)
    k = 2 * len(PARITY_ROWS)
    drivers = [driver(i) for i in range(k)]
    worlds = [pair(s, PARITY_ROWS[i % len(PARITY_ROWS)], drivers[i].depth, 100 + i, stream,
                   fps=FPS[i % 3], order_base=BASES[(i + i // 3) % 3]) for i in range(k)]
    batch = EngineBatch([e for e, _ in worlds])
    assert batch.specialised() == (item != 0)
    rng = np.random.default_rng(item * 10 + rows)
    ticks = [0] * k
    for call in range(36):
        listed = [int(w) for w in rng.permutation(k)[:k if call % 3 == 0 else int(rng.integers(1, k + 1))]]
        calls = []
        for w in listed:
            calls.append((w,) + drivers[w].next(ticks[w]))
            ticks[w] += 1
        expect = [worlds[w][1].handle_requests(info, reqs) for w, info, reqs in calls]
        for (w, info, reqs), (status, cs), ex in zip(calls, batch.handle_requests(calls), expect):
            what = f"call {call} world {w} ({PARITY_ROWS[w % len(PARITY_ROWS)]} rows)"
            assert status == capi.BGR_OK and cs == ex, what
            drivers[w].saved(cs)
            lk = worlds[w][0].last_kernel()
            if item:
                assert lk.batched and lk.kind == "generic_nvrtc" and lk.item_rows == item, f"{what}: {lk}"
            else:
                assert not lk.batched, what
    for w, (e, o) in enumerate(worlds):
        assert_matches_oracle(e, o, f"world {w} ({PARITY_ROWS[w % len(PARITY_ROWS)]} rows)")
    batch.close()


# ------------------------------------------------------------------------------------------ default-selection hand-over
def test_default_selection_hands_over_between_kernels(batch_env, stream):
    """One small member under the default selection: solo vectors run the interpreter, batched ones the generated
    kernel.  Alternating them hands ring slots and deferred live images from one kernel to the other; growing past
    16 384 rows compiles the member's own generated kernel for its solo vectors.  Checksums against the oracle, every
    byte against a twin that only runs the interpreter."""
    s = schema()
    n, depth = 1500, 9
    e = Engine(max_entities=n + 8, max_depth=depth, flags=GROW, stream=stream)
    with _env({"BGR_TUNE_JIT": "0"}):
        twin = Engine(max_entities=40000, max_depth=depth)
    o = OracleWorld(max_entities=40000, max_depth=depth)
    for w in (e, twin, o):
        populate(s, w, n, 7, ring=8)
    other, other_o = pair(s, 300, depth, 8, stream, ring=8)
    batch = EngineBatch([e, other])
    assert batch.specialised()
    rng = np.random.default_rng(11)
    saved_by, frame_rows, seen = {}, {}, Counter()
    pattern = ["solo", "batched", "batched", "solo", "solo", "batched"]
    grown = False
    for tick in range(72):
        way = pattern[tick % len(pattern)]
        f, frames = o.rollback_frame_count(), o.snapshot_frames()
        shape = ["rollback", "plain", "catchup", "rollback", "plain"][tick % 5]
        near = [g for g in frames if 0 < f - g <= 6]
        if shape == "rollback" and near:
            g = int(rng.choice(near))
            seen["loads_of_other_kernel"] += saved_by.get(g) not in (None, way)
            reqs, kf = [Request(LOAD, g)], g
            while kf < f:
                if kf > g:
                    reqs.append(Request(SAVE, kf))
                reqs.append(Request(ADVANCE, 0, [tick & 15])); kf += 1
            reqs += [Request(SAVE, f), Request(ADVANCE, 0, [0])]
        elif shape == "catchup":
            reqs = [Request(ADVANCE, 0, [tick & 15])]
        else:
            reqs = [Request(SAVE, f), Request(ADVANCE, 0, [tick & 15])]
        rows = o.row_count()
        for q in reqs:   # the rows of each saved frame (no system spawns: only a Load changes them inside a vector)
            if q.kind == LOAD:
                rows = frame_rows[q.frame]
            elif q.kind == SAVE:
                saved_by[q.frame], frame_rows[q.frame] = way, rows
        expect = o.handle_requests(NOSESS, reqs)
        if way == "solo":
            got = e.handle_requests(NOSESS, reqs)
        else:
            ofr = other_o.rollback_frame_count()
            oreq = [Request(SAVE, ofr), Request(ADVANCE, 0, [1])]
            res = batch.handle_requests([(1, NOSESS, oreq), (0, NOSESS, reqs)] if tick % 2 else
                                        [(0, NOSESS, reqs), (1, NOSESS, oreq)])
            got = dict(zip((1, 0) if tick % 2 else (0, 1), [cs for _, cs in res]))
            assert got[1] == other_o.handle_requests(NOSESS, oreq), f"tick {tick}: the other member"
            got = got[0]
        assert got == expect, f"tick {tick} ({way} {shape}): checksums {got} != oracle {expect}"
        assert twin.handle_requests(NOSESS, reqs) == expect, f"tick {tick}: the interpreter twin"
        lk = e.last_kernel()
        want = "generic_nvrtc" if way == "batched" or grown else "generic_interpreter"
        assert lk.kind == want and lk.batched == (way == "batched"), f"tick {tick} ({way}): {lk}"
        seen[f"{way}_from_deferred"] += lk.from_deferred and pattern[(tick - 1) % len(pattern)] != way
        seen[f"{way}_deferred"] += lk.deferred_live
        if tick == 40:   # spawn past 16 384 rows: the member grows and compiles its own generated kernel
            add = 16000
            vals = [v for v in s.values(rng, add)]
            for w in (e, twin, o):
                first = w.spawn(add)
                for c, v in enumerate(vals):
                    w.write_component(c, first, v)
            assert e.capacity()[0] >= 16384
            grown = True
        if tick % 12 == 11:   # reads materialise the deferred image: only every few ticks
            assert_bytes_equal(e, twin, f"tick {tick}", frame_rows.get)
    assert_bytes_equal(e, twin, "end", frame_rows.get)
    assert_matches_oracle(e, o, "end", frame_rows.get)
    assert seen["loads_of_other_kernel"] >= 3, seen
    assert seen["solo_from_deferred"] >= 1 and seen["batched_from_deferred"] >= 1, seen
    batch.close()


# ------------------------------------------------------------------------------------------ the C contract
def raw_call(batch, calls, sessions=True, cap=None, sentinel=0x5A):
    """bgr_batch_handle_requests through ctypes, laid out as the header documents.  Returns (status, every checksum
    slot of an output array sized to the total, n_checksums_out, status_out); slots the call did not write keep
    ``sentinel`` bytes."""
    lib = capi.load_library()
    n = len(calls)
    worlds = (C.c_uint32 * max(1, n))(*[w for w, _, _ in calls])
    sess = (capi.bgr_session_info * max(1, n))(*[capi.make_session_info(si) for _, si, _ in calls]) if sessions else None
    reqs = capi.make_requests([q for _, _, r in calls for q in r])
    n_req = (C.c_uint32 * max(1, n))(*[len(r) for _, _, r in calls])
    total = sum(q.kind == SAVE for _, _, r in calls for q in r)
    out = (capi.bgr_checksum * max(1, total))()
    C.memset(out, sentinel, C.sizeof(out))
    n_cs = (C.c_uint32 * max(1, n))(*([0xFFFF] * max(1, n)))
    status = (C.c_int32 * max(1, n))(*([-77] * max(1, n)))
    rc = lib.bgr_batch_handle_requests(batch._h, worlds, n, sess, reqs, n_req, out, total if cap is None else cap, n_cs, status)
    return rc, [bytes(o) for o in out[:total]], list(n_cs[:n]), list(status[:n])


def checksum_bytes(frame, value):
    cs = capi.bgr_checksum(frame, 1, value & ((1 << 64) - 1), value >> 64)
    return bytes(cs)


def _plain(e_or_o, k):
    f = e_or_o.rollback_frame_count()
    return [q for i in range(k) for q in (Request(SAVE, f + i), Request(ADVANCE, 0, [i & 15]))]


@pytest.mark.parametrize("selection", ["generated", "sequential"])
def test_null_sessions_and_empty_vectors(batch_env, stream, selection):
    """sessions == NULL and worlds listed with n_requests[i] == 0: what bgr_handle_requests gives on twins, with the
    same launch counts."""
    batch_env({"BGR_TUNE_JIT": "2" if selection == "generated" else "0"})
    s = schema()
    sizes = [1, 700, 0, 1500, 512, 90]
    members = [pair(s, n, 9, 30 + i, stream, ring=8) for i, n in enumerate(sizes)]
    twins = []
    for i, n in enumerate(sizes):
        t = Engine(max_entities=n + 8, max_depth=9)
        populate(s, t, n, 30 + i, ring=8)
        twins.append(t)
    batch = EngineBatch([e for e, _ in members])
    assert batch.specialised() == (selection == "generated")
    rng = np.random.default_rng(5)
    for call in range(16):
        listed = [int(w) for w in rng.permutation(len(sizes))[:int(rng.integers(1, len(sizes) + 1))]]
        calls = [(w, NOSESS, [] if (w + call) % 3 == 0 else _plain(twins[w], int(rng.integers(1, 4)))) for w in listed]
        before = [(members[w][0].launch_count(), twins[w].launch_count()) for w in listed]
        rc, out, n_cs, status = raw_call(batch, calls, sessions=False)
        assert rc == capi.BGR_OK and status == [capi.BGR_OK] * len(calls), (call, rc, status)
        k = 0
        for (w, info, reqs), n, (lm, lt) in zip(calls, n_cs, before):
            expect = twins[w].handle_requests(info, reqs)
            assert n == len(expect), f"call {call} world {w}"
            assert out[k:k + n] == [checksum_bytes(f, v) for f, v in expect], f"call {call} world {w}"
            assert members[w][0].launch_count() - lm == twins[w].launch_count() - lt, f"call {call} world {w}: launches"
            k += n
    for w, (e, _) in enumerate(members):
        assert_bytes_equal(e, twins[w], f"world {w}")
    batch.close()


@pytest.mark.parametrize("cap_of", [lambda total: 0, lambda total: 1, lambda total: total // 2, lambda total: total - 1],
                         ids=["cap0", "cap1", "half", "one_short"])
def test_checksums_cap_below_the_total(batch_env, stream, cap_of):
    """A capped call writes the uncapped call's prefix and nothing past the cap; n_checksums_out counts every checksum
    and every status is OK.  The cap changes no world: both fleets stay identical."""
    batch_env({"BGR_TUNE_JIT": "2"})
    s = schema()
    sizes = [300, 1025, 5, 2000]
    fleets = [[pair(s, n, 9, 50 + i, stream, ring=8)[0] for i, n in enumerate(sizes)] for _ in range(2)]
    full, capped = EngineBatch(fleets[0]), EngineBatch(fleets[1])
    for call in range(6):
        order = [3, 0, 2, 1] if call % 2 else [1, 2, 3, 0]
        calls = [(w, NOSESS, _plain(fleets[0][w], 1 + (w + call) % 3)) for w in order]
        res = full.handle_requests(calls)
        every = [checksum_bytes(f, v) for _, cs in res for f, v in cs]
        cap = cap_of(len(every))
        rc, out, n_cs, status = raw_call(capped, calls, cap=cap)
        assert rc == capi.BGR_OK and status == [capi.BGR_OK] * len(calls)
        assert n_cs == [len(cs) for _, cs in res]
        assert out[:cap] == every[:cap]
        assert out[cap:] == [bytes([0x5A]) * C.sizeof(capi.bgr_checksum)] * (len(every) - cap), "written past the cap"
    for a, b in zip(*fleets):
        assert_bytes_equal(a, b, "capped fleet")
    full.close()
    capped.close()


@pytest.mark.timeout(600)
def test_one_call_over_a_thousand_worlds(batch_env, stream):
    """1 000 worlds of mixed sizes in one launch: the block -> world binary search over item0 runs ten levels deep."""
    batch_env({"BGR_TUNE_JIT": "2"})
    s = schema()
    rng = np.random.default_rng(1000)
    sizes = [int(x) for x in rng.choice([1, 7, 130, 511, 512, 513, 1500, 3000], 1000)]
    worlds = [pair(s, n, 9, 2000 + i, stream, fps=FPS[i % 3], order_base=BASES[i % 3], ring=8) for i, n in enumerate(sizes)]
    batch = EngineBatch([e for e, _ in worlds])
    assert batch.specialised()
    for call in range(4):
        order = [int(w) for w in rng.permutation(len(worlds))]
        calls = []
        for w in order:
            o = worlds[w][1]
            f = o.rollback_frame_count()
            if call == 3:   # a rollback to frame 1
                reqs = [Request(LOAD, 1), Request(ADVANCE, 0, [1]), Request(SAVE, 2), Request(ADVANCE, 0, [2]),
                        Request(SAVE, 3), Request(ADVANCE, 0, [3])]
            else:
                reqs = [Request(SAVE, f), Request(ADVANCE, 0, [w & 15])]
            calls.append((w, NOSESS, reqs))
        expect = [worlds[w][1].handle_requests(info, reqs) for w, info, reqs in calls]
        for (w, _, _), (status, cs), ex in zip(calls, batch.handle_requests(calls), expect):
            assert status == capi.BGR_OK and cs == ex, f"call {call} world {w} ({sizes[w]} rows)"
            assert worlds[w][0].last_kernel().batched
    for w in rng.choice(len(worlds), 40, replace=False):
        e, o = worlds[int(w)]
        assert_matches_oracle(e, o, f"world {w} ({sizes[int(w)]} rows)")
    batch.close()
