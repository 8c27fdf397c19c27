"""Seeded random interleavings of the engine's entry points, checked against the oracle and an engine twin.

Three worlds run the same actions: the engine under test, a twin with every elision that can be switched off switched
off (no deferred live image, no tile dependencies, the bundle kernel's instance without content stamps; it runs queued
vectors synchronously), and the oracle (``FlagsOracle``: desync capture and the digests of
retained frames), plus a ``FeedModel`` per change feed.  The generator draws every action from the oracle's state and the
engine's documented limits (existing snapshot frames, row count, capacity, at most 8 vectors in flight,
BGR_MAX_REQUESTS = 80), so the action log depends on the seed alone.

What is compared:
  - the checksums of every vector, synchronous or collected, in order, and the frame resources, snapshot frames and row
    count after every step: the oracle's;
  - alive rows, presence and the bytes of present components on alive rows, live and in every peek: the oracle's;
  - every byte below the row count, dead rows and absent components included, in the live image, every snapshot and
    every first image: the twin's;
  - feed records and FeedInfo: the FeedModel's on the oracle's world, and a Replica that applies them must match it;
  - desync diffs, digests, retained frames: the oracle's; export blobs: the twin's, and ``diff_remote`` of the engine's
    blob on the twin finds nothing.

The host bookkeeping behind the skipped work (passive-plane versions, content stamps, the deferred live image) is what
these interleavings exercise; a stale record does not fault, it skips a store, so only a comparison finds it.  Each run
counts what it reached (``Interleaving.tally``) so that a test can assert that it reached it.

``Fleet`` runs several such worlds with one registration as the members of one world batch (``EngineBatch``): batched
calls over random subsets of them, refused batched calls, and each member's own actions in between.

``REPLAY_ENV`` ("<configuration>:<seed>") restricts a test module to one configuration and seed.

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

import os
from collections import Counter
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, P2PTraceSession, Request, SyncTestSession
from change_feed_model import FeedModel, Replica, world_of
from oracle_backend import OracleWorld
from oracle_desync import _is_older
from oracle_p2p import BLOCK, RetainOracleWorld

REPLAY_ENV = "BGR_INTERLEAVE_REPLAY"
MAX_REQUESTS = capi.BGR_MAX_REQUESTS
MAX_QUEUED = 8
MAX_SAVES = 40
STAMP_LIMIT = 0xFFFFFFFF - (MAX_REQUESTS + 1)   # run_fused clears the stamp table when the next stamp is past this
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
TILE = 512
SEGMENT = 64
UNITS_PER_SEGMENT = 33   # 64-byte units of one 64-row segment's active planes: 8 word planes of 4 units, the alive plane 1
TRACE_CAP = 4096
TWIN_ENV = {"BGR_TUNE_DEFER_LIVE": "0", "BGR_TUNE_TILEDEP": "0", "BGR_TUNE_JIT_TILEDEP": "0", "BGR_TUNE_PASSIVE_EARLY": "1"}


def replay_filter() -> Optional[Tuple[str, int]]:
    v = os.environ.get(REPLAY_ENV)
    if not v:
        return None
    name, seed = v.rsplit(":", 1)
    return name, int(seed)


@dataclass
class World:
    """A registration and its initial population, applied identically to every world."""
    sizes: List[int]
    strategies: List[int]
    cks: List[Tuple[int, int, int, int]]               # (column, byte offset, byte length, flags)
    systems: List[Tuple[int, List[int], List[int]]]
    data: List[np.ndarray]                              # initial element bytes per column, [n, size] u8
    removes: List[Tuple[int, int]] = field(default_factory=list)   # (column, row) made absent after the population
    spawn_rate: int = 0                                 # BGR_SYS_PARTICLES_SPAWN's rate (0: not registered)
    bundle: bool = False                                # the particles schema: Transform, Velocity, Ttl
    feed_fields: List[Tuple[int, int, int]] = field(default_factory=list)

    @property
    def n(self) -> int:
        return len(self.data[0])

    @property
    def optional(self) -> List[bool]:
        return [bool(s & capi.BGR_STRATEGY_OPTIONAL) for s in self.strategies]

    def register(self, w, retain: Optional[Tuple[int, int]]) -> None:
        for i, (s, st) in enumerate(zip(self.sizes, self.strategies)):
            w.rollback_component(f"C{i}", s, st)
        for c, off, ln, fl in self.cks:
            w.checksum_component(c, off, ln, fl)
        for sid, c, p in self.systems:
            w.add_system(sid, c, p)
        if retain:
            w.retain_confirmed(*retain)
        w.build()
        w.spawn(self.n)
        for c, d in enumerate(self.data):
            w.write_component(c, 0, d)
        for c, r in self.removes:
            w.remove_component(c, r)


@dataclass
class Config:
    name: str
    world: Callable[[np.random.Generator], World]
    flags: int = 0
    retain: Optional[Tuple[int, int]] = None
    env: Dict[str, str] = field(default_factory=dict)
    kind: Optional[str] = None          # the kernel every vector must run (Engine.last_kernel().kind)
    stamped: bool = False               # every bundle launch runs the instance with content stamps
    steps: int = 60
    digests: int = 1_000_000            # frame digests per run (the oracle's digest is a Python loop)
    grow_margin: int = 4096             # rows the sequence may add (the twin's capacity past the initial rows)
    fps: int = 60                       # bgr_config.fps: Time<GgrsTime>'s dt reaches the systems through each Advance
    order_base: int = 0                 # bgr_config.order_base: the RollbackOrdered index of row 0 (no spawns past the
                                        # first vector then, so the generator draws none)


class FlagsOracle(RetainOracleWorld):
    """The oracle of an engine with any of the flags: ``RetainOracleWorld``'s retention and ``CaptureOracleWorld``'s first
    images (the witness release rules of ring.hpp) on the same Saves."""

    def handle_requests(self, session_info, requests):
        out = []
        for r in requests:
            if r.kind != SAVE:
                out += OracleWorld.handle_requests(self, session_info, [r])
                continue
            frame = self.rollback_frame_count()
            if frame in self._retained:
                self._retained.remove(frame)
            before = set(self.snapshot_frames())
            out += OracleWorld.handle_requests(self, session_info, [r])
            left = before - set(self.snapshot_frames())
            confirmed = self.confirmed_frame_count()
            for f in [f for f in self._first if f < confirmed]:
                del self._first[f]
            for f in sorted(left):
                if _is_older(f, frame):
                    self._first.pop(f, None)
                    if self.count and f >= 0 and f % self.interval == 0:
                        self._retained.append(f)
                        del self._retained[:-self.count]
            snap = self._snapshot(frame)
            self._first.setdefault(frame, snap)
            self._latest[frame] = snap
        return out


def _inputs_spawn(rng, rate: int) -> int:
    return int(rng.integers(0, 16)) | (capi.BGR_INPUT_SPAWN if rate and rng.random() < 0.5 else 0)


class CheckFailed(AssertionError):
    pass


class Interleaving:
    """One configuration and seed.  ``new_engine(role, max_entities, flags, env, fps=, order_base=)`` makes the engine
    ("engine") and its twin ("twin"); the oracle is made here."""

    def __init__(self, cfg: Config, seed: int, new_engine, stamp_first: Optional[int] = None):
        self.cfg, self.seed = cfg, seed
        self.rng = np.random.default_rng(7919 * seed + sum(map(ord, cfg.name)))
        self.world = cfg.world(self.rng)
        w = self.world
        self.growable = bool(cfg.flags & capi.BGR_CFG_GROWABLE)
        self.capture = bool(cfg.flags & capi.BGR_CFG_DESYNC_CAPTURE)
        self.twin_cap = w.n + cfg.grow_margin
        eng_cap = w.n + 8 if self.growable else self.twin_cap
        env = dict(cfg.env)
        if cfg.stamped and stamp_first is None:   # a few launches below the rollover: it happens mid-sequence
            stamp_first = STAMP_LIMIT - int(self.rng.integers(20, 100))
        self.stamp_next = stamp_first
        if stamp_first is not None:
            env["BGR_TEST_STAMP_FIRST"] = str(stamp_first)
        world_cfg = dict(fps=cfg.fps, order_base=cfg.order_base)
        self.eng = new_engine("engine", eng_cap, cfg.flags, env, **world_cfg)
        self.twin = new_engine("twin", self.twin_cap, cfg.flags & ~capi.BGR_CFG_GROWABLE, {**cfg.env, **TWIN_ENV}, **world_cfg)
        self.orc = FlagsOracle(max_entities=self.twin_cap, max_depth=9, **world_cfg)
        for x in (self.eng, self.twin, self.orc):
            w.register(x, cfg.retain)
            x.set_depth(8)   # a ring of at most 8 frames fits max_depth = 9 (twice that with desync capture)
        self.cols = list(range(len(w.sizes)))
        self.feeds: List[Tuple[int, int, FeedModel, Replica]] = []   # (engine feed, twin feed, model, replica)
        for k in range(len(w.feed_fields) and 2):
            fields = w.feed_fields if k == 0 else w.feed_fields[:1]
            fe, ft = self.eng.feed_create(fields), self.twin.feed_create(fields)
            self.feeds.append((fe, ft, FeedModel(fields, self.twin_cap), Replica(len(fields), [f[2] for f in fields], self.twin_cap)))
        self.pending: List[Tuple[List[Tuple[int, int]], List[Request]]] = []   # (oracle's checksums, requests) per submit
        self.deferred_tail: Optional[int] = None   # trailing Advances of the engine's deferred live image, if any
        self.max_rows = w.n
        self.log: List[str] = []
        self.tag = ""                      # prefix of this world's log lines (a Fleet member's index)
        self.step = -1
        self.between_submits: Optional[Callable[[], None]] = None   # a Fleet's batched step, run between queued submits
        self.last_way: Optional[str] = None   # "solo" / "batched": how the last vector ran
        self.tally: Counter = Counter()
        self.digests_left = cfg.digests
        self.last_cap = self.eng.capacity()[0]
        self.tally["stamp_rollovers"] = 0
        self.witnesses, self.retained = set(), set()
        # stamped engines: the launch trace's word [3] counts the active-plane units each vector stored
        self.launched = 0                                  # vectors launched since trace_enable (their trace rows)
        self.plain_launches: List[Tuple[int, int]] = []    # (trace row, units a Save and live write of every plane store)
        self.rollover_launch: Optional[Tuple[int, int, int, bool]] = None   # (trace row, all units, Saves' units, exact)
        self.rollover_pending = False   # the range rolled over at a materialisation: the next vector is checked
        self.was_stamped = None                            # the last vector ran with stamps (None: none yet)
        if cfg.stamped:
            self.eng.trace_enable(TRACE_CAP)

    # ------------------------------------------------------------------ failure context
    def note(self, text: str) -> None:
        self.log.append(f"{self.step}: {self.tag}{text}")

    def fail(self, what: str) -> None:
        raise CheckFailed(what)

    def check(self, cond: bool, what: str) -> None:
        if not cond:
            self.fail(what)

    def run(self, steps: Optional[int] = None) -> Counter:
        steps = self.cfg.steps if steps is None else steps
        for self.step in range(steps + 1):
            try:
                if self.step == steps:
                    self.note("final: full comparison")
                    self.compare_everything()
                else:
                    self.one_step()
                    self.compare_host_state()
            except Exception as ex:
                tail = "\n".join("  " + a for a in self.log)
                raise CheckFailed(f"configuration {self.cfg.name} seed {self.seed} step {self.step}: "
                                  f"{type(ex).__name__}: {ex}\naction log:\n{tail}") from ex
        return self.tally

    def close(self) -> None:
        for x in (self.eng, self.twin, self.orc):
            x.close()

    # ------------------------------------------------------------------ the generator
    def one_step(self) -> None:
        if self.rollover_due():   # the launch the stamp range rolls over at is a plain tick (pick_vector)
            return self.act_vector()
        r = self.rng.random()
        actions = [(0.30, self.act_vector), (0.14, self.act_queued), (0.22, self.act_host_write), (0.22, self.act_read),
                   (0.07, self.act_frame_state), (0.05, self.act_vector_long)]
        acc = 0.0
        for p, fn in actions:
            acc += p
            if r < acc:
                return fn()
        return self.act_vector()

    def frame(self) -> int:
        return self.orc.rollback_frame_count()

    def room(self) -> int:
        """Rows the sequence may still add (the twin's capacity, every snapshot's rows included)."""
        return self.twin_cap - self.max_rows - 8

    def rollover_due(self) -> bool:
        return self.rollover_pending or bool(self.cfg.stamped and self.stamp_next is not None and self.stamp_next > STAMP_LIMIT)

    def pick_vector(self, shape: str) -> Tuple[str, tuple, List[Request]]:
        """``make_vector(shape)``, except that the launch the stamp range rolls over at is a plain tick: its stores are
        then known (every active plane of its Save and of the live write, the table having just been cleared)."""
        if self.rollover_due():
            # with a deferred live image pending, resume from its base slot: a plain tick could find the slot released
            # by a confirmation and materialise the image first, in an internal launch that the trace does not record
            shape = "plain" if self.deferred_tail is None else "resume"
        return (shape,) + self.make_vector(shape)

    def make_vector(self, shape: str) -> Tuple[tuple, List[Request]]:
        """A valid request vector of ``shape`` from the oracle's state; spawn inputs only while the rows fit."""
        rng, frames, f = self.rng, self.orc.snapshot_frames(), self.frame()
        rate = self.world.spawn_rate
        spawn_ok = rate and self.room() > rate * MAX_REQUESTS
        inp = lambda: [_inputs_spawn(rng, rate if spawn_ok else 0)]
        if shape == "synctest":
            mp = int(rng.integers(2, 9))
            d = int(rng.integers(1, mp))
            if f > d and f - d not in frames:
                d = next((k for k in range(1, mp) if f - k in frames), 0)
                if d == 0:
                    return NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, inp())]
            s = SyncTestSession(1, d, mp)
            s.current_frame = f
            s.add_local_input(0, inp()[0])
            return s.info(), s.advance_frame()
        if shape == "p2p":
            s = P2PTraceSession(2, int(rng.integers(2, 9)), input_delay=0, seed=int(rng.integers(1 << 30)),
                                p_clean=float(rng.choice([0.3, 0.7])))
            s.current_frame = f
            s.add_local_input(0, inp()[0]); s.add_local_input(1, int(rng.integers(0, 16)))
            reqs = s.advance_frame()
            if reqs[0].kind == LOAD and reqs[0].frame not in frames:
                return NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, inp())]
            return s.info(), reqs
        near = [g for g in frames if 2 * (f - g) + 2 <= MAX_REQUESTS]   # catch-up runs leave old frames far behind
        if shape in ("rollback", "resume") and near:
            g = f - self.deferred_tail if shape == "resume" else int(rng.choice(near))
            reqs, k = [Request(LOAD, g)], g
            while k < f:
                if k > g:
                    reqs.append(Request(SAVE, k))
                reqs.append(Request(ADVANCE, 0, inp())); k += 1
            return NOSESS, reqs + [Request(SAVE, k), Request(ADVANCE, 0, inp())]
        if shape == "catchup":
            return NOSESS, [Request(ADVANCE, 0, inp()) for _ in range(int(rng.integers(1, 4)))]
        if shape == "long":    # 70..80 requests: a Load and Save / Advance pairs, or Advances only
            n = int(rng.integers(70, MAX_REQUESTS + 1))
            if frames and rng.random() < 0.5:
                g = int(rng.choice(frames))
                reqs, k = [Request(LOAD, g)], g
                while len(reqs) < n - 2 and sum(q.kind == SAVE for q in reqs) < MAX_SAVES - 1:
                    reqs.append(Request(ADVANCE, 0, inp())); k += 1
                    if len(reqs) < n - 2:
                        reqs.append(Request(SAVE, k))
                if reqs[-1].kind != SAVE:
                    reqs.append(Request(SAVE, k))
                return NOSESS, reqs + [Request(ADVANCE, 0, inp())]
            return NOSESS, [Request(ADVANCE, 0, inp()) for _ in range(n)]
        return NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, inp())]

    def random_shape(self) -> str:
        return str(self.rng.choice(["synctest", "p2p", "p2p", "rollback", "catchup", "plain"]))

    # ------------------------------------------------------------------ request vectors
    def _oracle_vector(self, info, reqs) -> List[Tuple[int, int]]:
        out = self.orc.handle_requests(info, reqs)
        self.max_rows = max(self.max_rows, self.orc.row_count())
        return out

    def _kernel_after(self, reqs, launches_before: int, rows_before: int, batched: bool = False) -> None:
        """Tally of one launched vector (last_kernel, launch_count) and the content-stamp mirror.  ``batched``: the
        vector ran in a world batch's call (Fleet)."""
        k = self.eng.last_kernel()
        row = self.launched
        self.launched += 1
        if self.cfg.kind is not None:
            self.check(k.kind == self.cfg.kind, f"the vector ran {k.kind}, not {self.cfg.kind}")
        way = "batched" if batched else "solo"
        if self.last_way is not None and self.last_way != way:
            self.tally[f"{way}_after_{self.last_way}"] += 1
        self.last_way = way
        self.tally[f"{way}_{k.kind}"] += 1
        extra = self.eng.launch_count() - launches_before - 1    # a materialisation runs before the vector
        if extra > 0 and k.kind in ("bundle", "generic_interpreter", "generic_nvrtc"):   # one launch per fused vector
            self.tally["materialisations"] += extra
            if self._stamp_launch(1 + (self.deferred_tail or 0)):
                self.rollover_pending = True
        n_ops = len(reqs) + ((1 + (self.deferred_tail or 0)) if k.from_deferred else 0)
        self.tally["from_deferred"] += k.from_deferred
        self.tally["deferred"] += k.deferred_live
        if self.cfg.stamped and k.kind == "bundle":
            self.check(k.stable_planes, "a launch of a stamped configuration ran without stamps")
        if k.kind == "bundle":   # a change of sides clears the whole stamp table (stamps_stale)
            if self.was_stamped is False and k.stable_planes:
                self.tally["stale_table_clears"] += 1
            self.was_stamped = k.stable_planes
        if k.stable_planes:
            self.tally["stamped_launches"] += 1
            rolled = self._stamp_launch(n_ops)
            # a plain tick, or the vector at the rollover (pick_vector): its Saves go to distinct slots, so with every
            # stamp unknown each of them, and the live write unless deferred, stores every active plane of every segment
            first = rolled or self.rollover_pending
            if first or (len(reqs) == 2 and reqs[0].kind == SAVE and reqs[1].kind == ADVANCE):
                seg_units = UNITS_PER_SEGMENT * (TILE // SEGMENT) * max(1, -(-max(rows_before, self.orc.row_count()) // TILE))
                n_saves = sum(q.kind == SAVE for q in reqs)
                full = seg_units * (n_saves + (0 if k.deferred_live else 1))
                if first:
                    # rolled over at a materialisation before it: image 0 holds fresh stamps, the slots still none, so
                    # only its Saves are known to store everything
                    self.rollover_launch = (row, full, seg_units * n_saves, rolled)
                    self.rollover_pending = False
                else:
                    self.plain_launches.append((row, full))
        tail = 0
        while tail < len(reqs) and reqs[len(reqs) - 1 - tail].kind == ADVANCE:
            tail += 1
        self.deferred_tail = tail if k.deferred_live else None

    def _stamp_launch(self, n_ops: int) -> bool:
        """run_fused's stamp range, restated: a stamped launch takes n_ops + 1 stamps, and the table is cleared and the
        range restarts at 1 when the next stamp is past STAMP_LIMIT.  True: this launch rolled over.  The restatement
        only predicts where; check_rollover reads from the engine's launch trace that the table was cleared there."""
        if self.stamp_next is None or not self.cfg.stamped:
            return False
        rolled = self.stamp_next > STAMP_LIMIT
        if rolled:
            self.tally["stamp_rollovers"] += 1
            self.log[-1] += "  [stamp rollover]"
            self.stamp_next = 1
        self.stamp_next += n_ops + 1
        return rolled

    def check_rollover(self) -> None:
        """From the launch trace (word [3]: 64-byte active-plane units stored): the vector the stamp range rolled over at
        stored every active plane of its Saves and of its live write (every stamp had just been cleared to unknown), and
        some other plain tick of the run stored fewer than all of them (stamps let it skip planes that did not change,
        so storing everything is not what every launch does).  The rollover comes a few dozen launches into the run,
        and most plain ticks right after a host write store everything too, so the skipping tick may come after it."""
        self.check(self.rollover_launch is not None, "no traced plain tick at the stamp rollover")
        tr = self.eng.trace_read(TRACE_CAP)
        stored = [int(x) for x in tr[:, 3]]
        row, full, saves, exact = self.rollover_launch
        self.check(row < len(stored), f"the rollover vector (trace row {row}) is past the trace ({len(stored)} rows)")
        if exact:
            self.check(stored[row] == full, f"the vector at the stamp rollover stored {stored[row]} units, not all {full}: "
                                            f"stamps from before the rollover survived it")
        else:
            self.check(saves <= stored[row] <= full, f"the first vector after the stamp rollover stored {stored[row]} units, "
                                                     f"not its Saves' {saves} at least: stamps from before it survived")
        fewer = [r for r, f in self.plain_launches if stored[r] < f]
        self.check(bool(fewer), "no plain tick skipped a plane: the trace shows no stamp at work")
        self.tally["rollover_verified"] += 1

    def _materialised_by(self, fn, *a):
        """Calls an entry point that launches nothing of its own but materialises a deferred live image."""
        before = self.eng.launch_count()
        out = fn(*a)
        extra = self.eng.launch_count() - before
        if extra:
            self.tally["materialisations"] += extra
            self.rollover_pending |= self._stamp_launch(1 + (self.deferred_tail or 0))
        self.deferred_tail = None
        return out

    def _touch(self) -> None:
        """An entry point that reads or writes image 0 materialised the deferred image (with the extra launch the
        materialisation counts, which the entry point's own launches hide): the mirror of the stamp range follows."""
        if self.deferred_tail is not None:
            self.tally["materialisations_hidden"] += 1
            self.rollover_pending |= self._stamp_launch(1 + (self.deferred_tail or 0))
        self.deferred_tail = None

    def run_vector(self, info, reqs, label: str) -> None:
        self.note(f"{label}: handle_requests {list(reqs)} session {info}")
        rows_before = self.orc.row_count()
        expect = self._oracle_vector(info, reqs)
        before = self.eng.launch_count()
        got = self.eng.handle_requests(info, reqs)
        self.check(got == expect, f"checksums {got} != oracle {expect}")
        self.check(self.twin.handle_requests(info, reqs) == expect, "the twin's checksums differ from the oracle's")
        self._kernel_after(reqs, before, rows_before)
        self.tally["vectors"] += 1
        self.tally["vectors_" + label] += 1

    def act_vector(self) -> None:
        if self.rng.random() < 0.06 and not self.rollover_due():
            return self.act_invalid_rollback()
        shape, info, reqs = self.pick_vector(self.random_shape())
        self.run_vector(info, reqs, shape)

    def act_vector_long(self) -> None:
        shape, info, reqs = self.pick_vector("long")
        self.run_vector(info, reqs, shape)

    def act_invalid_rollback(self, queued: bool = False) -> None:
        f = self.frame()
        self.note(f"invalid rollback Load({f + 1000}){' (submit)' if queued else ''}")
        before = (self.eng.snapshot_frames(), self.eng.rollback_frame_count(), self.eng.row_count(), self.eng.launch_count())
        try:
            (self.eng.submit_requests if queued else self.eng.handle_requests)(NOSESS, [Request(LOAD, f + 1000)])
        except BgrError as ex:
            self.check(ex.status == capi.BGR_ERR_NO_SNAPSHOT, f"invalid rollback returned {ex.status}")
        else:
            self.fail("an invalid rollback was accepted")
        after = (self.eng.snapshot_frames(), self.eng.rollback_frame_count(), self.eng.row_count(), self.eng.launch_count())
        self.check(after == before, f"an invalid rollback changed {before} to {after}")
        self.tally["invalid_rollbacks"] += 1

    def act_queued(self) -> None:
        """1..8 submits without a collect in between, reads / feed reports / host writes between them, then collects in
        random chunks; the calls that must refuse while vectors are pending are tried."""
        k = int(self.rng.integers(1, MAX_QUEUED + 1))
        self.note(f"queue of {k}")
        chained = False   # the previous launch is a submit still in flight, with nothing that drained in between
        for i in range(k):
            shape, info, reqs = self.pick_vector(self.random_shape())
            self.note(f"  submit {shape} {list(reqs)} session {info}")
            rows_before = self.orc.row_count()
            expect = self._oracle_vector(info, reqs)
            before = self.eng.launch_count()
            self.eng.submit_requests(info, reqs)
            self.check(self.twin.handle_requests(info, reqs) == expect, "the twin's checksums differ from the oracle's")
            self.pending.append((expect, reqs))
            self._kernel_after(reqs, before, rows_before)
            self.tally["vectors"] += 1
            self.tally["vectors_queued"] += 1
            self.tally["max_queue_depth"] = max(self.tally["max_queue_depth"], len(self.pending))
            if len(self.pending) >= 4:
                self.tally["queue_depth_4"] += 1
            # the vector's own spawns took the rows across a tile boundary behind an overlapping launch: run_fused
            # drains the stream before it (its tile range differs from the previous launch's)
            rows = self.orc.row_count()
            if chained and rows > rows_before and -(-rows // TILE) != -(-rows_before // TILE):
                self.tally["queued_tile_crossings"] += 1
            chained = True
            if i < k - 1 and self.between_submits is not None and self.rng.random() < 0.3:
                self.note("  (other worlds' batched call, this world's submits in flight on the shared stream)")
                self.between_submits()
                chained = False
            if i < k - 1 and not self.rollover_due():   # nothing but a plain tick may launch at the rollover
                r = self.rng.random()
                chained = r >= 0.65
                if r < 0.2:
                    self.try_refused()
                elif r < 0.3:
                    self.act_invalid_rollback(queued=True)
                elif r < 0.45:
                    self.act_feed_report()
                elif r < 0.55:
                    self.act_read()
                elif r < 0.65:
                    self.act_host_write()
        while self.pending:
            n = int(self.rng.integers(1, len(self.pending) + 1))
            self.note(f"  collect {n} of {len(self.pending)}")
            for _ in range(n):
                expect, reqs = self.pending.pop(0)
                got = self.eng.collect()
                self.check(got == expect, f"collected checksums {got} != oracle {expect} for {list(reqs)}")
            if self.pending and self.rng.random() < 0.4 and not self.rollover_due():
                self.act_read() if self.rng.random() < 0.5 else self.act_feed_report()

    def try_refused(self) -> None:
        self.note("  handle_requests / reset_session with vectors pending: refused")
        before = (self.eng.snapshot_frames(), self.eng.rollback_frame_count(), self.eng.confirmed_frame_count())
        for call in (lambda: self.eng.handle_requests(NOSESS, [Request(SAVE, self.frame()), Request(ADVANCE, 0, [0])]),
                     self.eng.reset_session):
            try:
                call()
            except BgrError as ex:
                self.check(ex.status == capi.BGR_ERR_STATE, f"refusal returned status {ex.status}")
            else:
                self.fail("a call that must refuse with vectors pending was accepted")
        after = (self.eng.snapshot_frames(), self.eng.rollback_frame_count(), self.eng.confirmed_frame_count())
        self.check(after == before, "a refused call changed the frame state")
        self.tally["refusals"] += 1

    # ------------------------------------------------------------------ host writers
    def all3(self, fn) -> None:
        """A host write of image 0 on every world."""
        self._touch()
        for x in (self.eng, self.twin, self.orc):
            fn(x)

    def act_host_write(self) -> None:
        w, rng, rows = self.world, self.rng, self.orc.row_count()
        opts = ["band", "band", "despawn", "presence"] + (["spawn"] if self.cfg.order_base == 0 else [])
        if w.spawn_rate:
            opts.append("startup")
        if self.growable:
            opts.append("reserve")
        what = str(rng.choice(opts))
        alive = np.flatnonzero(self.orc.read_alive(0, rows)) if rows else np.zeros(0, int)
        if what == "band" and rows:
            # on the particles schema Transform half the time: its rotation and scale are the passive planes
            c = 0 if w.bundle and rng.random() < 0.5 else int(rng.integers(0, len(w.sizes)))
            # a band across a 64-row segment or a 512-row tile boundary
            edge = int(rng.choice([SEGMENT, TILE])) * int(rng.integers(1, max(2, rows // SEGMENT)))
            edge = min(edge, rows - 1)
            first = max(0, edge - int(rng.integers(1, 80)))
            count = min(rows - first, int(rng.integers(1, 160)))
            vals = self.values(c, count)
            self.note(f"write_component col {c} rows [{first}, {first + count})")
            self.all3(lambda x: x.write_component(c, first, vals))
            self.tally["band_writes"] += 1
        elif what == "despawn" and alive.size:
            r = int(rng.choice(alive))
            self.note(f"despawn {r}")
            self.all3(lambda x: x.despawn(r))
            self.tally["despawns"] += 1
        elif what == "presence" and alive.size and any(w.optional):
            c = int(rng.choice([i for i, o in enumerate(w.optional) if o]))
            for r in rng.choice(alive, size=min(3, alive.size), replace=False):
                r = int(r)
                if self.orc.has_component(c, r, 1)[0]:
                    self.note(f"remove_component col {c} row {r}")
                    self.all3(lambda x: x.remove_component(c, r))
                else:
                    v = self.values(c, 1)[0]
                    self.note(f"insert_component col {c} row {r}")
                    self.all3(lambda x: x.insert_component(c, r, v))
            self.tally["presence_edits"] += 1
        elif what == "spawn" and self.room() > 200:
            # a count that crosses a segment or a tile boundary
            edge = (rows // SEGMENT + 1) * SEGMENT if rng.random() < 0.6 else (rows // TILE + 1) * TILE
            k = max(1, min(self.room() - 100, edge - rows + int(rng.integers(0, 40))))
            vals = [self.values(c, k) for c in range(len(w.sizes))]
            self.note(f"spawn {k} at row {rows} and write every column")
            def sp(x):
                first = x.spawn(k)
                for c in range(len(w.sizes)):
                    x.write_component(c, first, vals[c])
            self.all3(sp)
            self.max_rows = max(self.max_rows, self.orc.row_count())
            self.tally["spawns"] += 1
        elif what == "startup" and self.room() > w.spawn_rate:
            self.note("run_startup_system spawn_particles")
            self.all3(lambda x: x.run_startup_system(capi.BGR_SYS_PARTICLES_SPAWN))
            self.max_rows = max(self.max_rows, self.orc.row_count())
            self.tally["startup_systems"] += 1
        elif what == "reserve":
            target = int(min(self.twin_cap, self.eng.capacity()[0] + rng.integers(1, 3000)))
            self.note(f"reserve {target}")
            self.eng.reserve(target)
            self.twin.reserve(target)
            self.tally["reserves"] += 1
        else:
            self.note(f"(no {what}: nothing to do)")
        self.note_growth()

    def values(self, c: int, count: int) -> np.ndarray:
        """Element bytes for column c: random, and on the particles schema f32 edge values (-0.0, subnormals) in
        Transform / Velocity and ttl values just past 2^32.  Transform's rotation and scale are random too: no system
        writes them, so they are the bundle's passive planes, and only content that differs between images shows a
        passive store that was wrongly skipped."""
        w, rng, size = self.world, self.rng, self.world.sizes[c]
        if w.bundle and c in (0, 1):
            v = rng.uniform(-300, 300, (count, size // 4)).astype(np.float32)
            edge = np.array([-0.0, 1e-45, -1e-45, 1.1754942e-38, -5e-40, 0.0], np.float32)
            m = rng.random(v.shape) < 0.3
            v[m] = rng.choice(edge, size=int(m.sum()))
            return v.view(np.uint8).reshape(count, size)
        if w.bundle and c == 2:
            t = rng.integers(1, 30, count).astype(np.uint64)
            t[rng.random(count) < 0.3] += np.uint64(1 << 32) - np.uint64(3)
            return t.view(np.uint8).reshape(count, 8)
        out = rng.integers(0, 256, (count, size), dtype=np.uint8)
        if size % 4 == 0:
            out.view(np.uint32)[:] = rng.integers(20, 300, (count, size // 4), dtype=np.uint32)
        return out

    def note_growth(self) -> None:
        cap = self.eng.capacity()[0]
        if cap != self.last_cap:
            self.tally["growth_steps"] += 1
            self.last_cap = cap

    def act_frame_state(self) -> None:
        rng = self.rng
        if rng.random() < 0.6:
            d = int(rng.integers(2, 9))
            self.note(f"set_depth {d}")
            self._materialised_by(self.eng.set_depth, d)
            self.twin.set_depth(d); self.orc.set_depth(d)
            self.tally["set_depth"] += 1
        else:
            # back to the frame the session had: FlagsOracle restates Time<GgrsTime> at a Save of frame f as f / fps,
            # which a frame count moved without an Advance would break
            f = self.frame()
            self.note(f"reset_session, set_rollback_frame_count {f}")
            self._materialised_by(self.eng.reset_session)
            for x in (self.eng, self.twin, self.orc):
                if x is not self.eng:
                    x.reset_session()
                x.set_rollback_frame_count(f)
            self.tally["reset_sessions"] += 1

    # ------------------------------------------------------------------ reads
    def act_read(self) -> None:
        opts = ["live", "peek", "download", "feed"]
        if self.capture:
            opts += ["capture", "capture"]
        if self.cfg.retain:
            opts += ["retained", "retained"]
        what = str(self.rng.choice(opts))
        {"live": self.act_read_live, "peek": self.act_peek, "download": self.act_download, "feed": self.act_feed_report,
         "capture": self.act_capture, "retained": self.act_retained}[what]()

    def act_read_live(self) -> None:
        rows = self.orc.row_count()
        first = int(self.rng.integers(0, max(1, rows)))
        count = rows - first if self.rng.random() < 0.5 else min(rows - first, int(self.rng.integers(1, 700)))
        self.note(f"read the live world rows [{first}, {first + count})")
        self._touch()
        self.compare_live(first, count)
        self.check(self.eng.active_count() == self.orc.active_count(), "active_count differs from the oracle's")
        self.tally["live_reads"] += 1

    def compare_live(self, first: int, count: int) -> None:
        if count <= 0:
            return
        alive = self.orc.read_alive(first, count).astype(bool)
        self.check(np.array_equal(self.eng.read_alive(first, count).astype(bool), alive), "alive rows differ from the oracle's")
        for c in self.cols:
            vo, ho = self.orc.read_component_alive(c, first, count)
            he = self.eng.has_component(c, first, count).astype(bool)
            self.check(np.array_equal(he, ho.astype(bool)), f"presence of column {c} differs from the oracle's")
            ve = self.eng.read_component(c, first, count)
            bad = np.flatnonzero((ve[he] != vo[he]).any(axis=1))
            self.check(bad.size == 0, f"column {c} differs from the oracle's on present rows "
                                      f"{(np.flatnonzero(he)[bad] + first)[:8].tolist()}")
            vt = self.twin.read_component(c, first, count)
            bad = np.flatnonzero((ve != vt).any(axis=1))
            self.check(bad.size == 0, f"live bytes of column {c} differ from the twin's on rows {(bad + first)[:8].tolist()}")
            self.check(np.array_equal(he, self.twin.has_component(c, first, count).astype(bool)),
                       f"presence of column {c} differs from the twin's")

    def _snap_rows(self, frame: int, first: bool = False) -> int:
        snap = (self.orc._first if first else self.orc._latest).get(frame)
        return snap["rows"] if snap else 0

    def act_peek(self, frames: Optional[Sequence[int]] = None) -> None:
        frames = self.orc.snapshot_frames() if frames is None else frames
        if not frames:
            return self.note("(no snapshot to peek)")
        # every held frame: a Save whose passive or active store was wrongly skipped shows only in that slot's bytes
        picks = frames if len(frames) <= 2 or self.rng.random() < 0.7 else [int(self.rng.choice(frames))]
        self.note(f"peek {list(picks)}")
        for f in picks:
            rows = self._snap_rows(f)
            for c in self.cols:
                pe, po, pt = self.eng.peek(f, c, 0, rows), self.orc.peek(f, c, 0, rows), self.twin.peek(f, c, 0, rows)
                self.check(pe is not None and po is not None and pt is not None, f"frame {f} is not held")
                pres = po[1].astype(bool)
                self.check(np.array_equal(pe[1].astype(bool), pres), f"presence of column {c} in frame {f} differs from the oracle's")
                bad = np.flatnonzero((pe[0][pres] != po[0][pres]).any(axis=1))
                self.check(bad.size == 0, f"column {c} of frame {f} differs from the oracle's on rows "
                                          f"{np.flatnonzero(pres)[bad][:8].tolist()}")
                bad = np.flatnonzero((pe[0] != pt[0]).any(axis=1))
                self.check(bad.size == 0, f"snapshot bytes of column {c} in frame {f} differ from the twin's on rows {bad[:8].tolist()}")
        self.tally["peeks"] += 1

    def act_download(self) -> None:
        rows = self.orc.row_count()
        if not rows:
            return
        word_cols = [c for c, sz in enumerate(self.world.sizes) if sz >= 4]
        if not word_cols:
            return
        c = int(self.rng.choice(word_cols))
        words = self.world.sizes[c] // 4   # a 4-byte aligned field inside the element's whole words
        off = 4 * int(self.rng.integers(0, words))
        ln = 4 * int(self.rng.integers(1, words - off // 4 + 1))
        first = int(self.rng.integers(0, rows))
        count = rows - first
        self.note(f"download col {c} bytes [{off}, {off + ln}) rows [{first}, {rows})")
        self._touch()
        buf = self.eng.host_alloc(count, ln)
        t = self.eng.download_begin(c, off, ln, first, count, buf)
        self.eng.download_wait(t)
        got = np.array(buf[:count])
        vo, ho = self.orc.read_component_alive(c, first, count)
        pres = ho.astype(bool)
        self.check(np.array_equal(got[pres], vo[pres, off:off + ln]), f"download of column {c} differs from the oracle's")
        self.check(np.array_equal(got, self.twin.read_component(c, first, count)[:, off:off + ln]),
                   f"download of column {c} differs from the twin's live bytes")
        self.tally["downloads"] += 1

    def act_feed_report(self) -> None:
        if not self.feeds:
            return self.note("(no feed)")
        i = int(self.rng.integers(0, len(self.feeds)))
        fe, ft, model, replica = self.feeds[i]
        if self.rng.random() < 0.1:
            self.note(f"feed_reset {i}")
            self.eng.feed_reset(fe)
            model.reset()
            self.feeds[i] = (fe, ft, model, Replica(len(model.fields), [f[2] for f in model.fields], self.twin_cap))
            self.tally["feed_resets"] += 1
            return
        world = world_of(self.orc, [f[0] for f in model.fields])
        n_diff = len(model.differing(world))
        cap = int(self.rng.choice([0, max(0, n_diff - 1 - int(self.rng.integers(0, max(1, n_diff)))), n_diff + 5]))
        self.note(f"feed report {i} cap {cap} ({n_diff} rows differ)")
        self._touch()
        buf = self.eng.feed_alloc(fe, cap)
        recs, info = self.eng.feed_wait(self.eng.feed_begin(fe, buf, cap))
        expect, einfo = model.report(world, cap)
        self.check(tuple(info) == tuple(einfo), f"feed info {info} != model {einfo}")
        self.check(recs.tobytes() == expect.tobytes(), f"feed records differ from the model's "
                                                        f"(rows {recs['row'][:8].tolist()} vs {expect['row'][:8].tolist()})")
        replica.apply(recs)
        if einfo.pending == 0:
            self.check(replica.matches(model, world), "the replica does not match the model after a complete report")
        self.tally["feed_reports"] += 1
        if cap < n_diff:
            self.tally["feed_cap_hit"] += 1

    def act_capture(self, every: bool = False) -> None:
        frames = self.orc.desync_frames()
        self.check(self.eng.desync_frames() == frames, f"desync_frames {self.eng.desync_frames()} != oracle {frames}")
        self.note(f"desync frames {frames}")
        self.tally["capture_reads"] += 1
        for f in (frames if every else frames[:2]):   # the final comparison: every first image
            cap = int(self.rng.choice([3, 64]))
            a, b, t = self.eng.desync_diff(f, cap), self.orc.desync_diff(f, cap), self.twin.desync_diff(f, cap)
            # the oracle does not restate ParticleRng (host_state_differs bit 0): that bit is held to the twin's
            sa, sb = a.summary_tuple(), b.summary_tuple()
            self.check(sa == t.summary_tuple(), f"desync summary of frame {f}: {sa} != the twin's {t.summary_tuple()}")
            self.check(sa[:6] + (sa[6] & ~1,) + sa[7:] == sb[:6] + (sb[6] & ~1,) + sb[7:],
                       f"desync summary of frame {f}: {sa} != oracle {sb}")
            self.check(np.array_equal(a.records, b.records), f"desync records of frame {f} differ from the oracle's")
            self.check(all(a.columns[c] == b.columns[c] for c in self.cols), f"desync columns of frame {f} differ")
            rows = self._snap_rows(f, first=True)
            for c in self.cols:
                pe, po, pt = self.eng.peek_first(f, c, 0, rows), self.orc.peek_first(f, c, 0, rows), self.twin.peek_first(f, c, 0, rows)
                pres = po[1].astype(bool)
                self.check(np.array_equal(pe[1].astype(bool), pres), f"first image presence of column {c} in frame {f}")
                self.check(np.array_equal(pe[0][pres], po[0][pres]), f"first image of column {c} in frame {f} differs from the oracle's")
                self.check(np.array_equal(pe[0], pt[0]), f"first image bytes of column {c} in frame {f} differ from the twin's")
            self.tally["desync_diffs"] += 1
        if any(self.orc._first.get(f) is not None for f in frames):
            self.tally["witness_frames"] += 1

    def act_retained(self) -> None:
        ret = self.orc.retained_frames()
        self.check(self.eng.retained_frames() == ret, f"retained_frames {self.eng.retained_frames()} != oracle {ret}")
        self.note(f"retained frames {ret}")
        held = self.orc.snapshot_frames() + ret
        if not held:
            return
        picks = [int(self.rng.choice(held))]
        if ret and self.rng.random() < 0.5:
            picks = [ret[0]]
        for f in picks:
            if self.digests_left > 0:
                self.digests_left -= 1
                h, words = self.eng.frame_digest(f)
                rows, active, expect = self.orc.frame_digest(f)
                self.check((h.frame, h.rows, h.active, h.n_blocks) == (f, rows, active, -(-rows // BLOCK)),
                           f"digest header of frame {f}: {(h.frame, h.rows, h.active, h.n_blocks)} != oracle {(f, rows, active)}")
                self.check(np.array_equal(words, expect), f"digest words of frame {f} differ from the oracle's")
                self.tally["digests"] += 1
            n_blocks = -(-self._image_rows(f) // BLOCK)
            blocks = sorted(set(int(b) for b in self.rng.integers(0, max(1, n_blocks), 3))) if n_blocks else []
            if blocks:
                blob, tblob = self.eng.export_blocks(f, blocks), self.twin.export_blocks(f, blocks)
                self.check(blob == tblob, f"export blob of frame {f} blocks {blocks} differs from the twin's")
                rep = self.twin.diff_remote(f, blob)
                self.check(rep is not None and rep.rows_differing == 0 and len(rep.records) == 0,
                           f"diff_remote of the engine's blob of frame {f} on the twin reports differences")
                self.tally["exports"] += 1
        if ret:
            self.tally["retained_reads"] += 1

    def _image_rows(self, f: int) -> int:
        snap = self.orc.image(f)
        return snap["rows"] if snap else 0

    # ------------------------------------------------------------------ every step / the end
    def compare_host_state(self) -> None:
        e, o, t = self.eng, self.orc, self.twin
        self.check(e.rollback_frame_count() == o.rollback_frame_count(), "rollback_frame_count differs from the oracle's")
        self.check(e.confirmed_frame_count() == o.confirmed_frame_count(), "confirmed_frame_count differs from the oracle's")
        self.check(e.snapshot_frames() == o.snapshot_frames(), f"snapshot_frames {e.snapshot_frames()} != oracle {o.snapshot_frames()}")
        self.check(e.row_count() == o.row_count() == t.row_count(), "row_count differs from the oracle's")
        if self.cfg.retain:
            self.check(e.retained_frames() == o.retained_frames(), "retained_frames differs from the oracle's")
        self.note_growth()
        # a witness (first image) or a retained frame that is released hands its slot out again
        witnesses, retained = set(self.orc._first), set(self.orc.retained_frames())
        self.tally["witnesses_released"] += len(self.witnesses - witnesses) if self.capture else 0
        self.tally["retained_released"] += len(self.retained - retained)
        self.witnesses, self.retained = witnesses, retained

    def compare_everything(self) -> None:
        if self.cfg.stamped:
            self.check_rollover()
        self._touch()
        self.compare_live(0, self.orc.row_count())
        self.act_peek(self.orc.snapshot_frames())
        if self.capture:
            self.act_capture(every=True)
        if self.cfg.retain:
            self.act_retained()
        for i in range(len(self.feeds)):
            fe, ft, model, replica = self.feeds[i]
            world = world_of(self.orc, [f[0] for f in model.fields])
            buf = self.eng.feed_alloc(fe, self.twin_cap)
            recs, info = self.eng.feed_wait(self.eng.feed_begin(fe, buf, self.twin_cap))
            expect, einfo = model.report(world, self.twin_cap)
            self.check(tuple(info) == tuple(einfo) and recs.tobytes() == expect.tobytes(), "the final feed report differs")
            replica.apply(recs)
            self.check(replica.matches(model, world), "the replica does not match the model at the end")


# ---------------------------------------------------------------------------------------------------- world batches
@dataclass
class FleetConfig:
    """A world batch's configuration.  ``registration(rng)`` draws the registration once per fleet and returns
    ``make(rng, member)``, the maker of each member's World (its rows and data, drawn from the member's own generator).  ``members``: one Config
    per member for its flags, retention, fps, order_base and grow margin (their name, world, env and kind are set here)."""
    name: str
    registration: Callable[[np.random.Generator], Callable[[np.random.Generator, int], World]]
    members: List[Config]
    env: Dict[str, str] = field(default_factory=dict)
    steps: int = 80


class Fleet:
    """K ``Interleaving`` members whose engines share one stream and one ``EngineBatch``, each with its own oracle, twin
    and feed models.  A step is a batched call over a random non-empty subset of the members in random order (each
    member draws its own vector), sometimes with one world's vector refused, or one member's ordinary action
    (``Interleaving.one_step``: its solo and queued vectors, host writes, reads and feeds land between batched calls).
    While a member holds un-collected submits, a batched call over the other members may run on the shared stream.

    ``new_engine(member, role, max_entities, flags, env, fps=, order_base=)`` makes member ``member``'s engine (on the
    shared stream) and twin; ``new_batch(engines)`` makes the batch."""

    def __init__(self, fcfg: FleetConfig, seed: int, new_engine, new_batch):
        self.fcfg, self.seed = fcfg, seed
        self.rng = np.random.default_rng(104729 * seed + sum(map(ord, fcfg.name)))
        make = fcfg.registration(self.rng)
        self.log: List[str] = []
        self.step = -1
        self.tally: Counter = Counter()
        self.members: List[Interleaving] = []
        self.batch = None
        try:
            for i, mc in enumerate(fcfg.members):
                cfg = Config(**{**mc.__dict__, "name": f"{fcfg.name}/{i}", "world": lambda rng, _i=i: make(rng, _i), "env": {**fcfg.env, **mc.env},
                                "kind": None, "stamped": False})
                m = Interleaving(cfg, seed, lambda role, *a, _i=i, **kw: new_engine(_i, role, *a, **kw))
                m.log, m.tag = self.log, f"w{i} "
                m.between_submits = lambda _i=i: self.act_batch(exclude=_i)
                self.members.append(m)
            self.batch = new_batch([m.eng for m in self.members])
        except BaseException:
            self.close()
            raise
        self.specialised = self.batch.specialised()

    def note(self, text: str) -> None:
        self.log.append(f"{self.step}: {text}")

    def totals(self) -> Counter:
        """The fleet's tally and every member's, added up."""
        t = Counter(self.tally)
        for m in self.members:
            t.update(m.tally)
        return t

    def run(self, steps: Optional[int] = None) -> Counter:
        steps = self.fcfg.steps if steps is None else steps
        for self.step in range(steps + 1):
            for m in self.members:
                m.step = self.step
            try:
                if self.step == steps:
                    self.note("final: full comparison of every member")
                    for m in self.members:
                        m.compare_everything()
                else:
                    self.one_step()
                    for m in self.members:
                        m.compare_host_state()
            except Exception as ex:
                tail = "\n".join("  " + a for a in self.log)
                raise CheckFailed(f"fleet {self.fcfg.name} seed {self.seed} step {self.step}: "
                                  f"{type(ex).__name__}: {ex}\naction log:\n{tail}") from ex
        return self.totals()

    def close(self) -> None:
        if self.batch is not None:
            self.batch.close()   # before any of its engines
            self.batch = None
        for m in self.members:
            m.close()

    def one_step(self) -> None:
        if self.rng.random() < 0.45:
            return self.act_batch()
        self.members[int(self.rng.integers(0, len(self.members)))].one_step()

    def act_batch(self, exclude: Optional[int] = None) -> None:
        """A batched call over a random subset (``exclude``: a member with submits in flight, never listed)."""
        avail = [i for i in range(len(self.members)) if i != exclude]
        if not avail:
            return
        k = int(self.rng.integers(1, len(avail) + 1))
        worlds = [avail[int(j)] for j in self.rng.permutation(len(avail))[:k]]
        calls = []
        for i in worlds:
            m = self.members[i]
            shape, info, reqs = m.pick_vector(m.random_shape())
            calls.append((i, shape, info, reqs))
        if self.rng.random() < 0.08:
            return self.act_batch_refused(calls, exclude)
        self.note(f"batched call over worlds {worlds}" + (f" (w{exclude} has submits in flight)" if exclude is not None else ""))
        expected = []
        for i, shape, info, reqs in calls:   # the oracle of every listed world, before the call
            m = self.members[i]
            m.note(f"batched {shape}: {list(reqs)} session {info}")
            rows_before = m.orc.row_count()
            expected.append((m._oracle_vector(info, reqs), m.eng.launch_count(), rows_before))
        res = self.batch.handle_requests([(i, info, reqs) for i, _, info, reqs in calls])
        self.check(len(res) == len(calls), f"{len(res)} results for {len(calls)} worlds")
        for (i, shape, info, reqs), (status, got), (expect, before, rows_before) in zip(calls, res, expected):
            m = self.members[i]
            m.check(status == capi.BGR_OK, f"world {i}: batched status {status}")
            m.check(got == expect, f"world {i}: batched checksums {got} != oracle {expect}")
            lk = m.eng.last_kernel()
            if self.specialised:
                m.check(lk.batched and lk.kind == "generic_nvrtc", f"world {i}: a batched vector ran {lk}")
            else:
                m.check(not lk.batched, f"world {i}: an unspecialised batch reported a batched launch")
            m.check(m.twin.handle_requests(info, reqs) == expect, f"world {i}: the twin's checksums differ from the oracle's")
            m._kernel_after(reqs, before, rows_before, batched=True)
            m.tally["vectors"] += 1
            m.tally["vectors_batched"] += 1
        self.tally["batched_calls"] += 1
        self.tally["batched_worlds"] += len(calls)
        if exclude is not None:
            self.tally["batch_with_queued_member"] += 1

    def act_batch_refused(self, calls, exclude: Optional[int]) -> None:
        """One listed world loads a frame it does not hold: the call is refused, names that world and changes nothing
        anywhere (no oracle is advanced)."""
        j = int(self.rng.integers(0, len(calls)))
        bad = calls[j][0]
        f = self.members[bad].frame()
        calls[j] = (bad, "invalid", NOSESS, [Request(LOAD, f + 1000)])
        self.note(f"batched call over worlds {[c[0] for c in calls]}, w{bad} loads frame {f + 1000}: refused")
        state = lambda: [(m.eng.launch_count(), m.eng.snapshot_frames(), m.eng.rollback_frame_count(), m.eng.row_count(),
                          m.eng.confirmed_frame_count()) for m in self.members]
        before = state()
        try:
            self.batch.handle_requests([(i, info, reqs) for i, _, info, reqs in calls])
        except BgrError as ex:
            self.check(ex.status == capi.BGR_ERR_NO_SNAPSHOT, f"the refused batched call returned {ex.status}")
            self.check(str(ex).startswith(f"world {bad}: "), f"the refusal does not name world {bad}: {ex}")
        else:
            self.fail(f"a batched call in which world {bad} loads an unsaved frame was accepted")
        after = state()
        self.check(after == before, f"a refused batched call changed {before} to {after}")
        for m in self.members:
            m.compare_host_state()
        self.tally["batch_refusals"] += 1
        if exclude is not None:
            self.tally["batch_with_queued_member"] += 1

    def check(self, cond: bool, what: str) -> None:
        if not cond:
            self.fail(what)

    def fail(self, what: str) -> None:
        raise CheckFailed(what)
