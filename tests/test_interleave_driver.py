"""CPU test of the interleaving driver (tests/interleave_driver.py): it drives a fake engine made of the oracle itself
(queued submit / collect, FeedModel feeds, digests and exports from the oracle, a stub last_kernel), so every
action it generates must be accepted, the same seed must give the same action log, and a fake that corrupts one
observation at a chosen step (one byte of one read, one checksum bit, one feed record, one checkpoint blob byte, one
replay checksum bit, one byte of a restored world) must fail the run at that step.  Checkpoints, restores and replays
are drawn only by configurations that turn them on, so the action log of every existing seed stays what it was.
The same holds for a Fleet of such fakes in a FakeBatch, which runs the listed fakes' vectors one after another."""
import hashlib
import pickle
from types import SimpleNamespace

import numpy as np
import pytest

import checkpoint_codec as cc
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import LastKernel
from bevy_ggrs_b200.session import LOAD
from change_feed_model import FeedModel, world_of
from interleave_driver import CheckFailed, Config, Fleet, FleetConfig, FlagsOracle, Interleaving, World
from oracle_p2p import BLOCK
from schema_util import random_schema


class FakeEngine(FlagsOracle):
    """The Engine surface the driver uses, on the oracle.  ``corrupt`` = (kind, step) flips one observed bit there."""

    def __init__(self, max_entities, flags, growable=False, corrupt=None, fps=60, order_base=0, written=None):
        super().__init__(max_entities=max_entities, max_depth=9, fps=fps, order_base=order_base)
        # every blob the fakes of one run wrote: the stand-in for the engine's digest check of a restored world
        self.written = set() if written is None else written
        self.ticked = False
        self.cap, self.ceiling = max_entities, (1 << 20) if growable else max_entities
        self.queue = []
        self.feeds, self.tickets = [], {}
        self.corrupt, self.driver = corrupt, None

    def _hit(self, kind):
        if self.corrupt and self.driver is not None and self.corrupt == (kind, self.driver.step):
            self.corrupt = None   # one observation only
            return True
        return False

    # capacity
    def capacity(self):
        return self.cap, self.ceiling

    def _grow(self, rows):
        if rows > self.cap:
            if rows > self.ceiling:
                raise BgrError(capi.BGR_ERR_CAPACITY, "capacity")
            self.cap = max(rows, 2 * self.cap)

    def reserve(self, rows):
        self._grow(rows)

    def spawn(self, count):
        if self.order_base and self.ticked:
            raise BgrError(capi.BGR_ERR_UNSUPPORTED, "spawn with order_base != 0")
        self._grow(self.row_count() + count)
        return super().spawn(count)

    # vectors
    def _refusal(self, reqs):
        if self.queue:
            return BgrError(capi.BGR_ERR_STATE, "pending")
        if reqs and reqs[0].kind == LOAD and reqs[0].frame not in self.snapshot_frames():
            return BgrError(capi.BGR_ERR_NO_SNAPSHOT, "Could not rollback")
        return None

    def _run(self, info, reqs, batched=False):
        if reqs and reqs[0].kind == LOAD and reqs[0].frame not in self.snapshot_frames():
            raise BgrError(capi.BGR_ERR_NO_SNAPSHOT, "Could not rollback")
        self.ticked = True
        out = super().handle_requests(info, reqs)
        if batched and out and self._hit("batch_checksum"):
            out[-1] = (out[-1][0], out[-1][1] ^ (1 << 17))
        self._grow(self.row_count())
        if out and self._hit("checksum"):
            out[0] = (out[0][0], out[0][1] ^ 1)
        return out

    def handle_requests(self, info, reqs):
        if self.queue:
            raise BgrError(capi.BGR_ERR_STATE, "pending")
        return self._run(info, reqs)

    def submit_requests(self, info, reqs):
        if len(self.queue) >= 8:
            raise BgrError(capi.BGR_ERR_STATE, "too many")
        self.queue.append(self._run(info, reqs))

    def collect(self):
        return self.queue.pop(0)

    def reset_session(self):
        if self.queue:
            raise BgrError(capi.BGR_ERR_STATE, "pending")
        super().reset_session()

    def last_kernel(self):
        return LastKernel.decode(0)

    def launch_count(self):
        return 0

    # reads
    def read_component(self, col, first, count):
        out = super().read_component(col, first, count)
        if count and self._hit("read"):
            out[0, 0] ^= 1
        return out

    def host_alloc(self, count, ln):
        return np.zeros((count, ln), np.uint8)

    def download_begin(self, col, off, ln, first, count, dst):
        dst[:count] = super().read_component(col, first, count)[:, off:off + ln]
        return 0

    def download_wait(self, ticket):
        pass

    def feed_create(self, fields):
        self.feeds.append(FeedModel(fields, 1 << 16))
        return len(self.feeds) - 1

    def feed_reset(self, feed):
        self.feeds[feed].reset()

    def feed_alloc(self, feed, cap):
        return None

    def feed_begin(self, feed, buf, cap):
        m = self.feeds[feed]
        self.tickets[feed] = m.report(world_of(self, [f[0] for f in m.fields]), cap)
        return feed

    def feed_wait(self, ticket):
        recs, info = self.tickets.pop(ticket)
        if len(recs) and self._hit("feed"):
            recs = recs.copy()
            recs["state"][0] ^= 1
        return recs, info

    # retention
    def frame_digest(self, frame):
        d = super().frame_digest(frame)
        if d is None:
            return None
        rows, active, words = d
        return SimpleNamespace(frame=frame, rows=rows, active=active, n_blocks=-(-rows // BLOCK)), words

    def export_blocks(self, frame, blocks):
        snap = self.image(frame)
        return None if snap is None else pickle.dumps((frame, list(blocks), self.frame_digest(frame)[1][list(blocks)].tobytes()))

    def diff_remote(self, frame, blob):
        f, blocks, words = pickle.loads(blob)
        same = f == frame and self.export_blocks(frame, blocks) == blob
        return SimpleNamespace(rows_differing=0 if same else 1, records=[] if same else [0])

    # checkpoints and replays
    def checkpoint(self, frame):
        blob = self.checkpoint_of(frame, self.order_base, (0, 0, 0, 0))   # the layout fingerprint: order_base alone
        if blob is not None:
            self.written.add(blob)
        if blob is not None and self._hit("blob"):
            blob = blob[:-1] + bytes([blob[-1] ^ 1])
        return blob

    def restore(self, blob):
        if self.queue:
            raise BgrError(capi.BGR_ERR_STATE, "pending")
        try:
            h, planes, mask = cc.decode(blob)
        except cc.CodecError as ex:
            raise BgrError(capi.BGR_ERR_INVALID_ARGUMENT, str(ex))
        absent = np.concatenate([[b] * ((eb + 3) // 4) for b, eb in zip(self.absent_bit, self.elem_bytes)]).astype(np.uint32)
        planes, mask = cc.canonical(planes, mask, h["rows"], absent)
        header = {k: h[k] for k in ("layout", "frame", "rows", "n_columns", "fps", "active", "elapsed_ns", "rng", "digest_root")}
        unused = int(np.bitwise_or.reduce(mask.reshape(-1), initial=0)) & ~(1 | int(np.bitwise_or.reduce(absent, initial=0)))
        if (h["fps"] != self.fps or h["layout"] != self.order_base or unused or cc.encode(planes, mask, **header) != blob
                or blob not in self.written):
            raise BgrError(capi.BGR_ERR_INVALID_ARGUMENT, "corrupt checkpoint")
        self._grow(h["rows"])
        super().restore(blob)
        if self._hit("restore"):   # one byte of one present component of the restored world
            for c in range(len(self.elem_bytes)):
                v, has = self.read_component_alive(c, 0, h["rows"])
                if has.any():
                    r = int(np.flatnonzero(has)[0])
                    v[r, 0] ^= 1
                    self.write_component(c, r, v[r:r + 1])
                    break

    def _replay_refusal(self, inputs):
        if np.asarray(inputs).shape[1] > capi.BGR_MAX_PLAYERS:
            return BgrError(capi.BGR_ERR_INVALID_ARGUMENT, "n_players > BGR_MAX_PLAYERS")
        if self.queue:
            return BgrError(capi.BGR_ERR_STATE, "pending")
        return None

    def replay(self, inputs, k=0):
        err = self._replay_refusal(inputs)
        if err is not None:
            raise err
        rate = self.driver.world.spawn_rate if self.driver is not None else 0
        spawning = int((np.asarray(inputs) & capi.BGR_INPUT_SPAWN).any(axis=1).sum()) if rate else 0
        if self.row_count() + rate * spawning > self.ceiling:
            raise BgrError(capi.BGR_ERR_CAPACITY, "spawns past the capacity")
        out = super().replay(inputs, k)
        self._grow(self.row_count())
        if out and self._hit("replay_checksum"):
            out[0] = (out[0][0], out[0][1] ^ (1 << 5))
        return out


def _generic_world(rng):
    s = random_schema(rng, words=int(rng.integers(4, 14)))
    n = int(rng.integers(500, 1300))
    data = s.values(rng, n)
    strategies = [(capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL) if o else capi.BGR_STRATEGY_CLONE for o in s.optional]
    removes = [(c, int(r)) for c, o in enumerate(s.optional) if o for r in rng.choice(n, 5, replace=False)]
    feed = [(c, 0, min(8, sz)) for c, sz in enumerate(s.sizes) if sz % 4 == 0][:2]
    return World(s.sizes, strategies, [(c, off, ln, 0) for c, off, ln in s.cks],
                 [(k, c, p) for k, c, p in s.systems], data, removes, feed_fields=feed)


FLAGS = [0, capi.BGR_CFG_DESYNC_CAPTURE, "retain", capi.BGR_CFG_GROWABLE, capi.BGR_CFG_GROWABLE | capi.BGR_CFG_DESYNC_CAPTURE]


def _config(flags, steps=40, match=False):
    retain = (2, 4) if flags == "retain" else None
    return Config("fake", _generic_world, flags=0 if flags == "retain" else flags, retain=retain, steps=steps,
                  grow_margin=3000, checkpoints=match, input_replays=match)


def _run(flags, seed, corrupt=None, steps=40, match=False):
    fakes, written = [], set()

    def new_engine(role, cap, fl, env, fps=60, order_base=0):
        f = FakeEngine(cap, fl, growable=bool(fl & capi.BGR_CFG_GROWABLE),
                       corrupt=corrupt if role == "engine" else None, fps=fps, order_base=order_base, written=written)
        fakes.append(f)
        return f
    drv = Interleaving(_config(flags, steps, match), seed, new_engine)
    for f in fakes:
        f.driver = drv
    try:
        drv.run()
    finally:
        drv.close()
    return drv


@pytest.mark.parametrize("flags", FLAGS, ids=str)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_every_generated_action_is_accepted(flags, seed):
    drv = _run(flags, seed)
    t = drv.tally
    assert t["vectors"] > 10 and t["vectors_queued"] > 0 and t["band_writes"] + t["spawns"] + t["despawns"] > 0
    assert t["live_reads"] + t["peeks"] + t["feed_reports"] > 0


def test_the_same_seed_gives_the_same_action_log():
    a, b = _run(capi.BGR_CFG_DESYNC_CAPTURE, 5), _run(capi.BGR_CFG_DESYNC_CAPTURE, 5)
    assert a.log == b.log and len(a.log) > 40
    assert _run(capi.BGR_CFG_DESYNC_CAPTURE, 6).log != a.log


def test_every_action_kind_is_reached_over_a_few_seeds():
    total = {}
    for seed, flags in enumerate(FLAGS):
        for k, v in _run(flags, 10 + seed, steps=60).tally.items():
            total[k] = total.get(k, 0) + v
    for k in ["vectors_synctest", "vectors_p2p", "vectors_rollback", "vectors_catchup", "vectors_long", "vectors_queued",
              "invalid_rollbacks", "refusals", "band_writes", "spawns", "despawns", "presence_edits", "reserves",
              "set_depth", "reset_sessions", "live_reads", "peeks", "downloads", "feed_reports", "feed_cap_hit",
              "capture_reads", "digests", "exports", "queue_depth_4"]:
        assert total.get(k, 0) > 0, k


def _first_step(log, marker):
    for line in log:
        step, text = line.split(": ", 1)
        if marker(text):
            return int(step)
    raise AssertionError("the clean run never reached the observation")


@pytest.mark.parametrize("kind,marker", [
    ("read", lambda t: t.startswith("read the live world") and not t.endswith(", 0)")),
    ("checksum", lambda t: "handle_requests" in t and "Save" in t),
    ("feed", lambda t: t.startswith("feed report") and " cap 0 " not in t and "(0 rows differ)" not in t),
])
def test_a_corrupted_observation_fails_at_its_step(kind, marker):
    seed, flags = 3, capi.BGR_CFG_DESYNC_CAPTURE
    clean = _run(flags, seed, steps=50)
    step = _first_step(clean.log[10:], marker)
    with pytest.raises(CheckFailed) as ei:
        _run(flags, seed, corrupt=(kind, step), steps=50)
    msg = str(ei.value)
    assert f"configuration fake seed {seed} step {step}:" in msg
    assert "action log:" in msg and f"  {step}: " in msg


@pytest.mark.parametrize("flags", FLAGS, ids=str)
def test_checkpoints_restores_and_replays_are_accepted(flags):
    t = _run(flags, 20, steps=60, match=True).tally
    assert t["checkpoints"] + t["restores"] + t["input_replays"] > 5, dict(t)


def test_match_state_actions_reach_every_case_over_a_few_seeds():
    total = {}
    for seed, flags in enumerate(FLAGS):
        for k, v in _run(flags, 30 + seed, steps=60, match=True).tally.items():
            total[k] = total.get(k, 0) + v
    for k in ["checkpoints", "checkpoints_oracle", "checkpoints_in_flight", "checkpoint_none", "restores",
              "restores_older_rows", "restore_refusals", "input_replays", "loads_across_replay", "refusals"]:
        assert total.get(k, 0) > 0, (k, total)


# sha256 of the action logs below, recorded before checkpoints, restores and replays were added to the driver
LOG_DIGESTS = {"single": "3c6ac4b0152d3a94648544c767ef6a78c525d23986c7014464c58aa9176938a7",
               "retain": "6211fa30d397988381cb543aa9c67982c0a43f14ff88d443b6bfbc753cbe8c00",
               "fleet": "e407a8a8f7c74289c48e12e454c05553708cbc7a9f33fcafb55062c5e296afc4"}


def _log_digest(log):
    return hashlib.sha256("\n".join(log).encode()).hexdigest()


def test_match_state_actions_leave_existing_action_logs_alone():
    """The new actions are drawn only when a configuration turns them on: with them off, a seed gives exactly the
    action log it gave before they existed (the tally minimums of the GPU modules were tuned on those logs)."""
    assert _log_digest(_run(capi.BGR_CFG_DESYNC_CAPTURE, 5).log) == LOG_DIGESTS["single"]
    assert _log_digest(_run("retain", 1).log) == LOG_DIGESTS["retain"]
    assert _log_digest(_run_fleet(5).log) == LOG_DIGESTS["fleet"]
    assert _run(capi.BGR_CFG_DESYNC_CAPTURE, 5, match=True).log != _run(capi.BGR_CFG_DESYNC_CAPTURE, 5).log


@pytest.mark.parametrize("kind,marker", [
    ("blob", lambda t: t.lstrip().startswith("checkpoint of frame") and "no image holds it" not in t),
    ("replay_checksum", lambda t: t.startswith("input log") and "(0 checksums)" not in t),
    ("restore", lambda t: t.startswith("restore the checkpoint")),
])
def test_a_corrupted_match_state_fails_at_its_step(kind, marker):
    """A checkpoint blob with one bit flipped, a replay checksum with one bit flipped, one byte of a restored world."""
    seed, flags = 4, capi.BGR_CFG_DESYNC_CAPTURE
    clean = _run(flags, seed, steps=60, match=True)
    step = _first_step(clean.log[10:], marker)
    with pytest.raises(CheckFailed) as ei:
        _run(flags, seed, corrupt=(kind, step), steps=60, match=True)
    msg = str(ei.value)
    assert f"configuration fake seed {seed} step {step}:" in msg
    assert "action log:" in msg and f"  {step}: " in msg


class FakeBatch:
    """EngineBatch's surface over FakeEngines: every listed world is checked before any runs (a refusal names the
    world and runs nothing), then each runs its vector in list order."""

    def __init__(self, fakes):
        self.engines = list(fakes)

    def specialised(self):
        return False

    def close(self):
        pass

    def handle_requests(self, calls):
        seen = set()
        for w, _, reqs in calls:
            assert w not in seen and 0 <= w < len(self.engines)
            seen.add(w)
            ex = self.engines[w]._refusal(reqs)
            if ex is not None:
                raise BgrError(ex.status, f"world {w}: {ex}")
        return [(capi.BGR_OK, self.engines[w]._run(info, reqs, batched=True)) for w, info, reqs in calls]

    def replay(self, calls):
        seen = set()
        for w, log, _ in calls:
            assert w not in seen and 0 <= w < len(self.engines)
            seen.add(w)
            ex = self.engines[w]._replay_refusal(log)
            if ex is not None:
                raise BgrError(ex.status, f"world {w}: {ex}")
        return [(capi.BGR_OK, self.engines[w].replay(log, k)) for w, log, k in calls]


GROW, CAPTURE = capi.BGR_CFG_GROWABLE, capi.BGR_CFG_DESYNC_CAPTURE


def _fleet_config(steps=40, match=False):
    def registration(rng):
        s = random_schema(rng, words=int(rng.integers(4, 14)))
        strategies = [(capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL) if o else capi.BGR_STRATEGY_CLONE
                      for o in s.optional]
        feed = [(c, 0, min(8, sz)) for c, sz in enumerate(s.sizes) if sz % 4 == 0][:2]

        def member(rng, i):
            n = int(rng.integers(300, 1300))
            removes = [(c, int(r)) for c, o in enumerate(s.optional) if o for r in rng.choice(n, 5, replace=False)]
            return World(s.sizes, strategies, [(c, off, ln, 0) for c, off, ln in s.cks],
                         [(k, c, p) for k, c, p in s.systems], s.values(rng, n), removes, feed_fields=feed)
        return member
    members = [Config("", None, flags=0), Config("", None, flags=CAPTURE, fps=30),
               Config("", None, flags=GROW, fps=144, grow_margin=3000), Config("", None, retain=(2, 4), order_base=(1 << 32) + 12345),
               Config("", None, flags=GROW | CAPTURE, grow_margin=3000), Config("", None, order_base=(1 << 32) - 700)]
    if match:
        members = [Config(**{**m.__dict__, "checkpoints": True, "input_replays": True}) for m in members]
    return FleetConfig("fake_fleet", registration, members, steps=steps, match_state=match)


def _run_fleet(seed, corrupt=None, steps=40, match=False):
    fakes, written = [], set()

    def new_engine(member, role, cap, fl, env, fps=60, order_base=0):
        f = FakeEngine(cap, fl, growable=bool(fl & GROW), corrupt=corrupt if (member, role) == (1, "engine") else None,
                       fps=fps, order_base=order_base, written=written)
        fakes.append((member, f))
        return f
    fl = Fleet(_fleet_config(steps, match), seed, new_engine, FakeBatch)
    for member, f in fakes:
        f.driver = fl.members[member]
    try:
        fl.run()
    finally:
        fl.close()
    return fl


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_every_generated_batched_call_is_accepted(seed):
    fl = _run_fleet(seed)
    t = fl.totals()
    assert t["batched_calls"] > 5 and t["batched_worlds"] > t["batched_calls"] and t["vectors_batched"] == t["batched_worlds"]
    assert t["solo_after_batched"] > 0 and t["batched_after_solo"] > 0
    assert all(m.tally["vectors_batched"] > 0 for m in fl.members)
    assert t.get("spawns", 0) == sum(m.tally["spawns"] for m in fl.members if m.cfg.order_base == 0)


def test_fleet_reaches_refusals_and_queued_members_over_a_few_seeds():
    total = {}
    for seed in range(3, 7):
        for k, v in _run_fleet(seed, steps=60).totals().items():
            total[k] = total.get(k, 0) + v
    for k in ["batched_calls", "batch_refusals", "batch_with_queued_member", "solo_after_batched", "batched_after_solo",
              "vectors_queued", "band_writes", "spawns", "growth_steps", "peeks", "live_reads"]:
        assert total.get(k, 0) > 0, k


def test_the_same_fleet_seed_gives_the_same_action_log():
    a, b = _run_fleet(5), _run_fleet(5)
    assert a.log == b.log and len(a.log) > 60
    assert _run_fleet(6).log != a.log


def test_a_corrupted_batched_checksum_fails_at_its_step():
    seed = 3
    clean = _run_fleet(seed, steps=50)
    step = _first_step(clean.log[10:], lambda t: t.startswith("w1 batched") and "Save" in t)
    with pytest.raises(CheckFailed) as ei:
        _run_fleet(seed, corrupt=("batch_checksum", step), steps=50)
    msg = str(ei.value)
    assert f"fleet fake_fleet seed {seed} step {step}:" in msg
    assert "world 1: batched checksums" in msg and f"  {step}: w1 batched" in msg


@pytest.mark.parametrize("seed", [0, 1])
def test_batched_replays_and_cross_restores_are_accepted(seed):
    t = _run_fleet(seed, steps=60, match=True).totals()
    assert t["batch_replays"] + t["cross_restores"] + t["cross_restore_refusals"] > 3, dict(t)


def test_fleet_match_state_reaches_every_case_over_a_few_seeds():
    total = {}
    for seed in range(10, 14):
        for k, v in _run_fleet(seed, steps=60, match=True).totals().items():
            total[k] = total.get(k, 0) + v
    for k in ["batch_replays", "batch_replay_refusals", "batch_replays_with_queued_member", "input_replays_batched",
              "cross_restores", "cross_restores_grown", "cross_restore_refusals", "checkpoints"]:
        assert total.get(k, 0) > 0, (k, total)


def test_a_corrupted_batched_replay_checksum_fails_at_its_step():
    seed = 3
    clean = _run_fleet(seed, steps=60, match=True)
    step = _first_step(clean.log[10:], lambda t: t.startswith("w1 batched input log") and "checksum interval 0" not in t)
    with pytest.raises(CheckFailed) as ei:
        _run_fleet(seed, corrupt=("replay_checksum", step), steps=60, match=True)
    msg = str(ei.value)
    assert f"fleet fake_fleet seed {seed} step {step}:" in msg and "world 1: batched replay checksums" in msg
