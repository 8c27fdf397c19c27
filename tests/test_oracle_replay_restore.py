"""The oracle's two restatements behind the interleavings' checkpoints and replays (tests/interleave_driver.py), held to
the oracle's own request path:

  - ``FlagsOracle.replay(log, k)`` (orc_checksum_world, then an Advance outside any session) gives the checksums and
    the live world of the stream [Save(f) if f % k == 0, Advance] on a second oracle, and leaves the ring, the confirmed
    frame and the held frames' bytes alone;
  - ``FlagsOracle.restore(checkpoint_of(F))`` (orc_restore from the numpy decoder) continues like ``Load(F)`` on a twin
    oracle over the vectors that follow: checksums, rows, presence and bytes, spawns included (ParticleRng comes from a
    Python restatement of the generator, which the oracle's snapshots do not expose)."""
import numpy as np
import pytest

import checkpoint_codec as cc
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request, Xoshiro256pp
from bevy_ggrs_b200.stress import register_particles, synth_particles
from interleave_driver import NOSESS, FlagsOracle
from schema_util import random_schema

RATE, SEED = 5, 123


def _particles(n, seed):
    o = FlagsOracle(max_entities=1 << 16, max_depth=9)
    cols = register_particles(o, spawn_rate=RATE, rng_seed=SEED)
    tf, vel, ttl = synth_particles(n, seed, 3, 40, z_fraction=0.2)
    o.spawn(n)
    for c, a in zip(cols, (tf, vel, ttl)):
        o.write_component(c, 0, np.ascontiguousarray(a).view(np.uint8).reshape(n, -1))
    o.set_depth(8)
    return o


def _schema_world(n, seed):
    s = random_schema(np.random.default_rng(seed), words=9, n_opt=2)
    o = FlagsOracle(max_entities=1 << 16, max_depth=9)
    s.register(o)
    o.spawn(n)
    rng = np.random.default_rng(seed + 1)
    for c, d in enumerate(s.values(rng, n)):
        o.write_component(c, 0, d)
    for c, opt in enumerate(s.optional):
        if opt:
            for r in rng.choice(n, n // 5, replace=False):
                o.remove_component(c, int(r))
    o.set_depth(8)
    return o


WORLDS = {"particles": lambda seed: _particles(700, seed), "schema": lambda seed: _schema_world(900, seed)}


def _state(o):
    rows = o.row_count()
    out = [o.rollback_frame_count(), rows, o.active_count(), o.read_alive(0, rows).tobytes()]
    for c in range(len(o.elem_bytes)):
        v, has = o.read_component_alive(c, 0, rows)
        out += [v.tobytes(), has.tobytes()]
    return out


def _rows(o, f):
    return o._latest[f]["rows"]


def _held_bytes(o):
    return {f: [o.peek(f, c, 0, _rows(o, f))[0].tobytes() for c in range(len(o.elem_bytes))]
            for f in o.snapshot_frames()}


def _log(rng, n, players, spawn):
    log = rng.integers(0, 16, (n, players), dtype=np.uint8)
    if spawn:
        log[rng.random(n) < 0.3, 0] |= capi.BGR_INPUT_SPAWN
    return log


def _ticks(o, rng, k, spawn):
    for _ in range(k):
        f = o.rollback_frame_count()
        o.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, [int(_log(rng, 1, 1, spawn)[0, 0])])])


@pytest.mark.parametrize("world", sorted(WORLDS))
@pytest.mark.parametrize("k", [0, 1, 3, 7, 1000])
def test_replay_equals_the_save_advance_stream(world, k):
    a, b, c = WORLDS[world](1), WORLDS[world](1), WORLDS[world](1)
    rng = np.random.default_rng(k)
    spawn = world == "particles"
    for o in (a, b, c):
        _ticks(o, np.random.default_rng(5), 12, spawn)
    frames, confirmed, held = a.snapshot_frames(), a.confirmed_frame_count(), _held_bytes(a)
    f0 = a.rollback_frame_count()
    log = _log(rng, 40, 3, spawn)
    got = a.replay(log, k)
    expect = []
    for j in range(len(log)):
        reqs = ([Request(SAVE, f0 + j)] if k and (f0 + j) % k == 0 else []) + [Request(ADVANCE, 0, [int(v) for v in log[j]])]
        expect += b.handle_requests(NOSESS, reqs)
    assert got == expect and len(got) == sum(1 for j in range(40) if k and (f0 + j) % k == 0)
    assert _state(a) == _state(b)
    if spawn:
        assert a.row_count() > 700
    # the ring is untouched: the same frames, the same bytes, the same confirmed frame
    assert a.snapshot_frames() == frames and a.confirmed_frame_count() == confirmed and _held_bytes(a) == held
    # a Load of a frame from before the replay still works: it continues like the world that never replayed
    g = frames[len(frames) // 2]
    tail = [Request(LOAD, g)] + [q for i in range(3) for q in (Request(ADVANCE, 0, [i]), Request(SAVE, g + i + 1))]
    assert a.handle_requests(NOSESS, tail) == c.handle_requests(NOSESS, tail)
    assert _state(a)[2:] == _state(c)[2:]   # rows: RollbackOrdered keeps the replay's spawns


@pytest.mark.parametrize("world", sorted(WORLDS))
def test_restore_of_the_oracle_checkpoint_continues_like_a_load(world):
    spawn = world == "particles"
    a, b = WORLDS[world](2), WORLDS[world](2)
    n0 = a.row_count()
    rng = np.random.default_rng(9)
    for o in (a, b):
        _ticks(o, np.random.default_rng(6), 10, spawn)
    f = a.snapshot_frames()[2]   # newest first: still held after three more Saves
    rows_f = _rows(a, f)
    rng_f = (0, 0, 0, 0)
    if spawn:
        x = Xoshiro256pp(SEED)
        for _ in range(2 * (rows_f - n0)):
            x.next_u64()
        rng_f = tuple(x.s)
    blob = a.checkpoint_of(f, 0, rng_f)
    h, planes, mask = cc.decode(blob)
    assert (h["frame"], h["rows"], h["fps"]) == (f, rows_f, 60)
    assert h["active"] == int(np.count_nonzero(mask.reshape(-1)[:rows_f] & 1))
    for o in (a, b):   # both move on past f, the restore then goes back to it
        _ticks(o, np.random.default_rng(7), 3, spawn)
    a.restore(blob)
    assert a.snapshot_frames() == [f] and a.rollback_frame_count() == f and a.row_count() == rows_f
    assert a.checkpoint_of(f, 0, rng_f) == blob   # the restored slot holds the blob's world
    b.handle_requests(NOSESS, [Request(LOAD, f)])
    assert _state(a) == _state(b)
    for i in range(12):
        g = a.rollback_frame_count()
        inp = [int(v) for v in _log(rng, 1, 2, spawn)[0]]
        if i % 4 == 3:   # a rollback of two frames
            reqs = [Request(LOAD, g - 2), Request(ADVANCE, 0, inp), Request(SAVE, g - 1), Request(ADVANCE, 0, inp),
                    Request(SAVE, g), Request(ADVANCE, 0, inp)]
        else:
            reqs = [Request(SAVE, g), Request(ADVANCE, 0, inp)]
        assert a.handle_requests(NOSESS, reqs) == b.handle_requests(NOSESS, reqs), f"vector {i}"
        assert _state(a) == _state(b), f"vector {i}"
    if spawn:
        assert a.row_count() > rows_f
