"""-m gpu: replays (bgr_replay) held to the oracle driven through the request stream a replay stands for,
[Save(f) at the checksum frames, Advance] in vectors of at most BGR_MAX_REQUESTS, on random registrations
(schema_util.random_schema: sub-word and whole-word columns, up to seven optional columns, whole and partial checksum
ranges, U32_ADD / U32_SATSUB_DESPAWN), with despawn_on_input (which reads the inputs by player handle), with the call
counter, with spawn_particles, wider than the generated kernel takes (the chunked fallback), and with more systems than
the generic program takes (the stepwise path).  Intervals 0, 1, 10 and past the log, from start frames that are and are
not multiples of the interval, on the default kernel selection and with BGR_TUNE_JIT=0.

Compared: the checksums, every column on the rows that exist, presence and alive bytes, the row count, the active
count and the frame count; then both tick on through the request path with spawning inputs, which holds Time<GgrsTime>,
ParticleRng and the call counter to the oracle too."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request
from bevy_ggrs_b200.stress import synth_particles
from oracle_backend import OracleWorld
from schema_util import random_schema

pytestmark = pytest.mark.gpu
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
SPECTATOR = (capi.BGR_SESSION_SPECTATOR, 0, 0, 0)
SPAWN = capi.BGR_INPUT_SPAWN
FRAMES = 150
# (interval, start frame): 0; every frame; 10 from a multiple of 10 and from a frame that is not; past the log
POINTS = [(0, 7), (1, 0), (10, 10), (10, 7), (FRAMES + 5, 3)]
KINDS = ["random", "random_words", "despawn_on_input", "counter", "spawning", "wide", "many_systems"]


def registration(kind, rng):
    """(schema, spawn rate, player count) of one drawn registration of `kind`."""
    def words(budget):   # whole-word columns (what the generated kernel takes), at most `budget` bytes
        sz = [int(x) for x in rng.choice([4, 8, 12, 16, 40], int(rng.integers(2, 6)))]
        while sum(sz) > budget:
            sz.pop()
        return sz or [4]
    if kind == "wide":   # 30 words: past the generated kernel's 24
        return random_schema(rng, words=30), 0, 2
    if kind == "random":   # sub-word columns and partial ranges too: mostly the chunked fallback
        return random_schema(rng, words=int(rng.integers(3, 16))), 0, 2
    if kind == "random_words":
        return random_schema(rng, sizes=words(96), ranges=("none", "whole")), 0, 2
    if kind == "counter":
        return random_schema(rng, sizes=[8] + words(88), store_call_count=True, ranges=("none", "whole")), 0, 2
    s = random_schema(rng, sizes=words(36 if kind == "spawning" else 96), ranges=("none", "whole"))
    if kind == "despawn_on_input":
        c = int(rng.integers(0, len(s.sizes)))
        s.systems.append((capi.BGR_SYS_DESPAWN_ON_INPUT, [c], [int(rng.integers(0, 3)), 0x0F]))
        return s, 0, 3
    if kind == "many_systems":   # nine systems: the generic program takes eight
        c = next(i for i, sz in enumerate(s.sizes) if sz % 4 == 0) if any(sz % 4 == 0 for sz in s.sizes) else None
        if c is None:
            s.sizes.append(4)
            s.optional.append(False)
            c = len(s.sizes) - 1
        s.systems = [(capi.BGR_SYS_U32_ADD, [c], [0, k + 1]) for k in range(9)]
        return s, 0, 1
    if kind == "spawning":   # Transform / Velocity / Ttl behind the random columns, spawn_particles with them
        t = len(s.sizes)
        s.sizes += [40, 12, 8]
        s.optional += [False, False, False]
        if len(s.cks) < 6:
            s.cks.append((t, 0, 40))
        rate = int(rng.integers(1, 40))
        s.systems += [(capi.BGR_SYS_PARTICLES_SPAWN, [t, t + 1, t + 2], [rate, 9, 0xC0FFEE, 0]),
                      (capi.BGR_SYS_PARTICLES_UPDATE, [t, t + 1], []), (capi.BGR_SYS_PARTICLES_DESPAWN, [t + 2], [])]
        return s, rate, 2
    return s, 0, 2


def worlds(kind, seed, n):
    rng = np.random.default_rng(0xBEEF + 97 * seed + KINDS.index(kind))
    s, rate, players = registration(kind, rng)
    data = s.values(rng, n)
    if rate:   # particle columns: finite floats and small ttls, as the example spawns them
        tf, vel, ttl = synth_particles(n, seed, 2, 40)
        data[-3:] = [tf.view(np.uint8).reshape(n, 40), vel.view(np.uint8).reshape(n, 12), ttl.view(np.uint8).reshape(n, 8)]
    removes = [(c, int(r)) for c, o in enumerate(s.optional) if o for r in rng.choice(n, min(n, 9), replace=False)]
    out = []
    for w in (Engine(max_entities=n + rate * FRAMES + rate * 40 + 8, max_depth=4), OracleWorld()):
        cols = s.register(w)
        w.build()
        w.spawn(n)
        for c, d in zip(cols, data):
            w.write_component(c, 0, d)
        for c, r in removes:
            w.remove_component(cols[c], r)
        out.append(w)
    eng, orc = out
    return eng, orc, cols, s, rate, players, rng


def log_for(rng, n_frames, players, spawning, despawn_value=0x0F):
    log = rng.integers(0, 15, (n_frames, players), dtype=np.uint8)   # never the despawn value but on chosen frames
    log[rng.choice(n_frames, 3, replace=False), rng.integers(0, players)] = despawn_value
    if spawning:
        log[rng.choice(n_frames, n_frames // 6, replace=False), 0] |= SPAWN
    return log


def stream_of(f0, log, k):
    vecs, cur = [], []
    for j, row in enumerate(log):
        reqs = ([Request(SAVE, f0 + j)] if k and (f0 + j) % k == 0 else []) + [Request(ADVANCE, 0, [int(v) for v in row])]
        if len(cur) + len(reqs) > capi.BGR_MAX_REQUESTS:
            vecs.append(cur)
            cur = []
        cur += reqs
    return vecs + ([cur] if cur else [])


def oracle_stream(orc, f0, log, k):
    return [cs for v in stream_of(f0, log, k) for cs in orc.handle_requests(NOSESS, v)]


def assert_state(eng, orc, cols):
    n = eng.row_count()
    assert n == orc.row_count()
    assert eng.rollback_frame_count() == orc.rollback_frame_count()
    assert eng.active_count() == orc.active_count()
    alive = eng.read_alive(0, n).astype(bool)
    assert np.array_equal(alive, orc.read_alive(0, n).astype(bool))
    for c in cols:
        has_e = eng.has_component(c, 0, n).astype(bool)
        do, has_o = orc.read_component_alive(c, 0, n)
        has_o = has_o.astype(bool)
        assert np.array_equal(has_e[alive], has_o[alive]), f"presence of column {c}"
        m = alive & has_o
        assert np.array_equal(eng.read_component(c, 0, n)[m], do[m]), f"column {c}"


def fast_expected(s, env):
    return env == "default" and s.words <= 24 and s.nvrtc_ranges and len(s.systems) <= 8


@pytest.mark.parametrize("env", ["default", "jit0"])
@pytest.mark.parametrize("point", range(len(POINTS)))
@pytest.mark.parametrize("kind", KINDS)
def test_replay_matches_the_oracle(monkeypatch, kind, point, env):
    if env == "jit0":
        monkeypatch.setenv("BGR_TUNE_JIT", "0")
    k, f0 = POINTS[point]
    eng, orc, cols, s, rate, players, rng = worlds(kind, point, int(np.random.default_rng(point).integers(200, 1500)))
    for w in (eng, orc):
        w.set_rollback_frame_count(f0)
    log = log_for(rng, FRAMES, players, bool(rate))
    got = eng.replay(log, k)
    assert got == oracle_stream(orc, f0, log, k)
    assert len(got) == sum(1 for j in range(FRAMES) if k and (f0 + j) % k == 0)
    assert eng.last_kernel().replay == fast_expected(s, env)
    assert_state(eng, orc, cols)
    if rate:
        assert eng.row_count() > 0 and eng.row_count() == orc.row_count()
    # on through the request path: the frame's time, the ParticleRng draws and the counter continue from the replay's
    f1 = eng.rollback_frame_count()
    tail = log_for(rng, 20, players, bool(rate))
    tail[::4, 0] |= SPAWN if rate else 0
    for v in stream_of(f1, tail, 1):   # the engine's spectator ring (depth 0) checksums without storing, like the replay
        assert eng.handle_requests(SPECTATOR, v) == orc.handle_requests(NOSESS, v)
    assert_state(eng, orc, cols)
