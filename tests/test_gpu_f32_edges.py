"""-m gpu: the f32 systems on IEEE binary32 edge values, on every kernel, against the plain restatement (f32_ref.py).

What holds (DESIGN.md "Oracle and parity status"):
  * every finite or infinite result is bit-identical to the restatement and to the oracle: subnormal results, signed
    zeros, ties-to-even, overflow to +-inf;
  * where the CPU produces a NaN the engine produces a NaN (payload not compared with the CPU);
  * every GPU kernel variant produces the same bytes, NaN bits included (two peers on different kernels agree);
  * bytes no system writes (rotation, scale, other columns) are copied verbatim, signalling NaNs included;
  * the finite assertion never fires for a row the query does not match.
"""
import numpy as np
import pytest

import f32_ref as R
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request, SyncTestSession
from oracle_backend import OracleError, OracleWorld
from schema_util import path_env

FPS = R.KAT_FPS

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
COPY, CLONE = capi.BGR_STRATEGY_COPY, capi.BGR_STRATEGY_CLONE
STEPWISE = capi.BGR_CFG_FORCE_STEPWISE
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
N = 1500
TTL0 = 1_000_000
GENERIC = {"BGR_TUNE_BUNDLE": "0"}
NVRTC = dict(GENERIC, BGR_TUNE_JIT="2")

# name: (environment, engine flags, extra optional column, expected (kind, mode or item rows))
VARIANTS = {
    "bundle_mode0": ({}, 0, False, ("bundle", 0)),
    "bundle_mode2": ({}, 0, True, ("bundle", 2)),
    "interpreter": (dict(GENERIC, BGR_TUNE_JIT="0"), 0, False, ("generic_interpreter", None)),
    "nvrtc_512_rows4": (dict(NVRTC, BGR_TUNE_JIT_ITEM="512"), 0, False, ("generic_nvrtc", 512)),
    "nvrtc_512_rows2": (dict(NVRTC, BGR_TUNE_JIT_ITEM="512", BGR_TUNE_JIT_ROWS="2"), 0, False, ("generic_nvrtc", 512)),
    "nvrtc_512_rows1": (dict(NVRTC, BGR_TUNE_JIT_ITEM="512", BGR_TUNE_JIT_ROWS="1"), 0, False, ("generic_nvrtc", 512)),
    "nvrtc_128": (NVRTC, 0, False, ("generic_nvrtc", 128)),
    "stepwise_tma": ({}, STEPWISE, False, ("stepwise_tma", None)),
    "stepwise_flat": ({"BGR_TUNE_TMA": "0"}, STEPWISE, False, ("stepwise_flat", None)),
}


def _vectors(n_ticks, players=2, inputs=lambda tick, h: 0):
    sess = SyncTestSession(players, 2, 8)
    out = []
    for tick in range(n_ticks):
        for h in range(players):
            sess.add_local_input(h, inputs(tick, h))
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        out.append(reqs)
    return sess.info(), out


class _States:
    """The restatement's state at every frame: states[f] = (t bits (n, 10), v bits (n, 3)) after f Advances."""

    def __init__(self, t, v, fps, step):
        self.frames, self.fps, self.step = [(t, v)], fps, step

    def at(self, f, inputs=None):
        while len(self.frames) <= f:
            k = len(self.frames)
            t, v = self.frames[-1]
            nt, nv = self.step(t, v, R.dt_bits_of(self.fps, k), k)
            t = t.copy()
            t[:, 0:3] = nt
            self.frames.append((t, nv))
        return self.frames[f]


def _walk(vector, cur):
    """Frame the world is at after the vector, and the frames it saved."""
    saved = []
    for r in vector:
        if r.kind == LOAD:
            cur = r.frame
        elif r.kind == ADVANCE:
            cur += 1
        else:
            assert r.frame == cur
            saved.append(r.frame)
    return cur, saved


def _register_particles(w, fin, opt_tag):
    t = w.rollback_component("Transform", 40, CLONE)
    v = w.rollback_component("Velocity", 12, COPY)
    l = w.rollback_component("Ttl", 8, COPY)
    w.checksum_component(v, 0, 12, FIN if fin else 0)
    w.checksum_component(t, 0, 12, FIN if fin else 0)
    w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
    w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
    cols = [t, v, l]
    if opt_tag:
        cols.append(w.rollback_component("Tag", 12, COPY | OPT))
    return cols


def _particles_world(w, t, v, fin=False, opt_tag=False):
    cols = _register_particles(w, fin, opt_tag)
    w.build()
    w.spawn(N)
    w.write_component(cols[0], 0, t)
    w.write_component(cols[1], 0, v)
    w.write_component(cols[2], 0, np.full(N, TTL0, np.uint64))
    if opt_tag:
        w.write_component(cols[3], 0, np.roll(t[:, 3:6], 1, axis=0).copy())
    return cols


def _check_state(got_t, got_v, got_l, want, frame, t0):
    """Live or peeked bytes of every row against the restatement at `frame`."""
    wt, wv = want
    gt, gv = got_t.view(np.uint32), got_v.view(np.uint32)
    assert R.same_f32(gt[:, 0:3], wt[:, 0:3]).all(), np.argwhere(~R.same_f32(gt[:, 0:3], wt[:, 0:3]))[:5]
    assert R.same_f32(gv, wv).all(), np.argwhere(~R.same_f32(gv, wv))[:5]
    assert np.array_equal(gt[:, 3:10], t0[:, 3:10])   # rotation / scale: verbatim
    assert (got_l.view(np.uint64)[:, 0] == TTL0 - frame).all()


def _run_particles(eng, cols, info, vectors, states, t0):
    """Every vector: checksums, live state against the restatement, every ring frame peeked.  Returns the bytes seen."""
    seen, cur = [], 0
    for vec in vectors:
        cks = eng.handle_requests(info, vec)
        cur, saved = _walk(vec, cur)
        assert [f for f, _ in cks] == saved
        live = [eng.read_component(c, 0, N) for c in cols]
        _check_state(live[0], live[1], live[2], states.at(cur), cur, t0)
        peeks = {}
        for f in eng.snapshot_frames():
            pk = [eng.peek(f, c, 0, N) for c in cols]
            assert all(p is not None and p[1].all() for p in pk)
            _check_state(pk[0][0], pk[1][0], pk[2][0], states.at(f), f, t0)
            peeks[f] = [p[0] for p in pk[:3]]
        seen.append((cks, [x for x in live[:3]], peeks, eng.last_kernel()))
    return seen


def _has_nan(state):
    return bool(R.is_nan_bits(state[0][:, 0:3]).any() or R.is_nan_bits(state[1]).any())


def _oracle_checksums(t, v, fin, info, vectors, fps):
    orc = OracleWorld(fps=fps)
    _particles_world(orc, t, v, fin=fin)
    try:
        return [orc.handle_requests(info, vec) for vec in vectors]
    finally:
        orc.close()


@pytest.mark.parametrize("fps", FPS)
def test_particles_edge_values_on_every_kernel(monkeypatch, fps):
    """The edge table through 10 SyncTest ticks (check distance 2) on every kernel that runs update_particles."""
    t, v = R.edge_table(R.dt_bits_of(fps, 1), N, seed=fps)
    step = lambda t_, v_, dt, k: R.particle_step(t_[:, 0:3], v_, dt)
    states = _States(t, v, fps, step)
    info, vectors = _vectors(10)
    want = _oracle_checksums(t, v, False, info, vectors, fps)
    results = {}
    for name, (env, flags, opt_tag, (kind, sub)) in VARIANTS.items():
        with monkeypatch.context() as m:
            for k, val in env.items():
                m.setenv(k, val)
            eng = Engine(max_entities=N, max_depth=8, fps=fps, flags=flags)
            cols = _particles_world(eng, t, v, opt_tag=opt_tag)
            seen = _run_particles(eng, cols[:3], info, vectors, states, t)
            if opt_tag:   # the optional column no system touches: verbatim
                assert np.array_equal(eng.read_component(cols[3], 0, N).view(np.uint32), np.roll(t[:, 3:6], 1, axis=0))
            eng.close()
        k = seen[-1][3]
        assert k.kind == kind, (name, k)
        if kind == "bundle":
            assert k.mode == sub, (name, k)
        elif kind == "generic_nvrtc":
            assert k.item_rows == sub, (name, k)
        results[name] = seen
    # every variant: the same checksums and the same bytes, NaN bits included
    first = results["bundle_mode0"]
    for name, seen in results.items():
        for a, b in zip(first, seen):
            assert a[0] == b[0], name
            assert all(np.array_equal(x, y) for x, y in zip(a[1], b[1])), name
            assert a[2].keys() == b[2].keys() and all(np.array_equal(x, y) for f in a[2] for x, y in zip(a[2][f], b[2][f])), name
    # the oracle wherever no NaN is hashed
    cur = 0
    for vec, got, exp in zip(vectors, first, want):
        cur, saved = _walk(vec, cur)
        for (f, ck), (fo, cko) in zip(got[0], exp):
            assert f == fo
            if not _has_nan(states.at(f)):
                assert ck == cko, (f, fps)


@pytest.mark.parametrize("fps", FPS)
def test_particles_finite_edge_values_with_the_finite_assertion(fps):
    """MODE 1 (both columns checksummed with the finite assertion): the table without the rows that are or become
    non-finite, so nothing raises; bit-identical with the restatement and the oracle's checksums."""
    t, v = R.edge_table(R.dt_bits_of(fps, 1), N, seed=fps)
    info, vectors = _vectors(10)
    last = 0
    for vec in vectors:
        last, _ = _walk(vec, last)
    step = lambda t_, v_, dt, k: R.particle_step(t_[:, 0:3], v_, dt)
    probe = _States(t, v, fps, step)
    bad = np.zeros(N, bool)
    for f in range(last + 1):
        st, sv = probe.at(f)
        bad |= ((st[:, 0:3] & 0x7F800000) == 0x7F800000).any(1) | ((sv & 0x7F800000) == 0x7F800000).any(1)
    t, v = t.copy(), v.copy()
    t[bad, 0:3] = 0
    v[bad] = 0
    assert (~bad).sum() > N // 2
    states = _States(t, v, fps, step)
    want = _oracle_checksums(t, v, True, info, vectors, fps)
    eng = Engine(max_entities=N, max_depth=8, fps=fps)
    cols = _particles_world(eng, t, v, fin=True)
    seen = _run_particles(eng, cols, info, vectors, states, t)
    assert [s[0] for s in seen] == want
    k = seen[-1][3]
    assert (k.kind, k.mode) == ("bundle", 1)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# move_cube_system at scale, bit-exact
# ---------------------------------------------------------------------------------------------------------------------
BOX_PATHS = {"interpreter": (dict(BGR_TUNE_JIT="0"), 0, "generic_interpreter"),
             "nvrtc_512": (dict(BGR_TUNE_JIT="2", BGR_TUNE_JIT_ITEM="512"), 0, "generic_nvrtc"),
             "nvrtc_128": (dict(BGR_TUNE_JIT="2"), 0, "generic_nvrtc"),
             "stepwise": ({}, STEPWISE, "stepwise_tma")}
BOX_INPUTS = lambda tick, h: (0b0001, 0b1000, 0b0101, 0, 0b0010, 0b1010, 0b0100, 0b1001, 0b0011, 0b1100)[(tick + 3 * h) % 10]


def _box_table(rng):
    hw = float(R.f32(R.bits_of(R.r32(R.r32(5.0 - float(np.float32(0.2))) * 0.5))))
    t = np.zeros((N, 10), np.float32)
    t[:, 0:3] = rng.uniform(-2.4, 2.4, (N, 3))
    t[:, 6] = 1.0
    t[:, 7:10] = 1.0
    t[0::5, 0] = hw; t[1::5, 0] = -hw; t[2::5, 2] = hw; t[3::5, 2] = -hw      # on the clamp
    d = rng.normal(size=(N, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    mag = rng.choice([0.0, 1e-40, 2.9, 3.0, 3.0000002, 3.5, 40.0], N)
    v = (d * mag[:, None]).astype(np.float32)
    v[0::11] = (3.0, 0.0, 0.0); v[1::11] = (0.0, 0.0, -3.0); v[2::11] = (0.0, 3.0, 0.0)   # |v|^2 = 9 exactly
    tb, vb = t.view(np.uint32), v.view(np.uint32)
    sub = np.array(R.EDGE[:8], np.uint32)   # +-0, +-min / max subnormal, +-FLT_MIN
    tb[4::13, 0:3] = sub[rng.integers(0, 8, (len(tb[4::13]), 3))]
    vb[5::13] = sub[rng.integers(0, 8, (len(vb[5::13]), 3))]
    return tb.copy(), vb.copy()


@pytest.mark.parametrize("path", list(BOX_PATHS))
@pytest.mark.parametrize("fps", FPS)
def test_box_move_bit_exact_at_scale(monkeypatch, fps, path):
    """1,500 cubes, 8 players, an optional Velocity removed from some rows (the query skips them), host despawns, 12
    SyncTest ticks: live state and every ring frame bit-identical with the restatement, checksums with the oracle."""
    env, flags, kind = BOX_PATHS[path]
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    rng = np.random.default_rng(fps)
    t, v = _box_table(rng)
    no_vel = sorted({3, 511, 512, 513} | set(range(17, N, 7)))
    dead = [6, 600, N - 1]
    has = np.ones(N, bool); has[no_vel] = False
    alive = np.ones(N, bool); alive[dead] = False
    info, vectors = _vectors(12, players=8, inputs=BOX_INPUTS)
    inputs_at = {}

    def step(t_, v_, dt, k):
        inp = np.zeros(N, np.uint32)
        inp[:8] = inputs_at[k]
        nt, nv = R.box_move_step(t_[:, 0:3], v_, dt, inp)
        m = has & alive
        return np.where(m[:, None], nt, t_[:, 0:3]), np.where(m[:, None], nv, v_)

    states = _States(t, v, fps, step)
    worlds = []
    for w in (Engine(max_entities=N, max_depth=8, fps=fps, flags=flags), OracleWorld(fps=fps)):
        tf = w.rollback_component("Transform", 40, CLONE)
        vel = w.rollback_component("Velocity", 12, COPY | OPT)
        w.checksum_component(tf, 0, 12)
        w.checksum_component(vel, 0, 12)
        w.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
        w.build()
        w.spawn(N)
        w.write_component(tf, 0, t)
        w.write_component(vel, 0, v)
        for r in no_vel:
            w.remove_component(vel, r)
        for r in dead:
            w.despawn(r)
        worlds.append((w, tf, vel))
    (eng, tf, vel), (orc, _, _) = worlds
    cur = 0
    for vec in vectors:
        for r in vec:
            if r.kind == ADVANCE:
                cur += 1
                inputs_at.setdefault(cur, list(r.inputs))
                assert inputs_at[cur] == list(r.inputs)
            elif r.kind == LOAD:
                cur = r.frame
        assert eng.handle_requests(info, vec) == orc.handle_requests(info, vec)
        wt, wv = states.at(cur)
        live = eng.read_alive(0, N).astype(bool)
        assert np.array_equal(live, alive)
        gt = eng.read_component(tf, 0, N).view(np.uint32)
        gv = eng.read_component(vel, 0, N).view(np.uint32)
        assert np.array_equal(gt[alive], wt[alive]), np.argwhere(gt[alive] != wt[alive])[:4]
        assert np.array_equal(gv[alive & has], wv[alive & has])
        for f in eng.snapshot_frames():
            pt, pv = eng.peek(f, tf, 0, N), eng.peek(f, vel, 0, N)
            ft, fv = states.at(f)
            assert np.array_equal(pt[0].view(np.uint32)[alive], ft[alive])
            assert np.array_equal(pv[0].view(np.uint32)[alive & has], fv[alive & has])
    assert eng.last_kernel().kind == kind
    if path.startswith("nvrtc"):
        assert eng.last_kernel().item_rows == int(path.split("_")[1])
    v_end = states.at(cur)[1].view(np.float32)
    assert (np.linalg.norm(v_end[alive & has].astype(np.float64), axis=1) <= 3.0 + 1e-6).all()
    eng.close(); orc.close()


# ---------------------------------------------------------------------------------------------------------------------
# the finite assertion never fires for a row the query skips
# ---------------------------------------------------------------------------------------------------------------------
# hash implementation: (path of schema_util.WIDE_PATHS or "bundle", Transform's checksummed range, expected kind)
HASHERS = {"bundle": ("bundle", (0, 12), "bundle"),
           "generic_inline": ("generic", (0, 12), None),       # 12-byte range: the interpreter's branch-free path
           "generic_general": ("generic", (0, 20), None),      # 20 bytes: hash_row_range (NVRTC: its own 5-word hash)
           "stepwise_tma": ("stepwise_tma", (0, 12), "stepwise_tma"),
           "stepwise_flat": ("stepwise_flat", (0, 12), "stepwise_flat")}


@pytest.mark.parametrize("pattern", [0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFC01234])
@pytest.mark.parametrize("case", ["despawned", "dies_while_overflowing", "column_removed"])
@pytest.mark.parametrize("hasher", list(HASHERS))
def test_finite_assertion_skips_rows_outside_the_query(monkeypatch, generic_kernel, hasher, case, pattern):
    """A non-finite value in a despawned row, in a row whose Ttl reaches 0 in the Advance in which its translation
    overflows, or in a row whose Velocity was removed: the checksummed queries do not match the row, so neither the
    oracle nor any hash implementation raises, and the checksums agree."""
    path, (off, ln), kind = HASHERS[hasher]
    if path == "bundle":
        if generic_kernel != "interpreter":
            pytest.skip("the bundle does not depend on the generic kernel: run once")
        flags = 0
    else:
        flags = path_env(monkeypatch, path, generic_kernel)
        monkeypatch.setenv("BGR_TUNE_BUNDLE", "0")
    if case == "dies_while_overflowing" and pattern != 0x7F800000:
        pytest.skip("the overflow makes its own +inf")
    if kind is None:
        kind = "generic_interpreter" if generic_kernel == "interpreter" else "generic_nvrtc"
    n, row = 700, 517
    rng = np.random.default_rng(pattern & 0xFFFF)
    tf = np.zeros((n, 10), np.float32)
    tf[:, 0:3] = rng.uniform(-100, 100, (n, 3)); tf[:, 6:10] = 1.0
    vel = rng.uniform(-50, 50, (n, 3)).astype(np.float32)
    ttl = np.full(n, 50, np.uint64)
    tb, vb = tf.view(np.uint32), vel.view(np.uint32)
    if case == "dies_while_overflowing":
        tb[row, 0] = vb[row, 0] = 0x7F7FFFFF   # FLT_MAX + FLT_MAX * dt = +inf, in the Advance that despawns the row
        ttl[row] = 1
    else:
        vb[row, 1] = pattern
    if case == "despawned":
        tb[row, 4] = pattern                   # also inside the 20-byte range (rotation.y)
    res = []
    for w in (Engine(max_entities=n, max_depth=8, flags=flags), OracleWorld()):
        t = w.rollback_component("Transform", 40, CLONE)
        v = w.rollback_component("Velocity", 12, COPY | (OPT if case == "column_removed" else 0))
        l = w.rollback_component("Ttl", 8, COPY)
        w.checksum_component(v, 0, 12, FIN)
        w.checksum_component(t, off, ln, FIN)
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        w.build()
        w.spawn(n)
        w.write_component(t, 0, tb); w.write_component(v, 0, vb); w.write_component(l, 0, ttl)
        if case == "despawned":
            w.despawn(row)
        elif case == "column_removed":
            w.remove_component(v, row)
        out = []
        try:
            for f in range(3):
                out.append(w.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, [0])]))
        except (BgrError, OracleError) as ex:
            out.append(("raised", ex.status, str(ex)))
        res.append((out, w))
    (got, eng), (want, orc) = res
    assert got == want
    assert all(isinstance(x, list) for x in got), got
    k = eng.last_kernel()
    assert k.kind == kind
    if kind == "bundle":
        assert k.mode == (2 if case == "column_removed" else 1)
    eng.close(); orc.close()
