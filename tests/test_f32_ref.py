"""The binary32 restatement (f32_ref.py) against numpy float32 arithmetic and against the oracle, without a GPU:
what the GPU edge-value tests compare the kernels with has to be right first."""
import json
import os

import numpy as np
import pytest

import f32_ref as R
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.session import ADVANCE, Request
from oracle_backend import OracleWorld

NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
KATS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "third_party_kats.json")))
FPS = R.KAT_FPS


def _np32_particle_step(t, v, dt_bits):
    """update_particles in numpy float32 (IEEE per operation on the CPU): an independent second restatement."""
    dt = np.uint32(dt_bits).view(np.float32)
    tf, vf = t.view(np.float32).copy(), v.view(np.float32).copy()
    g = np.array([np.float32(0) * np.float32(200), np.float32(-1) * np.float32(200), np.float32(0) * np.float32(200)], np.float32)
    with np.errstate(all="ignore"):
        vf = vf + g * dt
        tf = tf + vf * dt
    return tf.view(np.uint32), vf.view(np.uint32)


def _np32_box_move_step(t, v, dt_bits, inputs):
    dt = np.uint32(dt_bits).view(np.float32)
    fr = np.uint32(R.friction_bits(dt_bits)).view(np.float32)
    tf, vf = t.view(np.float32).copy(), v.view(np.float32).copy()
    f = np.float32
    with np.errstate(all="ignore"):
        for r in range(t.shape[0]):
            i = int(inputs[r])
            up, down, left, right = bool(i & 1), bool(i & 2), bool(i & 4), bool(i & 8)
            x, y, z = vf[r]
            a = f(18.0) * dt
            if up and not down: z = z - a
            if not up and down: z = z + a
            if left and not right: x = x - a
            if not left and right: x = x + a
            if not up and not down: z = z * fr
            if not left and not right: x = x * fr
            y = y * fr
            ls = x * x + y * y + z * z
            if ls > f(3.0) * f(3.0):
                ln = np.sqrt(ls)
                x, y, z = f(3.0) * (x / ln), f(3.0) * (y / ln), f(3.0) * (z / ln)
            vf[r] = (x, y, z)
            tf[r] = tf[r] + vf[r] * dt
            hw = (f(5.0) - f(0.2)) * f(0.5)
            for k in (0, 2):
                tf[r, k] = -hw if tf[r, k] < -hw else (hw if tf[r, k] > hw else tf[r, k])
    return tf.view(np.uint32), vf.view(np.uint32)


def _random_bits(rng, n, k):
    """Half random bit patterns, half moderate values (where box move's clamps and friction act)."""
    a = rng.integers(0, 2 ** 32, (n, k), dtype=np.uint64).astype(np.uint32)
    b = rng.uniform(-4.0, 4.0, (n, k)).astype(np.float32).view(np.uint32)
    return np.where(rng.random((n, 1)) < 0.5, a, b)


def test_dt_bits_match_the_duration_kats():
    for v in KATS["duration_as_secs_f32"]["vectors"]:
        assert R.dt_bits_of(v["fps"], v["frame"]) == v["bits"], v


def test_friction_is_the_correctly_rounded_powf_at_every_kat_frame_rate():
    """The C library's powf(0.0018f, dt) for every distinct dt of the KAT frame rates is the correctly rounded binary32
    value (float64 pow of the same inputs, rounded, where no float64 error can reach a rounding boundary)."""
    dts = sorted({R.dt_bits_of(f, k) for f in FPS for k in range(1, 25)})
    assert len(dts) >= 18
    for d in dts:
        exact = np.float64(np.float32(0.0018)) ** R.f32(d)
        lo = np.float64(np.float32(exact))
        ulp = float(np.spacing(np.float32(exact)))
        assert abs(abs(exact - lo) / ulp - 0.5) > 1e-6   # far from a midpoint at float64 precision
        assert R.friction_bits(d) == int(np.float32(exact).view(np.uint32)), hex(d)


@pytest.mark.parametrize("fps", FPS)
def test_particle_step_matches_numpy_float32_on_the_edge_table(fps):
    dt = R.dt_bits_of(fps, 1)
    t, v = R.edge_table(dt, 1500, seed=fps)
    rt, rv = R.particle_step(t[:, :3], v, dt)
    nt, nv = _np32_particle_step(t[:, :3], v, dt)
    assert R.same_f32(rt, nt).all() and R.same_f32(rv, nv).all()
    # the table reaches what it is for: subnormal and zero results, overflow, NaN from -inf + inf
    sub = ((rt & 0x7F800000) == 0) & ((rt & 0x7FFFFF) != 0)
    assert sub.any() and ((rt & 0x7FFFFFFF) == 0x7F800000).any()
    created = R.is_nan_bits(rt) & ~R.is_nan_bits(t[:, :3]) & ~R.is_nan_bits(np.repeat(v[:, :1], 3, 1))
    assert created.any()


@pytest.mark.parametrize("fps", FPS)
def test_ties_round_to_even(fps):
    dt = R.dt_bits_of(fps, 1)
    ties = R.tie_rows(dt)
    assert len(ties) >= 8
    t = np.array([[a, 0, a] for a, _ in ties], np.uint32)
    v = np.array([[b, 0, b] for _, b in ties], np.uint32)
    rt, _ = R.particle_step(t, v, dt)
    for (a, _), got in zip(ties, rt[:, 0]):
        even = int(got) & 1 == 0
        assert even and got in (a, a + 1, a - 1)


@pytest.mark.parametrize("fps", FPS)
def test_box_move_step_matches_numpy_float32(fps):
    rng = np.random.default_rng(fps)
    dt = R.dt_bits_of(fps, 1)
    n = 600
    t, v = _random_bits(rng, n, 3), _random_bits(rng, n, 3)
    t[:40], v[:40] = np.array(R.EDGE, np.uint32)[rng.integers(0, len(R.EDGE), (2, 40, 3))]
    inputs = rng.integers(0, 16, n)
    rt, rv = R.box_move_step(t, v, dt, inputs)
    nt, nv = _np32_box_move_step(t, v, dt, inputs)
    assert R.same_f32(rt, nt).all() and R.same_f32(rv, nv).all()


@pytest.mark.parametrize("fps", FPS)
def test_both_systems_match_the_oracle(fps):
    """One Advance of update_particles and of move_cube_system (8 players) on the oracle, NaN as a class."""
    n = 1500
    dt = R.dt_bits_of(fps, 1)
    t, v = R.edge_table(dt, n, seed=3 * fps)
    inputs = [0b0001, 0b0010, 0b0100, 0b1000, 0b0101, 0b1010, 0b1001, 0b0110]
    for system in (capi.BGR_SYS_PARTICLES_UPDATE, capi.BGR_SYS_BOX_MOVE):
        orc = OracleWorld(fps=fps)
        vel = orc.rollback_component("Velocity", 12)
        tf = orc.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
        orc.add_system(system, [tf, vel])
        orc.spawn(n)
        orc.write_component(tf, 0, t)
        orc.write_component(vel, 0, v)
        orc.handle_requests(NOSESS, [Request(ADVANCE, 0, inputs)])
        assert orc.last_dt_bits() == dt
        ot = orc.read_component(tf, 0, n).view(np.uint32)
        ov = orc.read_component(vel, 0, n).view(np.uint32)
        if system == capi.BGR_SYS_PARTICLES_UPDATE:
            rt, rv = R.particle_step(t[:, :3], v, dt)
        else:
            rt, rv = R.box_move_step(t[:, :3], v, dt, inputs + [0] * (n - 8))
        assert R.same_f32(ot[:, :3], rt).all() and R.same_f32(ov, rv).all()
        assert np.array_equal(ot[:, 3:], t[:, 3:])   # rotation / scale: no system writes them, NaN payloads included
        orc.close()
