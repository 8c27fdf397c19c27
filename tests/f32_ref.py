"""Plain binary32 restatement of the two f32 systems, on arrays of float32 BIT PATTERNS (uint32).

update_particles (particles.rs:272-280) and move_cube_system (box_game.rs:154-206) as the reference writes them: every
mul / add / sub / div / sqrt is evaluated in float64 and rounded to float32.  For these five operations that is the
correctly rounded binary32 result (float64 carries more than 2 * 24 + 2 significand bits, so the double rounding is
innocuous), including subnormal results, signed zeros, ties-to-even and overflow to +-inf.  No numpy float32
arithmetic is used, so the restatement does not depend on how numpy evaluates float32.

NaN is a class here: a NaN result has SOME NaN bit pattern; which one is not specified (Rust leaves NaN payloads
unspecified, and the reference's hasher calls non-finite values non-deterministic).  Compare with `same_f32`.

`FRICTION.powf(dt)` is the C library's powf, called through ctypes: the function the reference and the oracle call.

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import json
import os

import numpy as np

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]
_libm.powf.restype = ctypes.c_float

ACCELERATION, MAX_SPEED, FRICTION, PLANE_SIZE, CUBE_SIZE = 18.0, 3.0, 0.0018, 5.0, 0.2
UP, DOWN, LEFT, RIGHT = 1, 2, 4, 8
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "third_party_kats.json")) as _f:
    KAT_FPS = sorted({v["fps"] for v in json.load(_f)["duration_as_secs_f32"]["vectors"]})   # the frame rates of the KATs


def f32(bits) -> np.ndarray:
    """float32 bit patterns -> float64 values (exact; a signalling NaN comes back quiet, which the NaN class ignores)."""
    with np.errstate(invalid="ignore"):
        return np.asarray(bits, dtype=np.uint32).view(np.float32).astype(np.float64)


def bits_of(x) -> np.ndarray:
    """float64 values that are exactly binary32 -> their bit patterns."""
    return np.asarray(x, dtype=np.float64).astype(np.float32).view(np.uint32)


def r32(x):
    """Round float64 to the nearest binary32 (ties to even; past FLT_MAX + half an ulp: +-inf) and back to float64."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def _k(c: float) -> float:
    """A float32 literal of the reference (`0.2f`) as its exact float64 value."""
    return float(np.float32(c))


def friction_bits(dt_bits: int) -> int:
    """`0.0018f32.powf(dt)` with the C library's powf."""
    dt = float(np.uint32(dt_bits).view(np.float32))
    return int(np.float32(_libm.powf(_k(FRICTION), dt)).view(np.uint32))


def particle_step(t, v, dt_bits):
    """update_particles for rows t[:, 0:3] (translation bits) and v[:, 0:3] (velocity bits); returns new (t, v) bits."""
    dt = float(f32(dt_bits))
    g = (r32(0.0 * 200.0), r32(-1.0 * 200.0), r32(0.0 * 200.0))   # Vec3::NEG_Y * 200.0
    tf, vf = f32(t), f32(v)
    with np.errstate(invalid="ignore"):
        for k in range(3):
            vf[:, k] = r32(vf[:, k] + r32(g[k] * dt))              # velocity += gravity * time_step
            tf[:, k] = r32(tf[:, k] + r32(vf[:, k] * dt))          # translation += velocity * time_step
    return bits_of(tf), bits_of(vf)


def box_move_step(t, v, dt_bits, inputs):
    """move_cube_system for rows t[:, 0:3], v[:, 0:3] (bits) with each row's input byte; returns new (t, v) bits."""
    dt = float(f32(dt_bits))
    fr = float(f32(friction_bits(int(dt_bits))))
    inputs = np.asarray(inputs, dtype=np.uint32)
    up, down, left, right = ((inputs & b) != 0 for b in (UP, DOWN, LEFT, RIGHT))
    tf, vf = f32(t), f32(v)
    with np.errstate(invalid="ignore", divide="ignore"):
        a = r32(_k(ACCELERATION) * dt)
        vf[:, 2] = np.where(up & ~down, r32(vf[:, 2] - a), vf[:, 2])
        vf[:, 2] = np.where(~up & down, r32(vf[:, 2] + a), vf[:, 2])
        vf[:, 0] = np.where(left & ~right, r32(vf[:, 0] - a), vf[:, 0])
        vf[:, 0] = np.where(~left & right, r32(vf[:, 0] + a), vf[:, 0])
        vf[:, 2] = np.where(~up & ~down, r32(vf[:, 2] * fr), vf[:, 2])
        vf[:, 0] = np.where(~left & ~right, r32(vf[:, 0] * fr), vf[:, 0])
        vf[:, 1] = r32(vf[:, 1] * fr)
        # glam Vec3::clamp_length_max(MAX_SPEED): dot product left to right, then MAX_SPEED * (v / length)
        len_sq = r32(r32(r32(vf[:, 0] * vf[:, 0]) + r32(vf[:, 1] * vf[:, 1])) + r32(vf[:, 2] * vf[:, 2]))
        big = len_sq > r32(MAX_SPEED * MAX_SPEED)
        ln = r32(np.sqrt(len_sq))
        for k in range(3):
            vf[:, k] = np.where(big, r32(MAX_SPEED * r32(vf[:, k] / ln)), vf[:, k])
        for k in range(3):
            tf[:, k] = r32(tf[:, k] + r32(vf[:, k] * dt))
        hw = r32(r32(PLANE_SIZE - _k(CUBE_SIZE)) * 0.5)
        for k in (0, 2):   # f32::clamp(-hw, hw): a NaN stays NaN
            tf[:, k] = np.where(tf[:, k] < -hw, -hw, np.where(tf[:, k] > hw, hw, tf[:, k]))
    return bits_of(tf), bits_of(vf)


# ---- the edge-value table -------------------------------------------------------------------------------------------
EDGE = [0x00000000, 0x80000000,   # +-0
        0x00000001, 0x80000001,   # +-min subnormal
        0x007FFFFF, 0x807FFFFF,   # +-max subnormal
        0x00800000, 0x80800000,   # +-FLT_MIN
        0x7F7FFFFF, 0xFF7FFFFF,   # +-FLT_MAX
        0x7F800000, 0xFF800000,   # +-inf
        0x3F800000, 0xC3480000,   # 1.0, -200.0
        0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FFFFFFF, 0x7FC01234]   # quiet / signalling NaNs, payloads
NAN_PATTERNS = EDGE[-6:]


def tie_rows(dt_bits: int):
    """(tx, vx) pairs whose `tx + vx * dt` is EXACTLY halfway between two binary32 values: vx * dt rounds to 2^j and
    tx = 2^(j+24) (even last bit: the tie rounds down) or 2^(j+24) + 2^(j+1) (odd: it rounds up); both signs."""
    dt = float(f32(dt_bits))
    out = []
    for j in (-30, -12, -1, 3, 9):
        p = 2.0 ** j
        v0 = np.float32(p / dt)
        for v in (v0, np.nextafter(v0, np.float32(np.inf)), np.nextafter(v0, np.float32(-np.inf))):
            if r32(float(v) * dt) == p:
                break
        else:
            continue
        for t in (2.0 ** (j + 24), 2.0 ** (j + 24) + 2.0 ** (j + 1)):   # the ulp of t is 2^(j+1): t + 2^j is a midpoint
            assert r32(t + p) != t + p
            for s in (1.0, -1.0):
                out.append((int(bits_of(s * t)), int(bits_of(s * float(v)))))
    return out


def edge_table(dt_bits: int, n: int, seed: int):
    """n rows of particle state as bits: t (n, 10) = translation, rotation, scale; v (n, 3).  Every pair of EDGE values
    as (translation, velocity) of lane x (and swapped in y, negated velocity in z), the ties of tie_rows, then random
    bit patterns and random moderate values.  The table is laid down twice, the second copy at an odd row offset, so
    every case sits in both rows of a bundle thread, in several threads of a JIT work item, and around rows 511-513.
    Rotation and scale (passive planes) hold EDGE values and random bits."""
    rng = np.random.default_rng(seed)
    rows = [(a, b) for a in EDGE for b in EDGE] + tie_rows(dt_bits)
    base = np.zeros((len(rows), 6), np.uint32)
    for i, (a, b) in enumerate(rows):
        base[i] = (a, b, a, b, a, b ^ 0x80000000)   # tx ty tz | vx vy vz
    base[:, [1, 4]] = base[:, [4, 1]]              # lane y: the pair swapped
    tv = np.zeros((n, 6), np.uint32)
    k = min(len(rows), n)
    tv[:k] = base[:k]
    start = k + 1 if k % 2 == 0 else k   # the second copy starts at an odd row
    k2 = min(len(rows), n - start)
    if k2 > 0:
        tv[start:start + k2] = base[:k2]
    rest = np.ones(n, bool)
    rest[:k] = False
    if k2 > 0:
        rest[start:start + k2] = False
    m = int(rest.sum())
    rnd = rng.integers(0, 2 ** 32, (m, 6), dtype=np.uint64).astype(np.uint32)
    mod = bits_of(r32(rng.uniform(-400.0, 400.0, (m, 6))))
    tv[rest] = np.where(rng.random((m, 1)) < 0.5, rnd, mod)
    t = np.zeros((n, 10), np.uint32)
    t[:, 0:3] = tv[:, 0:3]
    passive = np.array(EDGE, np.uint32)[rng.integers(0, len(EDGE), (n, 7))]
    t[:, 3:10] = np.where(rng.random((n, 7)) < 0.5, passive, rng.integers(0, 2 ** 32, (n, 7), dtype=np.uint64).astype(np.uint32))
    return t, tv[:, 3:6].copy()


def dt_bits_of(fps: int, frame: int) -> int:
    """Time<GgrsTime>::delta_secs of AdvanceWorld number `frame` at `fps` (time.rs:63-76; Duration::as_secs_f32)."""
    delta = frame * 10 ** 9 // fps - (frame - 1) * 10 ** 9 // fps
    secs, nanos = divmod(delta, 10 ** 9)
    return int(bits_of(r32(r32(float(secs)) + r32(r32(float(nanos)) / 1e9))))


def is_nan_bits(b) -> np.ndarray:
    b = np.asarray(b, dtype=np.uint32)
    return ((b & 0x7F800000) == 0x7F800000) & ((b & 0x007FFFFF) != 0)


def same_f32(a, b) -> np.ndarray:
    """Element-wise: identical bits, or both NaN (any payload)."""
    a, b = np.asarray(a, dtype=np.uint32), np.asarray(b, dtype=np.uint32)
    return (a == b) | (is_nan_bits(a) & is_nan_bits(b))
