"""The stress-test schema and synthetic populations of BASELINE.md (examples/stress_tests/particles.rs).

Registered columns (particles.rs:191-200, render-only types excluded — SURVEY.md §8):
    Transform  40 B  = translation 3xf32 | rotation 4xf32 | scale 3xf32   rollback_component_with_clone
    Velocity   12 B  = Vec3                                               rollback_component_with_copy
    Ttl         8 B  = usize                                              rollback_component_with_copy
Checksums (particles.rs:107-120, 205-222): Velocity and Transform.translation, `to_bits` of x,y,z,
both asserting is_finite.  GgrsSchedule systems: update_particles, despawn_particles (:233-240).
"""
from __future__ import annotations

import numpy as np

from . import capi

TRANSFORM_BYTES, VELOCITY_BYTES, TTL_BYTES = 40, 12, 8
SLOT_BYTES_PER_ENTITY = TRANSFORM_BYTES + VELOCITY_BYTES + TTL_BYTES + 1  # + alive byte


def register_particles(world, spawn_rate: int = 0, spawn_ttl: int = 300, rng_seed: int = 123, checksums=None):
    """Same registration sequence as the example's main() on any Engine-shaped backend.
    spawn_rate > 0 also registers spawn_particles.run_if(spawn_pressed) with ParticleRng(seed_from_u64(rng_seed))
    (particles.rs:233-243; `--rate`, ttl = fps * 5).
    checksums(world, transform, velocity) replaces the example's two checksum registrations (other setups of the
    same world: one column, none, no finite assertion)."""
    t = world.rollback_component("Transform", TRANSFORM_BYTES, capi.BGR_STRATEGY_CLONE)
    v = world.rollback_component("Velocity", VELOCITY_BYTES, capi.BGR_STRATEGY_COPY)
    l = world.rollback_component("Ttl", TTL_BYTES, capi.BGR_STRATEGY_COPY)
    if checksums is not None:
        checksums(world, t, v)
    else:
        world.checksum_component(v, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)   # checksum_component_with_hash::<Velocity>()
        world.checksum_component(t, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)   # checksum_component::<Transform>(translation bits)
    if spawn_rate:
        world.add_system(capi.BGR_SYS_PARTICLES_SPAWN, [t, v, l],
                         [spawn_rate, spawn_ttl, rng_seed & 0xFFFFFFFF, (rng_seed >> 32) & 0xFFFFFFFF])
    world.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
    world.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
    return t, v, l


def synth_particles(n: int, seed: int, ttl_lo: int, ttl_hi: int, z_fraction: float = 0.0):
    """Seeded synthetic population: translation x,y ~ U(-360,360), velocity x,y ~ U(-200,200)
    (particles.rs:259,265), z = 0, identity rotation, unit scale, ttl ~ U{ttl_lo..ttl_hi}.
    z_fraction > 0 gives that share of the rows a non-zero z translation and velocity (the example itself is
    2-D; used by tests to exercise the general hash path next to the z == 0 fast path)."""
    rng = np.random.default_rng(seed)
    tf = np.zeros((n, 10), dtype=np.float32)
    tf[:, 0:2] = rng.uniform(-360.0, 360.0, size=(n, 2)).astype(np.float32)
    tf[:, 6] = 1.0            # rotation = (0,0,0,1)
    tf[:, 7:10] = 1.0         # scale = (1,1,1)
    vel = np.zeros((n, 3), dtype=np.float32)
    vel[:, 0:2] = rng.uniform(-200.0, 200.0, size=(n, 2)).astype(np.float32)
    ttl = rng.integers(ttl_lo, ttl_hi + 1, size=n, dtype=np.uint64)
    if z_fraction > 0:
        pick = rng.random(n) < z_fraction
        tf[pick, 2] = rng.uniform(-50.0, 50.0, size=int(pick.sum())).astype(np.float32)
        vel[pick, 2] = rng.uniform(-20.0, 20.0, size=int(pick.sum())).astype(np.float32)
    return tf, vel, ttl


def populate(world, cols, tf, vel, ttl, chunk: int = 1 << 20):
    t, v, l = cols
    n = tf.shape[0]
    first = world.spawn(n)
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        world.write_component(t, first + a, tf[a:b])
        world.write_component(v, first + a, vel[a:b])
        world.write_component(l, first + a, ttl[a:b])
    return first
