"""-m gpu: seeded random interleavings of every engine entry point (tests/interleave_driver.py) on every kernel, held to
the oracle and to a twin engine without elisions: synchronous and queued request vectors of every shape, host writes
across segment and tile boundaries, spawns, despawns, presence edits, growth, depth and session changes, reads, feeds,
desync capture and retention.  Each configuration's seeds cover the engine flags 0, BGR_CFG_DESYNC_CAPTURE, retention,
BGR_CFG_GROWABLE and BGR_CFG_GROWABLE | BGR_CFG_DESYNC_CAPTURE, and the stamped configurations start a few launches below
the content-stamp range's end (BGR_TEST_STAMP_FIRST), so the rollover that clears the stamp table happens mid-sequence.

Replay one configuration and seed: BGR_INTERLEAVE_REPLAY=<configuration>:<seed>."""
import contextlib
import os
from collections import Counter

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.stress import synth_particles
from interleave_driver import Config, Interleaving, World, replay_filter
from schema_util import random_schema

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
OPT = capi.BGR_STRATEGY_OPTIONAL
FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
CAPTURE, GROW = capi.BGR_CFG_DESYNC_CAPTURE, capi.BGR_CFG_GROWABLE
FLAG_SETS = [(0, None), (CAPTURE, None), (0, (2, 4)), (GROW, None), (GROW | CAPTURE, None)] * 2   # seed k: FLAG_SETS[k]


def _sms() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def particles(n, spawn_rate=0, optional=False):
    """The particles schema: Transform 40 B, Velocity 12 B, Ttl 8 B, both f32 columns checksummed with the finite
    assertion (the bundle kernel's MODE 1), or Velocity and Ttl optional (MODE 2)."""
    def make(rng):
        tf, vel, ttl = synth_particles(n, int(rng.integers(1 << 20)), 2, 25, z_fraction=0.3)
        opt = OPT if optional else 0
        systems = [(capi.BGR_SYS_PARTICLES_SPAWN, [0, 1, 2], [spawn_rate, 6, 123, 0])] if spawn_rate else []
        systems += [(capi.BGR_SYS_PARTICLES_UPDATE, [0, 1], []), (capi.BGR_SYS_PARTICLES_DESPAWN, [2], [])]
        removes = [(c, int(r)) for c in (1, 2) for r in rng.choice(n, 7, replace=False)] if optional else []
        data = [np.ascontiguousarray(a).view(np.uint8).reshape(n, -1) for a in (tf, vel, ttl)]
        return World([40, 12, 8], [capi.BGR_STRATEGY_CLONE, capi.BGR_STRATEGY_COPY | opt, capi.BGR_STRATEGY_COPY | opt],
                     [(1, 0, 12, FIN), (0, 0, 12, FIN)], systems, data, removes, spawn_rate=spawn_rate, bundle=True,
                     feed_fields=[(0, 0, 12), (2, 0, 8)])
    return make


def generic(nvrtc=False):
    """A random registration (schema_util.random_schema) of 1000..2500 rows; ``nvrtc``: whole-word columns and ranges
    the generated kernel accepts."""
    def make(rng):
        if nvrtc:
            sizes = [int(x) for x in rng.choice([4, 8, 12, 16, 40], int(rng.integers(2, 5)))]
            while sum(sizes) > 96:   # at most 24 words
                sizes.pop()
            s = random_schema(rng, sizes=sizes, ranges=("none", "whole"))
        else:
            s = random_schema(rng, words=int(rng.integers(4, 20)))
        n = int(rng.integers(1000, 2500))
        strategies = [(capi.BGR_STRATEGY_COPY | OPT) if o else capi.BGR_STRATEGY_CLONE for o in s.optional]
        removes = [(c, int(r)) for c, o in enumerate(s.optional) if o for r in rng.choice(n, 9, replace=False)]
        feed = [(c, 0, min(8, sz)) for c, sz in enumerate(s.sizes) if sz % 4 == 0][:3]   # whole words only
        return World(s.sizes, strategies, [(c, off, ln, 0) for c, off, ln in s.cks], s.systems, s.values(rng, n), removes,
                     feed_fields=feed)
    return make


def configs():
    one_wave = 3 * _sms() * 512   # rows of the largest grid that runs as one wave (run_fused: PF_PASSIVE_EARLY, no stamps)
    early0 = {"BGR_TUNE_PASSIVE_EARLY": "0"}
    return [
        Config("bundle_mode1_stamped", particles(5000, spawn_rate=37), env=early0, kind="bundle", stamped=True,
               grow_margin=16384),
        Config("bundle_mode1_one_wave", particles(3000, spawn_rate=37), kind="bundle", grow_margin=16384),
        Config("bundle_mode2_stamped", particles(4000, optional=True), env=early0, kind="bundle", stamped=True),
        Config("bundle_multi_wave", particles(one_wave + 300, spawn_rate=300), kind="bundle", stamped=True, steps=40,
               digests=2, grow_margin=32768),
        # starts one wave (no stamps); spawns take it to several waves and rollbacks bring it back: every change to the
        # stamped side clears the table the launches without stamps left stale
        Config("bundle_crossing_sides", particles(one_wave - 200, spawn_rate=300), kind="bundle", steps=40, digests=2,
               grow_margin=32768),
        Config("interpreter", generic(), env={"BGR_TUNE_JIT": "0"}, kind="generic_interpreter"),
        Config("nvrtc_whole_tiles", generic(nvrtc=True), env={"BGR_TUNE_JIT": "2", "BGR_TUNE_JIT_ITEM": "512"},
               kind="generic_nvrtc"),
        Config("nvrtc_quarter_tiles_overlapping", generic(nvrtc=True), env={"BGR_TUNE_JIT": "2", "BGR_TUNE_JIT_TILEDEP": "1"},
               kind="generic_nvrtc"),
        Config("stepwise_tma", generic(), env={"BGR_TUNE_TMA": "1"}, kind="stepwise_tma"),
        Config("stepwise_flat", generic(), env={"BGR_TUNE_TMA": "0"}, kind="stepwise_flat"),
    ]


CONFIG_NAMES = ["bundle_mode1_stamped", "bundle_mode1_one_wave", "bundle_mode2_stamped", "bundle_multi_wave",
                "bundle_crossing_sides", "interpreter",
                "nvrtc_whole_tiles", "nvrtc_quarter_tiles_overlapping", "stepwise_tma", "stepwise_flat"]
STEPWISE = {"stepwise_tma", "stepwise_flat"}


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


def new_engine(name):
    def make(role, max_entities, flags, env, fps=60, order_base=0):
        if name in STEPWISE:
            flags |= capi.BGR_CFG_FORCE_STEPWISE
        with _env(env):   # read once, at bgr_engine_create
            return Engine(max_entities=max_entities, max_depth=9, fps=fps, flags=flags, order_base=order_base)
    return make


def _selected(name, seed):
    r = replay_filter()
    return r is None or r == (name, seed)


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_random_interleavings_match_the_oracle_and_the_twin(name):
    cfg0 = {c.name: c for c in configs()}[name]
    total = Counter()
    ran = 0
    for seed, (flags, retain) in enumerate(FLAG_SETS):
        if not _selected(name, seed):
            continue
        cfg = Config(**{**cfg0.__dict__, "flags": flags, "retain": retain})
        drv = Interleaving(cfg, seed, new_engine(name))
        try:
            t = drv.run()
        finally:
            drv.close()
        ran += 1
        depth = max(total["max_queue_depth"], t["max_queue_depth"])
        total.update(t)
        total["max_queue_depth"] = depth
        if cfg.stamped:   # predicted once by the driver, and seen in the launch trace at that launch
            assert t["stamp_rollovers"] == 1 and t["rollover_verified"] == 1, f"{name} seed {seed}: {t}"
    if not ran:
        pytest.skip("not the configuration BGR_INTERLEAVE_REPLAY selects")
    print(f"\n[interleavings] {name}: " + ", ".join(f"{k}={v}" for k, v in sorted(total.items())))
    if ran < len(FLAG_SETS):
        return   # a replay: the tally minimums are over every seed
    minimums = {"vectors": 60, "vectors_queued": 10, "queue_depth_4": 1, "vectors_long": 1, "invalid_rollbacks": 1,
                "refusals": 1, "band_writes": 3, "despawns": 1, "live_reads": 3, "peeks": 3, "feed_reports": 3,
                "feed_cap_hit": 1, "capture_reads": 1, "digests": 1, "exports": 1, "witnesses_released": 1,
                "retained_released": 1, "growth_steps": 1, "reserves": 1}
    if name not in STEPWISE:
        minimums.update({"deferred": 3, "from_deferred": 1, "materialisations": 1})
    if cfg0.stamped:
        minimums.update({"stamped_launches": 10})
    if cfg0.kind == "bundle" and name != "bundle_mode2_stamped":   # spawn_particles registered
        minimums.update({"queued_tile_crossings": 1})
    if name == "bundle_crossing_sides":
        minimums.update({"stale_table_clears": 1})
    if name.startswith("bundle_mode1"):
        minimums.update({"startup_systems": 1})
    missing = {k: (total[k], v) for k, v in minimums.items() if total[k] < v}
    assert not missing, f"{name}: tally below its minimum (reached, minimum): {missing}"
