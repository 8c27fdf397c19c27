"""-m gpu: checkpoints, restores and input-log replays inside the random interleavings (tests/interleave_driver.py), on
every kernel configuration of test_gpu_interleavings.py and in world batches, held to the oracle and the twin.

These entry points write or read the whole match outside the request path, so each one is where a stale host record
(passive-plane versions, content stamps and ids, the deferred live image, ring witnesses, retained frames) would skip a
store without faulting:
  - bgr_checkpoint_save of queued, retained and unheld frames, with submits in flight too: byte for byte the twin's blob
    and the oracle's (FlagsOracle.checkpoint_of, from the oracle's snapshot alone);
  - bgr_checkpoint_restore of a kept blob, mostly one from before spawns, growth or host writes, into the engine, the
    twin and the oracle (FlagsOracle.restore, from the numpy decoder), then every vector, host write and read after it;
    refused with submits pending and with one payload bit flipped, changing nothing;
  - bgr_replay of logs of 1..300 frames at every checksum interval, spawning where the registration spawns: checksums
    against FlagsOracle.replay, the replay kernel where the registration has one, the chunked fallback elsewhere (and
    with BGR_TUNE_REPLAY_POINTS=7, replays split into launches); refused past a fixed engine's capacity and with submits
    pending; then Loads of frames saved before the replay.

Replay one configuration and seed: BGR_INTERLEAVE_REPLAY=<configuration>:<seed>."""
import time
from collections import Counter

import pytest

from bevy_ggrs_b200.engine import EngineBatch
from interleave_driver import Config, Fleet, FleetConfig, Interleaving, replay_filter
from test_gpu_batch_oracle import CAPTURE, CROSS, MEMBERS, fleet_engines, registration
from test_gpu_interleavings import CONFIG_NAMES, FLAG_SETS, configs, new_engine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
MULTI_WAVE = {"bundle_multi_wave", "bundle_crossing_sides"}
SPAWNING = {"bundle_mode1_stamped", "bundle_mode1_one_wave", "bundle_multi_wave", "bundle_crossing_sides"}


def _config(name) -> Config:
    cfg = {c.name: c for c in configs()}[name]
    env = dict(cfg.env)
    if name == "nvrtc_quarter_tiles_overlapping":
        env["BGR_TUNE_REPLAY_POINTS"] = "7"   # a replay of more than 7 checksum frames runs in several launches
    # multi-wave worlds: the oracle advances every logged frame and restates every checksummed blob in Python
    return Config(**{**cfg.__dict__, "env": env, "checkpoints": True, "input_replays": True,
                     "max_log": 24 if name in MULTI_WAVE else 300, "oracle_blobs": 3 if name in MULTI_WAVE else 1_000_000})


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_checkpoints_restores_and_replays_match_the_oracle(name):
    cfg0 = _config(name)
    total, ran, t0 = Counter(), 0, time.perf_counter()
    for seed, (flags, retain) in enumerate(FLAG_SETS[:5]):
        r = replay_filter()
        if r is not None and r != (name, seed):
            continue
        cfg = Config(**{**cfg0.__dict__, "flags": flags, "retain": retain})
        drv = Interleaving(cfg, 300 + seed, new_engine(name))
        try:
            t = drv.run()
        finally:
            drv.close()
        ran += 1
        total.update(t)
        if cfg.stamped:
            assert t["stamp_rollovers"] == 1 and t["rollover_verified"] == 1, f"{name} seed {seed}: {t}"
    if not ran:
        pytest.skip("not the configuration BGR_INTERLEAVE_REPLAY selects")
    keys = ("checkpoint", "restore", "replay", "loads_across", "materialisations", "vectors", "growth")
    print(f"\n[restore / replay interleavings] {name}: {time.perf_counter() - t0:.1f} s, "
          + ", ".join(f"{k}={v}" for k, v in sorted(total.items()) if any(x in k for x in keys)))
    if ran < 5:
        return   # a replay: the tally minimums are over every seed
    replays = 4 if name in MULTI_WAVE else 8   # 40 steps: fewer draws
    minimums = {"checkpoints": 8, "checkpoints_in_flight": 1, "checkpoint_none": 1, "restores": 3, "restore_refusals": 2,
                "input_replays": replays}
    if name not in MULTI_WAVE:
        minimums["checkpoints_oracle"] = 5
    else:
        minimums["checkpoints_oracle"] = 3
    if name not in MULTI_WAVE and name != "bundle_mode2_stamped":   # a world without spawn_particles rarely grows
        minimums.update({"restores_older_rows": 1, "loads_across_replay": 1})
    if cfg0.kind in ("bundle", "generic_nvrtc"):
        minimums["input_replays_fast"] = replays
    else:
        minimums["input_replays_chunked"] = 1
    if name in SPAWNING:
        minimums["input_replays_spawning"] = 1
    missing = {k: (total[k], v) for k, v in minimums.items() if total[k] < v}
    assert not missing, f"{name}: tally below its minimum (reached, minimum): {missing}"


def _fleets():
    on = {"checkpoints": True, "input_replays": True}
    members = [Config(**{**m.__dict__, **on}) for m in MEMBERS]
    # order_base 2^32 - 700: RollbackOrdered crosses 2^32 inside tile 1 (no spawns, no growth with order_base != 0)
    crossing = [Config("", None, order_base=CROSS, **on), Config("", None, flags=CAPTURE, fps=30, order_base=CROSS, **on),
                Config("", None, retain=(2, 4), order_base=CROSS, **on)]
    return {"default_env": FleetConfig("default_env", registration(), members, steps=80, match_state=True),
            "order_base_crossing": FleetConfig("order_base_crossing", registration(), crossing, steps=80, match_state=True)}


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", ["default_env", "order_base_crossing"])
def test_batch_members_checkpoints_restores_and_replays_match_the_oracle(stream, monkeypatch, name):
    for k in ("BGR_TUNE_JIT", "BGR_TUNE_JIT_ITEM", "BGR_TUNE_JIT_ROWS"):
        monkeypatch.delenv(k, raising=False)
    fcfg = _fleets()[name]
    total, ran, t0 = Counter(), 0, time.perf_counter()
    for seed in range(3):
        r = replay_filter()
        if r is not None and r != (name, seed):
            continue
        fl = Fleet(fcfg, 300 + seed, fleet_engines(stream), EngineBatch)
        try:
            t = fl.run()
        finally:
            fl.close()
        ran += 1
        total.update(t)
    if not ran:
        pytest.skip("not the configuration BGR_INTERLEAVE_REPLAY selects")
    keys = ("checkpoint", "restore", "replay", "loads_across", "batched_calls", "cross")
    print(f"\n[restore / replay batch interleavings] {name}: {time.perf_counter() - t0:.1f} s, "
          + ", ".join(f"{k}={v}" for k, v in sorted(total.items()) if any(x in k for x in keys)))
    if ran < 3:
        return
    minimums = {"batched_calls": 20, "checkpoints": 5, "checkpoints_oracle": 3, "restores": 3, "restore_refusals": 1,
                "input_replays": 5, "batch_replays": 5, "input_replays_batched": 5, "batch_replay_refusals": 1,
                "cross_restores": 1, "cross_restore_refusals": 1, "checkpoint_none_below": 1}
    if name == "default_env":   # a growable member takes a checkpoint of more rows than its capacity
        minimums["cross_restores_grown"] = 1
    missing = {k: (total[k], v) for k, v in minimums.items() if total[k] < v}
    assert not missing, f"{name}: tally below its minimum (reached, minimum): {missing}"
