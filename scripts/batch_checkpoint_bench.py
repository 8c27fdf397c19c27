"""Batched checkpoints against the per-engine loop they replace, in one process on twin engines: host wall time of ONE
bgr_batch_checkpoint_save / bgr_batch_checkpoint_restore call over every world of a batch, and of the loop of
bgr_checkpoint_save / bgr_checkpoint_restore over the twins, alternated on every repetition.  Every repetition checks
that the batched blobs equal the loop's and that each restored world's frame digest equals its twin's.  Also a
batched seek (one batched restore of a keyframe per world, then one bgr_batch_replay of fewer than K frames) against
the single seeks (bgr_checkpoint_restore, then bgr_replay, per world), with equal checksums.

Workloads: box_game batches of 16, 256 and 1 024 worlds (2 rows each, 60 frames in), the presence world (2 000 rows)
x 256 worlds, the 15-word stress schema (the particles columns with a whole-Transform checksum, so it runs the
generic program and can be batched) at 100k rows x 8 worlds.  Median of --reps (>= 5) repetitions, in ms per call and
per world.  Prints one JSON line per workload with the card's name, power limit and max SM clock read in the same run.
`--profile` instead takes device times from torch.profiler in a run of its own: one batched save, one batched restore
and the two loops per workload after a warm-up, every kernel and copy summed by name.

    python scripts/batch_checkpoint_bench.py [--reps 5] [--only box_game,presence,stress] [--profile] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine, EngineBatch  # noqa: E402
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402

FIN = capi.BGR_HASH_FLAG_ASSERT_FINITE_F32
OPT = capi.BGR_STRATEGY_OPTIONAL
WARM_FRAMES = 60
SEEK_K = 60


def box_world(seed, stream):
    w = Engine(max_entities=2, max_depth=4, stream=stream)
    vel = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    tf = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
    w.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
    w.checksum_component(tf, 0, 12, FIN)
    w.checksum_component(vel, 0, 12)
    w.build()
    w.spawn(2)
    rng = np.random.default_rng(seed)
    t = np.zeros((2, 10), np.float32)
    t[:, 0:3] = rng.uniform(-2, 2, (2, 3)); t[:, 6] = 1.0; t[:, 7:10] = 1.0
    w.write_component(tf, 0, t)
    w.write_component(vel, 0, rng.uniform(-1, 1, (2, 3)).astype(np.float32))
    return w


def presence_world(seed, stream, n=2000):
    """Score (optional, +1 per frame), Health (optional, satsub-despawn), Tag (12 B), all checksummed."""
    w = Engine(max_entities=n, max_depth=4, stream=stream)
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = w.rollback_component("Tag", 12, capi.BGR_STRATEGY_COPY)
    for c, b in ((score, 4), (tag, 12), (health, 4)):
        w.checksum_component(c, 0, b)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(seed)
    w.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    w.write_component(health, 0, rng.integers(300, 900, n, dtype=np.uint32))
    w.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    for r in rng.choice(n, n // 5, replace=False):
        w.remove_component((score, health)[int(r) % 2], int(r))
    return w


def stress_world(seed, stream, n=100_000):
    w = Engine(max_entities=n, max_depth=4, stream=stream)
    c = register_particles(w, checksums=lambda e, t, v: (e.checksum_component(t, 0, 40, FIN), e.checksum_component(v, 0, 12)))
    w.build()
    populate(w, c, *synth_particles(n, seed, 10**6, 2 * 10**6))
    return w


def drive(batch, n_worlds, frames, seed):
    """`frames` P2P ticks of Save(f), Advance on every world of the batch, each frame confirmed one frame later."""
    rng = np.random.default_rng(seed)
    for _ in range(frames):
        f = batch.engines[0].rollback_frame_count()
        a = [int(v) for v in rng.integers(0, 16, 2)]
        info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))
        batch.handle_requests([(w, info, [Request(SAVE, f), Request(ADVANCE, 0, a)]) for w in range(n_worlds)])


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def setup(make, n_worlds):
    import torch
    s1, s2 = torch.cuda.Stream().cuda_stream, torch.cuda.Stream().cuda_stream
    batch = EngineBatch([make(i, s1) for i in range(n_worlds)])
    twins = EngineBatch([make(i, s2) for i in range(n_worlds)])
    for b in (batch, twins):
        drive(b, n_worlds, WARM_FRAMES, 1)
    return batch, twins


def digests(engines):
    return [(lambda d: (d[0].root, d[0].active))(e.frame_digest(e.rollback_frame_count())) for e in engines]


def bench(name, make, n_worlds, reps):
    batch, twins = setup(make, n_worlds)
    worlds = list(range(n_worlds))
    t_save_b, t_save_l, t_rest_b, t_rest_l = [], [], [], []
    for rep in range(reps + 1):   # repetition 0 warms up (buffer sizes, page-locked staging)
        f = batch.engines[0].rollback_frame_count() - 1   # the last Save: queued and unconfirmed
        ts, blobs = timed(lambda: batch.checkpoint([(w, f) for w in worlds]))
        tl, loop = timed(lambda: [e.checkpoint(f) for e in twins.engines])
        assert blobs == loop, "batched blobs differ from the per-engine loop's"
        src = blobs[1:] + blobs[:1]   # each world restores the next world's blob (same layout and fps)
        tr, _ = timed(lambda: batch.restore(list(zip(worlds, src))))
        tq, _ = timed(lambda: [e.restore(b) for e, b in zip(twins.engines, src)])
        assert digests(batch.engines) == digests(twins.engines), "restored worlds differ"
        drive(batch, n_worlds, 4, rep)
        drive(twins, n_worlds, 4, rep)
        if rep:
            t_save_b.append(ts); t_save_l.append(tl); t_rest_b.append(tr); t_rest_l.append(tq)
    med = lambda xs: 1e3 * statistics.median(xs)  # noqa: E731
    out = {"workload": name, "worlds": n_worlds, "rows": batch.engines[0].row_count(), "reps": reps,
           "blob_bytes": sum(len(b) for b in blobs),
           "save_batched_ms": med(t_save_b), "save_loop_ms": med(t_save_l),
           "restore_batched_ms": med(t_rest_b), "restore_loop_ms": med(t_rest_l)}
    for k in ("save_batched", "save_loop", "restore_batched", "restore_loop"):
        out[k + "_ms_per_world"] = out[k + "_ms"] / n_worlds
    out.update(seek(batch, twins, n_worlds, reps))
    return out


def seek(batch, twins, n_worlds, reps):
    """Keyframes written by a batched replay (interval SEEK_K), then each world seeks to a frame K / 2 past its
    keyframe: one batched restore + one batched replay, against per world a restore + a replay on the twins."""
    worlds = list(range(n_worlds))
    rng = np.random.default_rng(7)
    f0 = batch.engines[0].rollback_frame_count()
    log = rng.integers(0, 16, (SEEK_K * 2, 2), dtype=np.uint8)
    res = batch.replay_keyframes([(w, log, 10, SEEK_K) for w in worlds])
    kf, blob = res[0][2][-1]
    rest = log[kf - f0: kf - f0 + SEEK_K // 2]
    t_b, t_l = [], []
    for rep in range(reps + 1):
        tb, rb = timed(lambda: (batch.restore([(w, blob) for w in worlds]), batch.replay([(w, rest, 10) for w in worlds]))[1])
        tl, rl = timed(lambda: [(e.restore(blob), e.replay(rest, 10))[1] for e in twins.engines])
        assert [cs for _, cs in rb] == rl, "batched seek and single seeks disagree"
        if rep:
            t_b.append(tb); t_l.append(tl)
    return {"seek_batched_ms": 1e3 * statistics.median(t_b), "seek_loop_ms": 1e3 * statistics.median(t_l),
            "seek_frames": len(rest)}


def profile_call(name, make, n_worlds):
    """Device time of one batched save, one batched restore and the two per-engine loops (microseconds by name)."""
    import torch
    from torch.profiler import ProfilerActivity
    batch, twins = setup(make, n_worlds)
    worlds = list(range(n_worlds))
    f = batch.engines[0].rollback_frame_count() - 1
    blobs = batch.checkpoint([(w, f) for w in worlds])
    out = {"workload": name, "worlds": n_worlds}
    calls = (("save_batched", lambda: batch.checkpoint([(w, f) for w in worlds])),
             ("save_loop", lambda: [e.checkpoint(f) for e in twins.engines]),
             ("restore_batched", lambda: batch.restore(list(zip(worlds, blobs)))),
             ("restore_loop", lambda: [e.restore(b) for e, b in zip(twins.engines, blobs)]))
    for tag, fn in calls:
        fn()   # warm-up: buffer sizes, staging
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        times = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                times[e.key[:60]] = [round(e.device_time_total, 1), e.count]
        out[tag + "_device_us"] = times
        out[tag + "_device_us_total"] = round(sum(t for t, _ in times.values()), 1)
    return out


WORKLOADS = {
    "box_game": [(f"box_game_{n}", box_world, n) for n in (16, 256, 1024)],
    "presence": [("presence_2000x256", presence_world, 256)],
    "stress": [("stress_100000x8", stress_world, 8)],
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as err:  # the numbers below still say what they measured
        return {"gpu": f"unknown ({err})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="box_game,presence,stress")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if args.reps < 5:
        ap.error("--reps must be at least 5 (the medians are of at least 5 repetitions)")
    info = card()
    rows = []
    for group in args.only.split(","):
        for name, make, n in WORKLOADS[group]:
            r = profile_call(name, make, n) if args.profile else bench(name, make, n, args.reps)
            r.update(info)
            print(json.dumps(r), flush=True)
            rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
