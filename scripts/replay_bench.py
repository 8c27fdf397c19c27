"""Replays against the request stream they stand for: host wall time of ONE replay call (bgr_replay / bgr_batch_replay)
versus the same frames as request vectors of at most 80 requests ([Save at the checksum frames, Advance] under a
spectator session, whose depth-0 ring makes every Save a checksum without a store), on twin engines in one process,
alternating, with the checksums of both compared on every repetition.  `--profile` instead measures the replay
kernel's device time with torch.profiler (a run of its own: tracing slows the host).

Workloads, the sizes the replay serves: batches of N box_game matches (2 entities) x 3 600 frames (a minute at
60 fps) at the examples' desync-detection interval of 10, as a service re-simulating uploaded matches runs them; one
spawning particles world (2 000 rows, a spawn every 60 frames) x 3 600 frames; the stress schema at 100k and 1M rows x
600 frames at intervals 10 and 1.  Prints one JSON line per workload, with the card's name and power limit read in the
same run.

    python scripts/replay_bench.py [--reps 5] [--only box_game,particles,stress] [--profile] [--out results.json]
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

SPECTATOR = (capi.BGR_SESSION_SPECTATOR, 0, 0, 0)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def box_world(seed, stream=None):
    w = Engine(max_entities=2, max_depth=4, stream=stream)
    vel = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY)
    tf = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
    w.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
    w.checksum_component(tf, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
    w.checksum_component(vel, 0, 12)
    w.build()
    w.spawn(2)
    rng = np.random.default_rng(seed)
    t = np.zeros((2, 10), np.float32)
    t[:, 0:3] = rng.uniform(-2, 2, (2, 3)); t[:, 6] = 1.0; t[:, 7:10] = 1.0
    w.write_component(tf, 0, t)
    return w


def particles_world(n, rate, reps):
    w = Engine(max_entities=n + rate * 64 * (reps + 2), max_depth=4)
    c = register_particles(w, spawn_rate=rate)
    w.build()
    populate(w, c, *synth_particles(n, 1, 60, 300))
    return w


def stress_world(n):
    w = Engine(max_entities=n, max_depth=4)
    c = register_particles(w)
    w.build()
    populate(w, c, *synth_particles(n, 1, 10**6, 2 * 10**6))
    return w


def stream_vectors(f0, log, k):
    vecs, cur = [], []
    for j, row in enumerate(log):
        reqs = ([Request(SAVE, f0 + j)] if k and (f0 + j) % k == 0 else []) + [Request(ADVANCE, 0, [int(v) for v in row])]
        if len(cur) + len(reqs) > capi.BGR_MAX_REQUESTS:
            vecs.append(cur)
            cur = []
        cur += reqs
    return vecs + ([cur] if cur else [])


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def bench_batch(n_worlds, frames, k, reps):
    import torch
    stream = torch.cuda.Stream().cuda_stream
    a = EngineBatch([box_world(i, stream) for i in range(n_worlds)])
    b = EngineBatch([box_world(i, stream) for i in range(n_worlds)])
    rng = np.random.default_rng(0)
    one, chunked, calls = [], [], 0
    for rep in range(reps + 1):
        log = rng.integers(0, 16, (frames, 2), dtype=np.uint8)
        f0 = a.engines[0].rollback_frame_count()
        t1, ra = timed(lambda: a.replay([(w, log, k) for w in range(n_worlds)]))
        vecs = stream_vectors(f0, log, k)
        calls = len(vecs)

        def run_chunked():
            res = [[] for _ in range(n_worlds)]
            for v in vecs:
                for w, (st, cs) in enumerate(b.handle_requests([(w, SPECTATOR, v) for w in range(n_worlds)])):
                    res[w] += cs
            return res
        t2, rb = timed(run_chunked)
        assert [cs for _, cs in ra] == rb, "replay and request stream disagree"
        assert a.engines[0].last_kernel().replay
        if rep:
            one.append(t1)
            chunked.append(t2)
    return {"workload": f"box_game_batch_{n_worlds}", "frames": frames, "interval": k, "calls_chunked": calls,
            "replay_ms": 1e3 * statistics.median(one), "chunked_ms": 1e3 * statistics.median(chunked),
            "speedup": statistics.median(chunked) / statistics.median(one)}


def bench_single(name, make, frames, k, reps, spawn_every=0):
    a, b = make(), make()
    rng = np.random.default_rng(1)
    one, chunked = [], []
    for rep in range(reps + 1):
        log = rng.integers(0, 16, (frames, 2), dtype=np.uint8)
        if spawn_every:
            log[::spawn_every, 0] |= capi.BGR_INPUT_SPAWN
        f0 = a.rollback_frame_count()
        t1, ca = timed(lambda: a.replay(log, k))
        vecs = stream_vectors(f0, log, k)
        t2, cb = timed(lambda: [cs for v in vecs for cs in b.handle_requests(SPECTATOR, v)])
        assert ca == cb, "replay and request stream disagree"
        assert a.last_kernel().replay
        if rep:
            one.append(t1)
            chunked.append(t2)
    return {"workload": name, "rows": a.row_count(), "frames": frames, "interval": k, "calls_chunked": len(vecs),
            "replay_ms": 1e3 * statistics.median(one), "chunked_ms": 1e3 * statistics.median(chunked),
            "speedup": statistics.median(chunked) / statistics.median(one)}


def workloads(reps, only):
    out = []
    if "box_game" in only:
        out += [lambda n=n: bench_batch(n, 3600, 10, reps) for n in (1, 16, 256, 1024)]
    if "particles" in only:
        out.append(lambda: bench_single("particles_spawning_2000", lambda: particles_world(2000, 5, reps), 3600, 10, reps, 60))
    if "stress" in only:
        out += [lambda n=n, k=k: bench_single(f"stress_{n}_k{k}", lambda: stress_world(n), 600, k, reps)
                for n in (100_000, 1_000_000) for k in (10, 1)]
    return out


def profile(reps, only):
    """Device time of the replay kernel per replay call, from torch.profiler (a run of its own)."""
    import torch
    from torch.profiler import ProfilerActivity
    res = []
    for fn in workloads(1, only):
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            r = fn()
        ev = [e for e in prof.key_averages() if "k_generic_jit_replay" in e.key]
        total_us = sum(e.device_time_total for e in ev) if ev else 0.0
        calls = sum(e.count for e in ev) if ev else 0
        res.append({"workload": r["workload"], "interval": r["interval"], "replay_kernel_launches": calls,
                    "replay_kernel_us_per_launch": total_us / max(1, calls)})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="box_game,particles,stress")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    only = set(a.only.split(","))
    info = card()
    rows = profile(a.reps, only) if a.profile else [fn() for fn in workloads(a.reps, only)]
    for r in rows:
        r.update(info)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
