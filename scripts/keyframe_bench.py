"""Replay keyframes against the two things they replace or extend, in one process on twin engines: host wall time of ONE
keyframe replay call (bgr_replay_keyframes / bgr_batch_replay_keyframes), of a plain replay of the same log (bgr_replay
/ bgr_batch_replay), and of the status-quo way to get the same blobs: the log split at every keyframe, each segment
replayed (batched across the worlds), then per world bgr_save_world and bgr_checkpoint_save.  The status quo's blobs
must equal the keyframe replay's.  Also times one seek: bgr_checkpoint_restore of a keyframe, then a replay of K - 1
frames.  The status quo of the 256- and 1 024-world batches is timed on their first 16 worlds only (it is one engine
call per world and keyframe) and reported per world.

Workloads: batches of 1, 16, 256 and 1 024 box_game matches x 3 600 frames at K = 60 and 600; one spawning particles
world (2 000 rows, a spawn every 60 frames) x 3 600 frames at K = 60; the stress schema at 100k and 1M rows x 600
frames at K = 60.  Checksums at the examples' interval of 10.  Prints one JSON line per workload, with the card's name,
power limit and max SM clock read in the same run.  `--profile` instead takes device times from torch.profiler in a run
of its own (tracing slows the host): one keyframe replay call and one plain replay call per workload after a warm-up
call, every kernel and copy summed by name.

    python scripts/keyframe_bench.py [--reps 3] [--only box_game,particles,stress] [--profile] [--out results.json]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine, EngineBatch  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402
from replay_bench import box_world  # noqa: E402

K_CHECKSUM = 10
STATUS_QUO_WORLDS = 16


def particles_world(n, rate, ttl, stream):
    """replay_bench.py's worlds, on a batch's stream: spawning particles (rate > 0) or the stress schema."""
    w = Engine(max_entities=n + rate * 64 * 8, max_depth=4, stream=stream)
    c = register_particles(w, spawn_rate=rate) if rate else register_particles(w)
    w.build()
    populate(w, c, *synth_particles(n, 1, *ttl))
    return w


class OneWorld:
    """EngineBatch's replay calls on one engine: the particles bundle's registrations cannot be batched."""
    def __init__(self, e):
        self.engines = [e]

    def replay(self, calls):
        return [(capi.BGR_OK, self.engines[0].replay(x, k)) for _, x, k in calls]

    def replay_keyframes(self, calls):
        return [(capi.BGR_OK, *self.engines[0].replay_keyframes(x, k, kk)) for _, x, k, kk in calls]


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def status_quo(batch, worlds, log, kk):
    """The keyframes of `log` the way a caller gets them without bgr_replay_keyframes."""
    blobs = [[] for _ in worlds]
    f0 = batch.engines[worlds[0]].rollback_frame_count()
    at = 0
    for j in range(len(log)):
        if (f0 + j) % kk:
            continue
        if j > at:
            batch.replay([(w, log[at:j], K_CHECKSUM) for w in worlds])
            at = j
        for i, w in enumerate(worlds):
            e = batch.engines[w]
            e.save_world()
            blobs[i].append((f0 + j, e.checkpoint(f0 + j)))
            e.confirm(f0 + j)  # the ring may release the frame: it holds at most max_depth unconfirmed ones
    if at < len(log):
        batch.replay([(w, log[at:], K_CHECKSUM) for w in worlds])
    return blobs


def bench(name, make, n_worlds, frames, kk, reps, spawn_every=0, batched=True):
    import torch
    stream = torch.cuda.Stream().cuda_stream
    group = (lambda es: EngineBatch(es)) if batched else (lambda es: OneWorld(es[0]))
    kfb, plain, sq = (group([make(i, stream) for i in range(n_worlds)]) for _ in range(3))
    sq_worlds = list(range(min(n_worlds, STATUS_QUO_WORLDS)))
    seeker = make(0, None)  # restores a keyframe of world 0 and replays to a frame after it
    rng = np.random.default_rng(0)
    t_kf, t_plain, t_sq, t_seek = [], [], [], []
    for rep in range(reps + 1):
        log = rng.integers(0, 16, (frames, 2), dtype=np.uint8)
        if spawn_every:
            log[::spawn_every, 0] |= capi.BGR_INPUT_SPAWN
        f0 = kfb.engines[0].rollback_frame_count()
        t1, ra = timed(lambda: kfb.replay_keyframes([(w, log, K_CHECKSUM, kk) for w in range(n_worlds)]))
        t2, rb = timed(lambda: plain.replay([(w, log, K_CHECKSUM) for w in range(n_worlds)]))
        t3, rc = timed(lambda: status_quo(sq, sq_worlds, log, kk))
        assert [cs for _, cs, _ in ra] == [cs for _, cs in rb], "keyframe replay and plain replay disagree"
        assert [kfs for _, _, kfs in ra[:len(sq_worlds)]] == rc, "keyframe blobs and the status quo's differ"
        assert kfb.engines[0].last_kernel().replay
        f, blob = ra[0][2][len(ra[0][2]) // 2]
        seg = log[f - f0: f - f0 + kk - 1]
        t4, _ = timed(lambda: (seeker.restore(blob), seeker.replay(seg, K_CHECKSUM)))
        if rep:
            t_kf.append(t1); t_plain.append(t2); t_sq.append(t3); t_seek.append(t4)
        n_kf = len(ra[0][2])
        blob_bytes = sum(len(x) for _, _, kfs in ra for _, x in kfs)
    med = lambda xs: 1e3 * statistics.median(xs)  # noqa: E731
    return {"workload": name, "worlds": n_worlds, "rows": kfb.engines[0].row_count(), "frames": frames,
            "keyframe_interval": kk, "keyframes_per_world": n_kf, "blob_bytes": blob_bytes,
            "keyframe_replay_ms": med(t_kf), "plain_replay_ms": med(t_plain),
            "keyframe_cost": statistics.median(t_kf) / statistics.median(t_plain),
            "status_quo_worlds": len(sq_worlds), "status_quo_ms": med(t_sq),
            "status_quo_ms_per_world": med(t_sq) / len(sq_worlds), "keyframe_ms_per_world": med(t_kf) / n_worlds,
            "seek_ms": med(t_seek)}


def profile_call(name, make, n_worlds, frames, kk, spawn_every=0, batched=True):
    """Device time of one keyframe replay call and one plain replay call, by kernel and copy name (microseconds)."""
    import torch
    from torch.profiler import ProfilerActivity
    stream = torch.cuda.Stream().cuda_stream
    group = (lambda es: EngineBatch(es)) if batched else (lambda es: OneWorld(es[0]))
    kfb, plain = (group([make(i, stream) for i in range(n_worlds)]) for _ in range(2))
    rng = np.random.default_rng(0)
    out = {"workload": name, "worlds": n_worlds, "frames": frames, "keyframe_interval": kk}
    for rep in range(2):  # the first call compiles the generated kernel and sizes the buffers
        log = rng.integers(0, 16, (frames, 2), dtype=np.uint8)
        if spawn_every:
            log[::spawn_every, 0] |= capi.BGR_INPUT_SPAWN
        for tag, fn in (("keyframe", lambda: kfb.replay_keyframes([(w, log, K_CHECKSUM, kk) for w in range(n_worlds)])),
                        ("plain", lambda: plain.replay([(w, log, K_CHECKSUM) for w in range(n_worlds)]))):
            if not rep:
                fn()
                continue
            with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            times = {}
            for e in prof.key_averages():
                if e.device_time_total > 0:
                    times[e.key[:60]] = round(e.device_time_total, 1)
            out[tag + "_device_us"] = times
            out[tag + "_device_us_total"] = round(sum(times.values()), 1)
    return out


def profiles(only):
    out = []
    if "box_game" in only:
        out += [lambda n=n, kk=kk: profile_call(f"box_game_{n}_k{kk}", lambda i, s: box_world(i, s), n, 3600, kk)
                for n, kk in ((16, 60), (1024, 60), (1024, 600))]
    if "stress" in only:
        out.append(lambda: profile_call("stress_1000000_k60", lambda i, s: particles_world(10**6, 0, (10**6, 2 * 10**6), s),
                                        1, 600, 60, batched=False))
    return out


def workloads(reps, only):
    out = []
    if "box_game" in only:
        for n in (1, 16, 256, 1024):
            for kk in (60, 600):
                out.append(lambda n=n, kk=kk: bench(f"box_game_{n}_k{kk}", lambda i, s: box_world(i, s), n, 3600, kk, reps))
    if "particles" in only:
        out.append(lambda: bench("particles_2000_k60", lambda i, s: particles_world(2000, 5, (60, 300), s), 1, 3600, 60, reps, 60, batched=False))
    if "stress" in only:
        for n in (100_000, 1_000_000):
            out.append(lambda n=n: bench(f"stress_{n}_k60", lambda i, s: particles_world(n, 0, (10**6, 2 * 10**6), s), 1, 600, 60, reps, batched=False))
    return out


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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="box_game,particles,stress")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    info = card()
    rows = []
    only = args.only.split(",")
    for w in (profiles(only) if args.profile else workloads(args.reps, only)):
        r = dict(w(), **info)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
