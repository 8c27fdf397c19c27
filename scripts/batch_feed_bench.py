"""Batched change-feed reports against the loop of single reports they replace, in one process on twin batches: per
tick, one batched tick (bgr_batch_handle_requests over every world) followed either by ONE bgr_batch_feed_begin /
bgr_batch_feed_wait over every world's feed, or by the single reports of the twins (every bgr_feed_begin, then every
bgr_feed_wait: the best a caller could do without the batched call).  The two alternate on every repetition and the
records of every world are compared every time.  Each world's feed tracks every row (cap = its rows).

Workloads: box_game batches of 16, 256 and 1 024 worlds (2 rows each), the presence world (2 000 rows) x 256 worlds,
the 15-word stress schema at 100k rows x 8 worlds (the world makers of batch_checkpoint_bench.py).  Host wall time per
tick (tick + report) and of the report alone, median of --reps (>= 5) repetitions, in ms.  Prints one JSON line per
workload with the card's name, power limit and max SM clock read in the same run.  `--profile` instead takes the
device time of one batched report and of one loop from torch.profiler in a run of its own, every kernel and copy
summed by name.

    python scripts/batch_feed_bench.py [--reps 5] [--only box_game,presence,stress] [--profile] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import EngineBatch  # noqa: E402
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request  # noqa: E402
from batch_checkpoint_bench import box_world, card, presence_world, stress_world  # noqa: E402

WARM_FRAMES = 8

# the fields each workload's feed tracks: (column, byte_offset, byte_len)
FIELDS = {
    box_world: [(1, 0, 12), (0, 0, 12)],                 # Transform.translation, Velocity
    presence_world: [(0, 0, 4), (2, 4, 8), (1, 0, 4)],   # Score (optional), a part of Tag, Health (optional)
    stress_world: [(0, 0, 12), (1, 0, 8)],               # Transform.translation, Velocity.xy
}


def tick(batch, n_worlds, rng):
    f = batch.engines[0].rollback_frame_count()
    a = [int(v) for v in rng.integers(0, 16, 2)]
    info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))
    batch.handle_requests([(w, info, [Request(SAVE, f), Request(ADVANCE, 0, a)]) for w in range(n_worlds)])


class Side:
    """A batch whose every world has one feed, reported batched (one call) or by the loop of single reports."""

    def __init__(self, make, n_worlds, stream):
        self.batch = EngineBatch([make(i, stream) for i in range(n_worlds)])
        fields = FIELDS[make]
        self.feeds = [e.feed_create(fields) for e in self.batch.engines]
        self.caps = [e.max_entities for e in self.batch.engines]
        self.calls = [(w, f, c) for w, (f, c) in enumerate(zip(self.feeds, self.caps))]
        self.buf = self.batch.feed_alloc(self.calls)
        self.bufs = [e.feed_alloc(f, c) for e, f, c in zip(self.batch.engines, self.feeds, self.caps)]

    def batched(self):
        return self.batch.feed_wait(self.batch.feed_begin(self.calls, self.buf))

    def loop(self):
        tickets = [e.feed_begin(f, b, c) for e, f, b, c in zip(self.batch.engines, self.feeds, self.bufs, self.caps)]
        return [e.feed_wait(t) for e, t in zip(self.batch.engines, tickets)]


def setup(make, n_worlds):
    import torch
    sides = [Side(make, n_worlds, torch.cuda.Stream().cuda_stream) for _ in range(2)]
    for s in sides:
        rng = np.random.default_rng(1)
        for _ in range(WARM_FRAMES):
            tick(s.batch, n_worlds, rng)
        s.loop()   # the first report lists every row: out of the timed window
    return sides


def same(a, b):
    return all(ra.tobytes() == rb.tobytes() and ia == ib for (ra, ia), (rb, ib) in zip(a, b)) and len(a) == len(b)


def bench(name, make, n_worlds, reps):
    batched, looped = setup(make, n_worlds)
    t_tb, t_rb, t_tl, t_rl = [], [], [], []
    records = 0
    for rep in range(reps + 1):   # repetition 0 warms up (staging sizes)
        seed = 100 + rep
        order = (batched, looped) if rep % 2 else (looped, batched)
        res = {}
        for side in order:
            rng = np.random.default_rng(seed)
            t0 = time.perf_counter()
            tick(side.batch, n_worlds, rng)
            t1 = time.perf_counter()
            res[id(side)] = side.batched() if side is batched else side.loop()
            t2 = time.perf_counter()
            if rep:
                (t_tb if side is batched else t_tl).append(t2 - t0)
                (t_rb if side is batched else t_rl).append(t2 - t1)
        assert same(res[id(batched)], res[id(looped)]), f"{name}: batched records differ from the single reports'"
        records = sum(info.n_records for _, info in res[id(batched)])
    med = lambda xs: 1e3 * statistics.median(xs)  # noqa: E731
    return {"workload": name, "worlds": n_worlds, "rows": batched.batch.engines[0].row_count(), "reps": reps,
            "records_per_report": records,
            "tick_and_batched_report_ms": med(t_tb), "tick_and_single_reports_ms": med(t_tl),
            "batched_report_ms": med(t_rb), "single_reports_ms": med(t_rl)}


def profile_call(name, make, n_worlds):
    """Device time of one batched report and of one loop of single reports (microseconds by kernel / copy name)."""
    import torch
    from torch.profiler import ProfilerActivity
    batched, looped = setup(make, n_worlds)
    out = {"workload": name, "worlds": n_worlds}
    for tag, side in (("batched", batched), ("single", looped)):
        tick(side.batch, n_worlds, np.random.default_rng(5))
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            side.batched() if side is batched else side.loop()
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
