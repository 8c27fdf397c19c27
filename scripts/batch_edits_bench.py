"""Batched host edits against the loop of single calls they replace, in one process on twin batches: per tick, the edits
of every world, either as ONE bgr_batch_apply_edits or as one bgr_apply_edits per world (the status quo), and one
batched tick (bgr_batch_handle_requests over every world).  The two ways alternate on every repetition and the live
state of every world (row count, alive bytes, every column) is compared every time.

Each world gets K field writes per tick (K = 1 or 16, Transform.translation on box_game, Score and a part of Tag on the
presence world, at rows drawn per world) and, every fourth tick, one spawned row that its records then write.
Workloads: box_game batches of 16, 256 and 1 024 worlds (2 rows each), the presence world (2 000 rows) x 256 worlds.

Reported per workload and K, medians of --reps (>= 5) repetitions of --ticks ticks each, in ms per tick:
  - pipelined: the edit call(s) then the tick, without waiting in between (what a server does); the edit step is the
    host time of the edit call(s), which return without waiting for the GPU;
  - synchronised: the edit call(s), a stream synchronise, then the tick; the edit step includes the synchronise, so it
    is the edits' own end-to-end time.
Prints one JSON line per row with the card's name, power limit and max SM clock read in the same run.  `--profile`
instead takes the device time of one batched edit call and of one loop from torch.profiler in a run of its own.

    python scripts/batch_edits_bench.py [--reps 5] [--ticks 8] [--only box_game,presence] [--profile] [--out f.json]
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
from bevy_ggrs_b200.engine import EDIT_DTYPE, Engine, EngineBatch  # noqa: E402
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request  # noqa: E402
from batch_checkpoint_bench import FIN, card  # noqa: E402

OPT = capi.BGR_STRATEGY_OPTIONAL
WARM_TICKS = 4
SPAWN_EVERY = 4
HEADROOM = 256   # rows the spawns may add


def box_world(seed, stream):
    """box_game (batch_checkpoint_bench.box_world) with room for spawned rows."""
    w = Engine(max_entities=2 + HEADROOM, max_depth=4, stream=stream)
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
    """batch_checkpoint_bench.presence_world with room for spawned rows."""
    w = Engine(max_entities=n + HEADROOM, max_depth=4, stream=stream)
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


# the fields each workload's records write: (column, byte_offset, byte_len)
FIELDS = {box_world: [(1, 0, 12)], presence_world: [(0, 0, 4), (2, 4, 8)]}
COLUMNS = {box_world: [0, 1], presence_world: [0, 1, 2]}


def edits(make, rows, k, spawn, rng):
    """One world's records for one tick: k field writes at rows drawn below `rows`, then (spawn) one spawned row and a
    write of it."""
    recs, values = [], bytearray()
    fields = FIELDS[make]

    def write(row, field):
        c, off, ln = field
        recs.append((capi.BGR_EDIT_WRITE, c, row, 1, off, ln, len(values), 0))
        values.extend(rng.uniform(-2, 2, ln // 4).astype(np.float32).tobytes())

    for j in range(k):
        write(int(rng.integers(0, rows)), fields[j % len(fields)])
    if spawn:
        recs.append((capi.BGR_EDIT_SPAWN, 0, 0, 1, 0, 0, 0, 0))
        write(rows, fields[0])
    return np.array(recs, dtype=EDIT_DTYPE), bytes(values)


class Side:
    def __init__(self, make, n_worlds, stream):
        self.make = make
        self.batch = EngineBatch([make(i, stream) for i in range(n_worlds)])
        self.n = n_worlds

    def draw(self, k, spawn, rng):
        return [(w, *edits(self.make, e.row_count(), k, spawn, rng)) for w, e in enumerate(self.batch.engines)]

    def apply(self, calls, batched):
        if batched:
            self.batch.apply_edits(calls)
        else:
            for w, x, v in calls:
                self.batch.engines[w].apply_edits(x, v)

    def tick(self, rng):
        f = self.batch.engines[0].rollback_frame_count()
        a = [int(v) for v in rng.integers(0, 16, 2)]
        info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))
        self.batch.handle_requests([(w, info, [Request(SAVE, f), Request(ADVANCE, 0, a)]) for w in range(self.n)])

    def state(self):
        out = []
        for e in self.batch.engines:
            n = e.row_count()
            out.append((n, e.read_alive(0, n).tobytes(), tuple(e.read_component(c, 0, n).tobytes() for c in COLUMNS[self.make])))
        return out


def run_ticks(side, batched, k, ticks, t0_tick, seed, synchronise):
    """`ticks` ticks of edits then tick; returns (edit step s, whole tick s) summed over them."""
    rng = np.random.default_rng(seed)
    edit_s = total_s = 0.0
    for t in range(ticks):
        calls = side.draw(k, (t0_tick + t) % SPAWN_EVERY == 0, rng)
        t0 = time.perf_counter()
        side.apply(calls, batched)
        if synchronise:
            side.batch.engines[0].synchronize()
        t1 = time.perf_counter()
        side.tick(rng)
        t2 = time.perf_counter()
        edit_s += t1 - t0
        total_s += t2 - t0
    return edit_s, total_s


def setup(make, n_worlds):
    import torch
    sides = [Side(make, n_worlds, torch.cuda.Stream().cuda_stream) for _ in range(2)]
    for s, batched in zip(sides, (True, False)):
        run_ticks(s, batched, 16, WARM_TICKS, 1, 7, False)   # staging sizes, module loads
    return sides


def bench(name, make, n_worlds, k, reps, ticks):
    batched, looped = setup(make, n_worlds)
    times = {key: [] for key in ("b_edit_p", "b_tick_p", "l_edit_p", "l_tick_p", "b_edit_s", "b_tick_s", "l_edit_s", "l_tick_s")}
    tick_no = 1 + WARM_TICKS
    for rep in range(reps):
        for sync in (False, True):
            seed = 1000 * rep + sync
            order = (batched, looped) if rep % 2 else (looped, batched)
            for side in order:
                e, t = run_ticks(side, side is batched, k, ticks, tick_no, seed, sync)
                tag = ("b" if side is batched else "l") + "_edit" + ("_s" if sync else "_p")
                times[tag].append(e / ticks)
                times[tag.replace("_edit", "_tick")].append(t / ticks)
            tick_no += ticks
            assert batched.state() == looped.state(), f"{name} K={k}: the batched call's worlds differ from the single calls'"
    med = lambda xs: round(1e3 * statistics.median(xs), 3)  # noqa: E731
    return {"workload": name, "worlds": n_worlds, "rows": batched.batch.engines[0].row_count(), "k": k, "reps": reps,
            "ticks_per_rep": ticks,
            "pipelined": {"batched_tick_ms": med(times["b_tick_p"]), "single_tick_ms": med(times["l_tick_p"]),
                          "batched_edit_ms": med(times["b_edit_p"]), "single_edit_ms": med(times["l_edit_p"])},
            "synchronised": {"batched_tick_ms": med(times["b_tick_s"]), "single_tick_ms": med(times["l_tick_s"]),
                             "batched_edit_ms": med(times["b_edit_s"]), "single_edit_ms": med(times["l_edit_s"])}}


def profile_call(name, make, n_worlds, k):
    """Device time of one batched edit call and of one loop of single calls (microseconds by kernel / copy name)."""
    import torch
    from torch.profiler import ProfilerActivity
    batched, looped = setup(make, n_worlds)
    out = {"workload": name, "worlds": n_worlds, "k": k}
    for tag, side in (("batched", batched), ("single", looped)):
        calls = side.draw(k, True, np.random.default_rng(5))
        side.batch.engines[0].synchronize()
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            side.apply(calls, side is batched)
            side.batch.engines[0].synchronize()
        times = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                times[e.key[:60]] = [round(e.device_time_total, 1), e.count]
        out[tag + "_device_us"] = times
        out[tag + "_device_us_total"] = round(sum(t for t, _ in times.values()), 1)
    assert batched.state() == looped.state(), f"{name} K={k}: the batched call's worlds differ from the single calls'"
    return out


WORKLOADS = {
    "box_game": [(f"box_game_{n}", box_world, n) for n in (16, 256, 1024)],
    "presence": [("presence_2000x256", presence_world, 256)],
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=8)
    ap.add_argument("--only", default="box_game,presence")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if args.reps < 5:
        ap.error("--reps must be at least 5 (the medians are of at least 5 repetitions)")
    info = card()
    rows = []
    for group in args.only.split(","):
        for name, make, n in WORKLOADS[group]:
            for k in (1, 16):
                r = profile_call(name, make, n, k) if args.profile else bench(name, make, n, k, args.reps, args.ticks)
                r.update(info)
                print(json.dumps(r), flush=True)
                rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
