"""Growable worlds (BGR_CFG_GROWABLE): what one growth step costs, and whether a grown engine ticks as fast as one
created at that capacity.

1. One growth step of the stress schema (particles: Transform 40 B, Velocity 12 B, Ttl 8 B + the alive byte = 61 B a
   row) at depth 8, 1M -> 2M rows, through bgr_reserve: the host time of the mapping calls (arena, side tables), the
   zeroing on the stream, the NVRTC compile (none for the bundle), the whole call, and device memory from
   cudaMemGetInfo before and after.
2. Ticks of 1M rows at depth 8 on an engine grown from 1024 rows (VMM-mapped arena) and on its twin created at the
   grown capacity (cudaMalloc arena), in alternating runs: synchronous (bgr_handle_requests per tick) and pipelined
   (four request vectors in flight).

Prints one JSON object with the card's name and power limit.  Run from the repository root after build():
    python scripts/growth_bench.py [--rows 1048576] [--ticks 300] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine  # noqa: E402
from bevy_ggrs_b200.session import SyncTestSession  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402

DEPTH = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def mem_used():
    import torch
    free, total = torch.cuda.mem_get_info(0)
    return total - free


def particles(cap, flags, rows):
    e = Engine(max_entities=cap, max_depth=DEPTH, flags=flags)
    cols = register_particles(e)
    e.build()
    if flags & capi.BGR_CFG_GROWABLE and e.capacity()[0] < rows:
        e.reserve(rows)
    populate(e, cols, *synth_particles(rows, 7, 30, 10_000))
    e.synchronize()
    return e


def growth_step(rows):
    """bgr_reserve(2 x rows) on a growable engine holding `rows` rows; phase times from BGR_GROW_VERBOSE."""
    os.environ["BGR_GROW_VERBOSE"] = "1"
    e = particles(rows, capi.BGR_CFG_GROWABLE, rows)
    before = mem_used()
    with tempfile.TemporaryFile(mode="w+") as log:
        saved = os.dup(2)
        os.dup2(log.fileno(), 2)
        try:
            t0 = time.perf_counter_ns()
            e.reserve(2 * rows)
            e.synchronize()
            t1 = time.perf_counter_ns()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        log.seek(0)
        text = log.read()
    after = mem_used()
    del os.environ["BGR_GROW_VERBOSE"]
    m = re.search(r"grew (\d+) -> (\d+) rows: map arena (\d+) ns, map side tables (\d+) ns, zero (\d+) ns, jit (\d+) ns, "
                  r"total (\d+) ns", text)
    cap = e.capacity()[0]
    e.close()
    out = {"from_rows": rows, "to_rows": cap, "call_ms": (t1 - t0) / 1e6,
           "device_bytes_before": before, "device_bytes_after": after, "device_bytes_added": after - before}
    if m:
        out.update({"map_arena_ms": int(m.group(3)) / 1e6, "map_side_tables_ms": int(m.group(4)) / 1e6,
                    "zero_ms": int(m.group(5)) / 1e6, "jit_ms": int(m.group(6)) / 1e6})
    return out


def ticks(e, sess, n, pipelined):
    """Seconds per tick of n ticks of `sess` (the engine's own session, continued from run to run), after 20 warm-up
    ticks."""
    vecs = []
    for t in range(n + 20):
        for h in range(2):
            sess.add_local_input(h, (t + h) & 0xF)
        reqs = sess.advance_frame()
        vecs.append((sess.info(), reqs))
        for r in reqs:
            if r.kind == 0:
                sess.save_cell(r.frame, 0)
    prepared = [(capi.make_session_info(i), capi.make_requests(r), len(r)) for i, r in vecs]
    queued = 0
    t0 = 0
    for k, (info, arr, m) in enumerate(prepared):
        if k == 20:
            while queued:
                e.collect()
                queued -= 1
            t0 = time.perf_counter_ns()
        e.submit_prepared(info, arr, m)
        queued += 1
        if queued > (4 if pipelined else 0):
            e.collect()
            queued -= 1
    while queued:
        e.collect()
        queued -= 1
    return (time.perf_counter_ns() - t0) / 1e9 / n


def lasting_cost(rows, n, rounds):
    grown = particles(1024, capi.BGR_CFG_GROWABLE, rows)
    cap = grown.capacity()[0]
    twin = particles(cap, 0, rows)
    # SyncTest, check distance 6 and prediction window 7: the depth-8 ring
    sess = {"grown": SyncTestSession(2, 6, DEPTH - 1, input_delay=2), "twin": SyncTestSession(2, 6, DEPTH - 1, input_delay=2)}
    res = {"rows": rows, "capacity": cap, "grown": {"sync_us": [], "pipelined_us": []}, "twin": {"sync_us": [], "pipelined_us": []}}
    for _ in range(rounds):
        for name, e in (("grown", grown), ("twin", twin)):
            res[name]["sync_us"].append(ticks(e, sess[name], n, False) * 1e6)
            res[name]["pipelined_us"].append(ticks(e, sess[name], n, True) * 1e6)
    for name in ("grown", "twin"):
        for k in ("sync_us", "pipelined_us"):
            res[name][k + "_median"] = statistics.median(res[name][k])
    grown.close()
    twin.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    out = {"card": card(), "depth": DEPTH, "growth_step": growth_step(a.rows), "ticks": lasting_cost(a.rows, a.ticks, a.rounds)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
