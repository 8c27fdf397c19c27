"""Change feed against the full per-tick mirror on one GPU.

Worlds of 1M rows.  "counter": Cnt (u32, +1 per frame by BGR_SYS_U32_ADD) and Life (u32, BGR_SYS_U32_SATSUB_DESPAWN);
a fraction p of the rows lives for the whole run, the others die on the first frame, so after it exactly p * 1M rows
change their Cnt every tick.  A feed over Cnt reports those rows (12 B each: row, state, 4 B); the full mirror
(bgr_download_begin of Cnt over every row) moves 4 B * 1M per tick whatever p is.  "particles": the stress test
itself (gravity moves every particle every tick), feed and mirror over Transform.translation (20 B against 12 B per
row).  Both loops are pipelined one tick behind, as INTEGRATION.md "Per-tick mirror" shows: submit tick t, wait for
the mirror of tick t-1, begin the mirror of tick t, collect tick t.

Reports, per world: wall time per tick of tick + feed and of tick + full mirror (runs alternate), the records and PCIe
bytes per tick of each, and the device time of the feed's passes on the engine stream (CUDA events around
bgr_feed_begin after a tick, which enqueues pass 1, the scan and pass 2 there; the copy runs on the copy stream).
Prints one JSON line per world and writes them to --out.

    python scripts/change_feed_bench.py --rows 1048576 --steps 200 --warmup 20 --out change_feed.json
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine  # noqa: E402
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402


def counter_world(n, p, seed=1):
    """(engine, column, byte_offset, byte_len, rows that change per tick)"""
    eng = Engine(max_entities=n, max_depth=9)
    cnt = eng.rollback_component("Cnt", 4, capi.BGR_STRATEGY_COPY)
    life = eng.rollback_component("Life", 4, capi.BGR_STRATEGY_COPY)
    eng.checksum_component(cnt, 0, 4)
    eng.add_system(capi.BGR_SYS_U32_ADD, [cnt], [0, 1])
    eng.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [life], [0, 1])
    eng.build()
    eng.spawn(n)
    rng = np.random.default_rng(seed)
    eng.write_component(cnt, 0, rng.integers(0, 1 << 20, n, dtype=np.uint32))
    lives = rng.random(n) < p
    eng.write_component(life, 0, np.where(lives, np.uint32(1 << 31), np.uint32(1)).astype(np.uint32))
    return eng, cnt, 0, 4, int(lives.sum())


def particles_world(n, seed=1):
    eng = Engine(max_entities=n, max_depth=9)
    cols = register_particles(eng)
    eng.build()
    tf, vel, ttl = synth_particles(n, seed, 4, 60)
    ttl[:] = 1 << 40   # nobody dies during the run
    populate(eng, cols, tf, vel, ttl)
    return eng, cols[0], 0, 12, n


def tick_arrays(n_ticks, start):
    """(session info, requests) of P2P ticks without rollback: Save(f), Advance, with frame f - 1 confirmed."""
    reqs = []
    for f in range(start, start + n_ticks):
        arr = capi.make_requests([Request(SAVE, f), Request(ADVANCE, f, [0])])
        reqs.append((capi.make_session_info((capi.BGR_SESSION_P2P, 8, 0, f - 1)), arr))
    return reqs


def run(eng, mode, feed, buf, field, n, steps, warmup, frame0):
    """Both loops leave the data in the page-locked buffer (the feed through the raw calls: no copy into numpy)."""
    ticks = tick_arrays(steps + warmup, frame0)
    lib, h, t, fi, dst = eng._lib, eng._h, C.c_uint32(), capi.bgr_feed_info(), buf.ctypes.data
    prev = None
    t0 = None
    for i, (info, arr) in enumerate(ticks):
        if i == warmup:
            eng.synchronize()
            t0 = time.perf_counter()
        eng.submit_prepared(info, arr, 2)
        if mode == "feed":
            if prev is not None:
                eng._check(lib.bgr_feed_wait(h, prev, C.byref(fi)))
            eng._check(lib.bgr_feed_begin(h, feed, dst, n, C.byref(t)))
            prev = t.value
        else:
            if prev is not None:
                eng.download_wait(prev)
            prev = eng.download_begin(*field, 0, n, buf)
        eng.collect()
    if mode == "feed":
        eng._check(lib.bgr_feed_wait(h, prev, C.byref(fi)))
    else:
        eng.download_wait(prev)
    eng.synchronize()
    return (time.perf_counter() - t0) / steps, frame0 + steps + warmup


def pass_time_us(eng, feed, buf, n, reps, frame0):
    import torch
    s = torch.cuda.ExternalStream(eng.stream())
    ticks = tick_arrays(reps, frame0)
    total, n_records = 0.0, 0
    for info, arr in ticks:
        eng.submit_prepared(info, arr, 2)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        t = eng.feed_begin(feed, buf, n)
        b.record(s)
        n_records = eng.feed_wait(t)[1].n_records
        eng.collect()
        total += a.elapsed_time(b) * 1000.0
    return total / reps, frame0 + reps, n_records


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--fractions", default="0,0.001,0.01,0.1,1", help="of the counter world")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    lines = []
    worlds = [(f"counter p={p}", lambda p=p: counter_world(a.rows, p)) for p in (float(x) for x in a.fractions.split(","))]
    worlds.append(("particles", lambda: particles_world(a.rows)))
    for name, make in worlds:
        eng, col, off, ln, changing = make()
        field = (col, off, ln)
        feed = eng.feed_create([field])
        fbuf = eng.feed_alloc(feed, a.rows)
        dbuf = eng.host_alloc(a.rows, ln)
        frame = 0
        eng.feed_wait(eng.feed_begin(feed, fbuf, a.rows))  # the first report lists every row
        feed_s, mirror_s = [], []
        for _ in range(a.runs):  # alternate the two loops
            s, frame = run(eng, "feed", feed, fbuf, field, a.rows, a.steps, a.warmup, frame)
            feed_s.append(s)
            s, frame = run(eng, "mirror", feed, dbuf, field, a.rows, a.steps, a.warmup, frame)
            mirror_s.append(s)
        eng.feed_wait(eng.feed_begin(feed, fbuf, a.rows))  # catch up with the mirror loop's ticks
        passes_us, frame, n_records = pass_time_us(eng, feed, fbuf, a.rows, 50, frame)
        rb = 8 + ln
        line = {"gpu": gpu, "world": name, "rows": a.rows, "changing_rows": changing, "records_per_tick": n_records,
                "runs": a.runs, "steps": a.steps,
                "tick_plus_feed_us": [round(x * 1e6, 2) for x in feed_s],
                "tick_plus_mirror_us": [round(x * 1e6, 2) for x in mirror_s],
                "feed_pcie_bytes_per_tick": n_records * rb + 16, "mirror_pcie_bytes_per_tick": ln * a.rows,
                "feed_passes_device_us": round(passes_us, 2)}
        print(json.dumps(line), flush=True)
        lines.append(line)
        eng.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
