"""Host edits against the single calls on one GPU: what a game that edits rollback rows between ticks pays.

The 1M-row stress world (particles, nobody dies during the run) runs P2P ticks [Save(f), Advance], pipelined with 4
vectors in flight and synchronously.  Every tick the host edits K random rows (Velocity, and Transform.translation
only) one of three ways: not at all, through the single calls (bgr_write_component of the element, once per row and
column: a game holds the whole element in its ECS), or as one bgr_apply_edits batch.  Reports, per (K, way, loop):
wall time per tick over the timed window (ended by collecting every vector) and, from a separate traced run, the
64-byte active-plane units the bundle kernel stored per tick (launch trace word [3]) and whether the ticks moved
passive planes.  Prints one JSON line per case and writes them to --out.

    python scripts/host_edits_bench.py --rows 1048576 --steps 200 --warmup 20 --out host_edits.json
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
from bevy_ggrs_b200.engine import EDIT_DTYPE, Engine  # noqa: E402
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402

IN_FLIGHT = 4


def world(n):
    eng = Engine(max_entities=n, max_depth=9)
    cols = register_particles(eng)
    eng.build()
    tf, vel, ttl = synth_particles(n, 1, 4, 60)
    ttl[:] = 1 << 40
    populate(eng, cols, tf, vel, ttl)
    return eng, cols


def tick_arrays(n_ticks, start):
    out = []
    for f in range(start, start + n_ticks):
        arr = capi.make_requests([Request(SAVE, f), Request(ADVANCE, f, [0])])
        out.append((capi.make_session_info((capi.BGR_SESSION_P2P, 8, 0, f - 1)), arr))
    return out


class Edits:
    """One tick's edits of K random rows, prepared before the timed loop: the batch (records + values) and the
    element arrays the single calls write."""

    def __init__(self, rng, n, k, cols, tf, vel):
        t_col, v_col, _ = cols
        self.rows = np.sort(rng.choice(n, k, replace=False)).astype(np.uint32)
        self.vel = np.ascontiguousarray(vel[self.rows])
        self.tf = np.ascontiguousarray(tf[self.rows])
        self.tf[:, 0:3] += rng.uniform(-1, 1, (k, 3)).astype(np.float32)
        self.vel[:, 0] += np.float32(0.5)
        recs = np.zeros(2 * k, EDIT_DTYPE)
        recs["kind"] = capi.BGR_EDIT_WRITE
        recs["count"] = 1
        recs["byte_len"] = 12
        recs["column"][0::2], recs["column"][1::2] = v_col, t_col
        recs["row"][0::2] = recs["row"][1::2] = self.rows
        recs["value_offset"] = np.arange(2 * k, dtype=np.uint32) * 12
        vals = np.empty((k, 2, 3), np.float32)
        vals[:, 0], vals[:, 1] = self.vel, self.tf[:, 0:3]
        self.recs, self.values = recs, np.ascontiguousarray(vals)


def run(eng, cols, way, loop, edits, ticks, warmup, traced=False):
    lib, h = eng._lib, eng._h
    t_col, v_col, _ = cols
    out = (capi.bgr_checksum * 8)()
    n_out = C.c_uint32()
    pending = 0
    if traced:
        eng.trace_enable(len(ticks))
    passive = 0
    t0 = None
    for i, (info, arr) in enumerate(ticks):
        if i == warmup:
            while pending:
                eng._check(lib.bgr_collect(h, out, 8, C.byref(n_out))); pending -= 1
            t0 = time.perf_counter()
        if loop == "sync":
            eng._check(lib.bgr_handle_requests(h, C.byref(info), arr, 2, out, 8, C.byref(n_out)))
        else:
            eng._check(lib.bgr_submit_requests(h, C.byref(info), arr, 2))
            pending += 1
            if pending >= IN_FLIGHT:
                eng._check(lib.bgr_collect(h, out, 8, C.byref(n_out))); pending -= 1
        passive += eng.last_kernel().passive_planes if i >= warmup else 0
        ed = edits[i % len(edits)]
        if way == "batch":
            eng._check(lib.bgr_apply_edits(h, ed.recs.ctypes.data, len(ed.recs), ed.values.ctypes.data, ed.values.nbytes))
        elif way == "single":
            for j, r in enumerate(ed.rows):
                eng._check(lib.bgr_write_component(h, v_col, int(r), 1, ed.vel[j].ctypes.data, 12))
                eng._check(lib.bgr_write_component(h, t_col, int(r), 1, ed.tf[j].ctypes.data, 40))
    while pending:
        eng._check(lib.bgr_collect(h, out, 8, C.byref(n_out))); pending -= 1
    us = (time.perf_counter() - t0) * 1e6 / (len(ticks) - warmup)
    units = None
    if traced:
        tr = eng.trace_read(len(ticks))
        units = float(np.mean(tr[warmup:, 3].astype(np.float64)))
        eng.trace_enable(0)
    return us, units, passive / (len(ticks) - warmup)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = ""
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--ks", default="1,64,4096")
    ap.add_argument("--single-budget", type=int, default=40000, help="single calls per timed run (K=4096 runs few ticks)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    n = a.rows
    tf, vel, _ = synth_particles(n, 1, 4, 60)
    eng, cols = world(n)
    rng = np.random.default_rng(3)
    frame = [eng.rollback_frame_count()]
    lines = []
    gpu = gpu_info()
    for k in [int(x) for x in a.ks.split(",")]:
        edits = [Edits(rng, n, k, cols, tf, vel) for _ in range(8)]
        for way in ("none", "single", "batch"):
            steps = a.steps if way != "single" else max(8, min(a.steps, a.single_budget // (2 * k)))
            warm = a.warmup if way != "single" else min(a.warmup, 4)
            for loop in ("pipelined", "sync"):
                res = {}
                for traced in (False, True):
                    ticks = tick_arrays(steps + warm, frame[0])
                    us, units, passive = run(eng, cols, way, loop, edits, ticks, warm, traced)
                    frame[0] += len(ticks)
                    res["us_per_tick" if not traced else "traced_us_per_tick"] = round(us, 2)
                    if traced:
                        res["stored_units_per_tick"] = round(units, 1)
                        res["passive_tick_share"] = round(passive, 3)
                line = {"rows": n, "k": k, "way": way, "loop": loop, "ticks": steps, "gpu": gpu, **res}
                print(json.dumps(line), flush=True)
                lines.append(line)
    eng.close()
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
