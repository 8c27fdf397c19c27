"""Bytes the headline tick actually moves, the bandwidth that gives, and the HBM ceiling of the same access mix.

bench.py counts 61 B per entity for every image a tick touches.  Every engine skips the passive planes of a Save into a
slot that already holds them (content versions, engine.cu HostState), so in the steady state a tick moves only the
active planes and bench.py's roofline figures are effective rates, not traffic.  This script counts per tick:

    images touched = 1 read (the Load, or the base slot / live image) + one write per Save + the live image unless deferred
    bytes          = images touched x rows x (33 B active + 28 B passive when bgr_last_kernel reports passive planes)

The passive planes are counted whenever the launch moved any (BGR_KERNEL_PASSIVE_PLANES), for every image touched: an
upper bound on a tick after a version bump, where some Saves may still skip them.  tick_bytes() is that schema-level
upper bound.  The bundle kernel also skips the active planes a slot already holds (content stamps,
BGR_KERNEL_STABLE_PLANES); the launch trace counts the 64-byte units of active planes it stored (a word plane of a
64-row segment is 4 units, its alive plane 1), and stored_bytes() turns that count into the bytes a tick actually moved:

    stored bytes   = read image x rows x 33 B + stored units x 64 B + stamp traffic
    stamp traffic  = (1 + Saves) x segments x 36 B read + one 4-byte stamp written per stored word plane-segment

A held Save (its slot already holds the content, host-side content ids, bgr_held_saves) stores nothing and reads no
stamps: held_stored_bytes() leaves its stamp reads out.  In the steady state 7 of the 8 Saves are held.

In the same process it runs tools/hbm_mix_bench.cu's fan-out (1 read : 8 writes) over the active footprint, and the
same fan-out with the writes cut to the stored share, and prints the card's name and power limit.  One JSON line on
stdout.

    python scripts/tick_bytes.py [--steps K] [--warmup W] [--entities N]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ACTIVE_BYTES = 12 + 12 + 8 + 1   # Transform.translation, Velocity, Ttl, alive byte: written by the tick's systems
PASSIVE_BYTES = 16 + 12          # Transform.rotation, scale: no registered system writes them
TILE_ROWS = 512
SEG_ROWS = 64
ACTIVE_PLANES = 9


def stored_bytes(rows: int, n_saves: int, units: int) -> int:
    segs = -(-rows // SEG_ROWS)
    return rows * ACTIVE_BYTES + units * 64 + (1 + n_saves) * segs * ACTIVE_PLANES * 4 + units


def held_stored_bytes(rows: int, n_saves: int, n_held: int, units: int) -> int:
    """stored_bytes() of a tick that held n_held of its Saves."""
    return stored_bytes(rows, n_saves - n_held, units)


def images_touched(n_saves: int, deferred_live: bool) -> int:
    return 1 + n_saves + (0 if deferred_live else 1)


def tick_bytes(rows: int, n_saves: int, deferred_live: bool, passive: bool) -> int:
    return images_touched(n_saves, deferred_live) * rows * (ACTIVE_BYTES + (PASSIVE_BYTES if passive else 0))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def fanout_ceiling(image_bytes: int, fan: int, write_bytes: int = 0) -> dict:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "hbm_mix_bench")
        subprocess.run([nvcc, "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                        os.path.join(ROOT, "tools", "hbm_mix_bench.cu")], check=True, capture_output=True)
        r = subprocess.run([exe, str(image_bytes), str(fan)] + ([str(write_bytes)] if write_bytes else []),
                           check=True, capture_output=True, text=True)
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--entities", type=int, default=0)
    args = ap.parse_args()
    import bench
    n, d, maxp = bench.WORKLOADS["stress_1m_d8"]
    n = args.entities or n
    K, W = args.steps, max(3, args.warmup)
    fill = max(d, maxp) + 2
    ticks = bench.pregenerate_ticks(fill + W + 2 * K + 2 * min(K, 256), d, maxp)
    steady_saves = len(ticks[-1][4])
    steady = tick_bytes(n, steady_saves, True, False)
    print(f"[tick_bytes] {n} entities, SyncTest d={d}: steady-state tick = {images_touched(steady_saves, True)} images x "
          f"{ACTIVE_BYTES} B = {steady / 1e6:.1f} MB (after a version bump {tick_bytes(n, steady_saves, True, True) / 1e6:.1f} MB)",
          file=sys.stderr, flush=True)

    import torch
    from bevy_ggrs_b200.engine import Engine
    eng = Engine(max_entities=n, max_depth=maxp, fps=60)
    bench.build_world(eng, n, d, bench.SEED)
    rows = eng.row_count()
    stream = torch.cuda.ExternalStream(eng.stream())
    pos = [0]

    def take(k):
        out = ticks[pos[0]: pos[0] + k]
        pos[0] += k
        return out

    held = []

    def submit(t, moved):
        eng.submit_prepared(t[3], t[0], t[1])
        k = eng.last_kernel()
        moved.append((tick_bytes(rows, len(t[4]), k.deferred_live, k.passive_planes), k.passive_planes))
        held.append(eng.held_saves()["last"])

    def traced(leg_fn, tl, moved):
        eng.trace_enable(len(tl))
        del held[:]
        leg_fn(tl, moved)
        tr = eng.trace_read(len(tl))
        eng.trace_enable(0)
        return [(held_stored_bytes(rows, len(t[4]), h, int(r[3])), int(r[3]) * 64 // max(1, len(t[4]) - h), h)
                for t, r, h in zip(tl, tr, held)]

    def pipelined(tl, moved):
        inflight = 0
        for t in tl:
            submit(t, moved)
            inflight += 1
            if inflight > 2:
                eng.collect()
                inflight -= 1
        while inflight:
            eng.collect()
            inflight -= 1

    pipelined(take(fill + W), [])
    torch.cuda.synchronize()
    # bytes actually stored, from the launch trace, in separate legs: the trace is off while the time is taken
    stored_p = traced(pipelined, take(min(K, 256)), [])

    def synchronous(tl, moved):
        for t in tl:
            submit(t, moved)
            eng.collect()

    stored_s = traced(synchronous, take(min(K, 256)), [])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    moved_p = []
    e0.record(stream)
    pipelined(take(K), moved_p)
    e1.record(stream)
    torch.cuda.synchronize()
    us_p = e0.elapsed_time(e1) * 1e3 / K

    moved_s = []
    t0 = time.perf_counter()
    for t in take(K):   # one synchronous request vector per tick: submit, then wait for its checksums
        submit(t, moved_s)
        eng.collect()
    us_s = (time.perf_counter() - t0) * 1e6 / K
    eng.close()

    image = ACTIVE_BYTES * (-(-n // TILE_ROWS) * TILE_ROWS)
    fan = fanout_ceiling(image, steady_saves)
    # the stored mix: each write carries the share of the image a steady-state Save stores
    per_save = sorted(w for _, w, _ in stored_p)[len(stored_p) // 2]   # data bytes one stored steady-state Save stores
    fan_stored = fanout_ceiling(image, steady_saves, min(image, per_save) // 16 * 16)

    def leg(us, moved, stored):
        b = sum(m for m, _ in moved) / len(moved)
        s = sum(b for b, _, _ in stored) / len(stored)
        return {"us_per_tick": us, "frames_per_s": ticks[-1][2] / (us * 1e-6), "bytes_per_tick": b,
                "ticks_with_passive_planes": sum(p for _, p in moved), "achieved_gbps": b / (us * 1e-6) / 1e9,
                "frac_of_fanout_stg": b / (us * 1e-6) / 1e9 / fan["fanout_stg"]["gbps"],
                "stored_bytes_per_tick": s, "stored_gbps": s / (us * 1e-6) / 1e9,
                "held_saves_per_tick": sum(h for _, _, h in stored) / len(stored),
                "frac_of_stored_mix_stg": s / (us * 1e-6) / 1e9 / fan_stored["fanout_stg"]["gbps"]}

    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(0), "entities": n, "check_distance": d,
                      "steps": K, "steady_state_bytes_per_tick": steady, "pipelined": leg(us_p, moved_p, stored_p),
                      "synchronous": leg(us_s, moved_s, stored_s), "fanout_ceiling": fan,
                      "stored_mix_ceiling": fan_stored}))


if __name__ == "__main__":
    main()
