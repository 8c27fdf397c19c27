"""Checkpoint deltas against full checkpoints on one GPU.

Worlds: the counter world of change_feed_bench.py at 100k and 1M rows, where a fraction p of the rows lives and
changes its Cnt every tick and the others die on the first frame, so between two later frames exactly p of the rows
differ; and the 1M-row particles stress world, where every live particle moves every tick.  Each world saves and
advances frames outside a session; the base B is a held frame after the first, the target T = B + 4.

Reports per world: blob bytes of the full checkpoint of T and of the delta of T against B (exact); whole-call times of
bgr_checkpoint_save against bgr_checkpoint_save_delta and of bgr_checkpoint_restore against
bgr_checkpoint_restore_delta, into and from page-locked buffers, alternated, as medians; and, in a pass of its own
under torch.profiler, the device time of each call's kernels.  Prints one JSON line per world, with the card's name
and power limit read in the same run.

    python scripts/checkpoint_delta_bench.py [--reps 15] [--out checkpoint_delta.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
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
from bevy_ggrs_b200.engine import Engine  # noqa: E402
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402
from change_feed_bench import counter_world  # noqa: E402

NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
KERNELS = ("k_ckpt_", "k_frame_digest")


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def particles_world(n: int) -> Engine:
    eng = Engine(max_entities=n, max_depth=9)
    cols = register_particles(eng)
    eng.build()
    populate(eng, cols, *synth_particles(n, 1, 400, 800))
    return eng


def run_frames(eng: Engine, frames: int) -> None:
    for _ in range(frames):
        f = eng.rollback_frame_count()
        eng.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, [0])])


def device_us(fn, reps: int) -> dict:
    """Mean device time per call of each kernel the call runs (torch.profiler's CUDA activity)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ka in prof.key_averages():
        if any(k in ka.key for k in KERNELS):
            name = ka.key.split("(")[0].split("::")[-1]
            out[name] = round(out.get(name, 0.0) + ka.self_device_time_total / reps, 1)
    return out


def bench(name: str, eng: Engine, reps: int, changed_rows=None) -> dict:
    eng.set_depth(8)
    run_frames(eng, 3)
    base_frame = eng.rollback_frame_count()
    run_frames(eng, 5)
    frame = base_frame + 4
    lib = eng._lib
    full, base, delta = eng.checkpoint(frame), eng.checkpoint(base_frame), eng.checkpoint_delta(frame, base_frame)
    size, found = C.c_size_t(), C.c_int32()
    p_full, p_base, p_delta = (eng.host_alloc(len(b), 1).reshape(-1) for b in (full, base, delta))
    p_base[:] = np.frombuffer(base, np.uint8)

    def save_full():
        eng._check(lib.bgr_checkpoint_save(eng._h, frame, p_full.ctypes.data, p_full.size, C.byref(size), C.byref(found)))

    def save_delta():
        eng._check(lib.bgr_checkpoint_save_delta(eng._h, frame, base_frame, p_delta.ctypes.data, p_delta.size,
                                                 C.byref(size), C.byref(found)))

    def restore_full():
        eng._check(lib.bgr_checkpoint_restore(eng._h, p_full.ctypes.data, p_full.size))

    def restore_delta():
        eng._check(lib.bgr_checkpoint_restore_delta(eng._h, p_base.ctypes.data, p_base.size, p_delta.ctypes.data,
                                                    p_delta.size))

    def alternate(a, b):
        a(), b()
        ta, tb = [], []
        for _ in range(reps):
            for fn, acc in ((a, ta), (b, tb)):
                t = time.perf_counter()
                fn()   # every call ends in a stream synchronise
                acc.append(time.perf_counter() - t)
        return round(statistics.median(ta) * 1e3, 3), round(statistics.median(tb) * 1e3, 3)

    save_full(), save_delta()
    assert p_full.tobytes() == full and p_delta.tobytes() == delta
    out = {"world": name, "rows": eng.row_count(), "changed_rows": changed_rows, **card(),
           "full_bytes": len(full), "delta_bytes": len(delta), "ratio": round(len(full) / len(delta), 2)}
    out["save_ms_full"], out["save_ms_delta"] = alternate(save_full, save_delta)
    out["save_kernels_us_full"] = device_us(save_full, reps)
    out["save_kernels_us_delta"] = device_us(save_delta, reps)
    # restores leave the ring holding the target alone, so they come after every save
    out["restore_ms_full"], out["restore_ms_delta"] = alternate(restore_full, restore_delta)
    out["restore_kernels_us_full"] = device_us(restore_full, reps)
    out["restore_kernels_us_delta"] = device_us(restore_delta, reps)
    assert eng.checkpoint(frame) == full
    eng.close()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--rows", type=int, nargs="+", default=[100_000, 1 << 20])
    ap.add_argument("--p", type=float, nargs="+", default=[0.001, 0.01, 0.1, 1.0])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []
    for n in a.rows:
        for p in a.p:
            eng, _, _, _, live = counter_world(n, p)
            lines.append(bench(f"counter p={p}", eng, a.reps, live))
            print(json.dumps(lines[-1]), flush=True)
    lines.append(bench("particles", particles_world(1 << 20), a.reps))
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()
