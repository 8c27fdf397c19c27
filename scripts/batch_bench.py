"""World batches against one engine per world: host wall time per tick of ONE bgr_batch_handle_requests over N worlds
versus N bgr_handle_requests calls on twin engines, alternating in one process, with the checksums of both compared on
every tick.  `--profile` instead measures the batch kernel's device time with torch.profiler (a run of its own: tracing
slows the host).

Workloads: N box_game worlds (2 rollback entities, move_cube_system) and N presence worlds of 2 000 rows (Score / Health /
Tag), every world in a SyncTest session with check distance 7, the sizes a server hosting many matches or a SyncTest
farm runs.  All worlds of a workload get the same inputs, so one request vector per tick serves them all; their
populations differ (seeded), so their checksums do too.

    python scripts/batch_bench.py [--ticks 40] [--warmup 10] [--out results.json] [--profile]
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

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine, EngineBatch  # noqa: E402
from bevy_ggrs_b200.session import SAVE, SyncTestSession  # noqa: E402

SEQ = [0b0001, 0b1000, 0b0101, 0, 0b0010, 0b1010, 0b0100, 0b1001]
WORKLOADS = [("box_game", n) for n in (1, 16, 256, 1024, 4096)] + [("presence_2000", n) for n in (1, 16, 256)]


def box_world(seed, stream=None):
    w = Engine(max_entities=2, max_depth=9, stream=stream)
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


def presence_world(seed, stream=None, n=2000):
    opt = capi.BGR_STRATEGY_OPTIONAL
    w = Engine(max_entities=n, max_depth=9, stream=stream)
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | opt)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | opt)
    tag = w.rollback_component("Tag", 12, capi.BGR_STRATEGY_COPY)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        w.checksum_component(c, 0, ln)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.build()
    w.spawn(n)
    rng = np.random.default_rng(seed)
    w.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    w.write_component(health, 0, rng.integers(100, 100000, n, dtype=np.uint32))
    w.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    return w


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def run(kind, n, ticks, warmup, profile):
    import torch
    stream = torch.cuda.Stream()
    make = box_world if kind == "box_game" else presence_world
    members = [make(i, stream.cuda_stream) for i in range(n)]
    twins = [] if profile else [make(i) for i in range(n)]
    batch = EngineBatch(members)
    lib = capi.load_library()
    sess = SyncTestSession(2, 7, 9)
    info1 = capi.make_session_info(sess.info())
    sessions = (capi.bgr_session_info * n)(*([info1] * n))
    worlds = (C.c_uint32 * n)(*range(n))
    status = (C.c_int32 * n)()
    n_cs = (C.c_uint32 * n)()
    t_batch, t_seq, kernel_us = [], [], []
    for tick in range(warmup + ticks):
        for h in range(2):
            sess.add_local_input(h, SEQ[(tick + 3 * h) % len(SEQ)])
        reqs = sess.advance_frame()
        k, k_s = len(reqs), sum(1 for r in reqs if r.kind == SAVE)
        one = capi.make_requests(reqs)
        flat = (capi.bgr_request * (n * k)).from_buffer_copy(bytes(one) * n)
        n_req = (C.c_uint32 * n)(*([k] * n))
        out_b = (capi.bgr_checksum * max(1, n * k_s))()
        out_s = (capi.bgr_checksum * max(1, n * k_s))()
        timed = tick >= warmup
        if profile and timed:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                rc = lib.bgr_batch_handle_requests(batch._h, worlds, n, sessions, flat, n_req, out_b, n * k_s, n_cs, status)
                torch.cuda.synchronize()
            # the first session of a process may miss its kernels while the tracer starts: only what was recorded counts
            kernel_us += [e.time_range.elapsed_us() for e in prof.events() if e.name == "k_generic_jit_batch"]
        else:
            t0 = time.perf_counter_ns()
            rc = lib.bgr_batch_handle_requests(batch._h, worlds, n, sessions, flat, n_req, out_b, n * k_s, n_cs, status)
            t1 = time.perf_counter_ns()
        assert rc == capi.BGR_OK, lib.bgr_last_error().decode()
        if not profile:
            cnt = C.c_uint32()
            info_ref, cnt_ref, handles = C.byref(info1), C.byref(cnt), [e._h for e in twins]
            outs = [C.cast(C.addressof(out_s) + i * k_s * C.sizeof(capi.bgr_checksum), C.POINTER(capi.bgr_checksum)) for i in range(n)]
            rcs = [0] * n
            t2 = time.perf_counter_ns()
            for i in range(n):
                rcs[i] = lib.bgr_handle_requests(handles[i], info_ref, one, k, outs[i], k_s, cnt_ref)
            t3 = time.perf_counter_ns()
            assert not any(rcs), lib.bgr_last_error().decode()
            assert bytes(out_b) == bytes(out_s), f"{kind} N={n} tick {tick}: batched checksums differ from the twins'"
            if timed:
                t_batch.append((t1 - t0) / 1e3)
                t_seq.append((t3 - t2) / 1e3)
        for j in range(k_s):
            sess.save_cell(out_b[j].frame, (out_b[j].hi << 64) | out_b[j].lo)
    res = {"workload": kind, "n_worlds": n, "specialised": batch.specialised(), "ticks": ticks}
    if profile:
        res["batch_kernel_us_median"] = statistics.median(kernel_us) if kernel_us else None
        res["kernels_recorded"] = len(kernel_us)
    else:
        res["batch_us_median"] = statistics.median(t_batch)
        res["sequential_us_median"] = statistics.median(t_seq)
        res["speedup"] = res["sequential_us_median"] / res["batch_us_median"]
        res["checksums_compared"] = (warmup + ticks) * n
    batch.close()
    for e in members + twins:
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile", action="store_true", help="device time of the batch kernel (torch.profiler)")
    ap.add_argument("--only", default="", help="comma-separated workload:n filter, e.g. box_game:16")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("batch_bench needs a GPU")
    gpu = card()
    print(f"card: {gpu}", flush=True)
    results = []
    for kind, n in WORKLOADS:
        if a.only and f"{kind}:{n}" not in a.only.split(","):
            continue
        r = run(kind, n, a.ticks, a.warmup, a.profile)
        r["card"] = gpu
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
