"""Spawning worlds on the generic one-launch program against the stepwise path they ran on before.

World leg: the particles columns with a whole-Transform checksum (checksum_component_with_hash::<Transform>, which is
not the bundle's layout) at 100k and 1M rows, SyncTest at check distance 8, 100 rows spawned per spawning frame on two
ticks in five.  Three engines with the same population tick the same vectors, alternating in one process: stepwise
(BGR_CFG_FORCE_STEPWISE), the interpreter (BGR_TUNE_JIT=0) and the generated kernel (BGR_TUNE_JIT=2).  Host wall time
per synchronous tick, median; checksums of the three compared on every tick.  `--profile` instead sums the device time
of every kernel of a tick with torch.profiler (a run of its own: tracing slows the host).

Batch leg: 16 and 256 spawning worlds of 2 000 rows (seeds differ per world) in one bgr_batch_handle_requests against
one bgr_handle_requests per twin engine, checksums compared on every tick.

    python scripts/generic_spawn_bench.py [--ticks 30] [--warmup 10] [--profile] [--out results.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from batch_bench import card  # noqa: E402
from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine, EngineBatch  # noqa: E402
from bevy_ggrs_b200.session import SAVE, SyncTestSession  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402

RATE = 100
VARIANTS = [("stepwise", capi.BGR_CFG_FORCE_STEPWISE, "2"), ("interpreter", 0, "0"), ("generated", 0, "2")]


def whole_transform(w, t, v):
    w.checksum_component(v, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
    w.checksum_component(t, 0, 40)


def world(n, cap, seed=5, flags=0, jit="2", stream=None, rate=RATE):
    os.environ["BGR_TUNE_JIT"] = jit  # read when the engine is built
    w = Engine(max_entities=cap, max_depth=9, flags=flags, stream=stream)
    cols = register_particles(w, spawn_rate=rate, spawn_ttl=300, rng_seed=seed, checksums=whole_transform)
    w.build()
    populate(w, cols, *synth_particles(n, seed, 100, 400))
    return w


def vectors(ticks, d=8):
    sess = SyncTestSession(2, d, 9)
    out = []
    for t in range(ticks):
        sess.add_local_input(0, capi.BGR_INPUT_SPAWN if t % 5 in (1, 2) else 0)
        sess.add_local_input(1, 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        out.append((sess.info(), reqs))
    return out


def world_leg(n, ticks, warmup, profile):
    import torch
    vs = vectors(warmup + ticks)
    cap = n + RATE * (warmup + ticks + 2)
    engines = {name: world(n, cap, flags=flags, jit=jit) for name, flags, jit in VARIANTS}
    kinds = {}
    wall = {name: [] for name in engines}
    dev = {name: [] for name in engines}
    for t, (info, reqs) in enumerate(vs):
        got = {}
        for name, e in engines.items():
            if profile and t >= warmup:
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    got[name] = e.handle_requests(info, reqs)
                    torch.cuda.synchronize()
                ks = [ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
                if ks:
                    dev[name].append(sum(ev.time_range.elapsed_us() for ev in ks))
            else:
                t0 = time.perf_counter_ns()
                got[name] = e.handle_requests(info, reqs)
                t1 = time.perf_counter_ns()
                if t >= warmup:
                    wall[name].append((t1 - t0) / 1e3)
            kinds[name] = e.last_kernel().kind
        assert got["stepwise"] == got["interpreter"] == got["generated"], f"{n} rows tick {t}: checksums differ"
    res = {"leg": "world", "rows": n, "rows_end": engines["generated"].row_count(), "ticks": ticks, "kernels": kinds}
    for name in engines:
        if profile:
            res[f"{name}_device_us_median"] = statistics.median(dev[name]) if dev[name] else None
        else:
            res[f"{name}_us_median"] = statistics.median(wall[name])
    res["checksums_compared"] = len(vs)
    for e in engines.values():
        e.close()
    return res


def batch_leg(n_worlds, ticks, warmup, rows=2000):
    import torch
    stream = torch.cuda.Stream()
    cap = rows + 30 * (warmup + ticks + 2)
    members = [world(rows, cap, seed=i, stream=stream.cuda_stream, rate=30) for i in range(n_worlds)]
    twins = [world(rows, cap, seed=i, rate=30) for i in range(n_worlds)]
    batch = EngineBatch(members)
    lib = capi.load_library()
    n = n_worlds
    worlds = (C.c_uint32 * n)(*range(n))
    status = (C.c_int32 * n)()
    n_cs = (C.c_uint32 * n)()
    t_batch, t_seq = [], []
    for t, (info, reqs) in enumerate(vectors(warmup + ticks, d=7)):
        k, k_s = len(reqs), sum(1 for r in reqs if r.kind == SAVE)
        si = capi.make_session_info(info)
        sessions = (capi.bgr_session_info * n)(*([si] * n))
        one = capi.make_requests(reqs)
        flat = (capi.bgr_request * (n * k)).from_buffer_copy(bytes(one) * n)
        n_req = (C.c_uint32 * n)(*([k] * n))
        out_b = (capi.bgr_checksum * max(1, n * k_s))()
        out_s = (capi.bgr_checksum * max(1, n * k_s))()
        outs = [C.cast(C.addressof(out_s) + i * k_s * C.sizeof(capi.bgr_checksum), C.POINTER(capi.bgr_checksum)) for i in range(n)]
        cnt = C.c_uint32()
        t0 = time.perf_counter_ns()
        rc = lib.bgr_batch_handle_requests(batch._h, worlds, n, sessions, flat, n_req, out_b, n * k_s, n_cs, status)
        t1 = time.perf_counter_ns()
        assert rc == capi.BGR_OK, lib.bgr_last_error().decode()
        rcs = [lib.bgr_handle_requests(twins[i]._h, C.byref(si), one, k, outs[i], k_s, C.byref(cnt)) for i in range(n)]
        t2 = time.perf_counter_ns()
        assert not any(rcs), lib.bgr_last_error().decode()
        assert bytes(out_b) == bytes(out_s), f"{n} worlds tick {t}: batched checksums differ from the twins'"
        if t >= warmup:
            t_batch.append((t1 - t0) / 1e3)
            t_seq.append((t2 - t1) / 1e3)
    res = {"leg": "batch", "n_worlds": n, "rows": rows, "specialised": batch.specialised(), "ticks": ticks,
           "batch_us_median": statistics.median(t_batch), "sequential_us_median": statistics.median(t_seq)}
    res["speedup"] = res["sequential_us_median"] / res["batch_us_median"]
    batch.close()
    for e in members + twins:
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile", action="store_true", help="device time per tick of each variant (torch.profiler)")
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--batches", default="16,256")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("generic_spawn_bench needs a GPU")
    gpu = card()
    print(f"card: {gpu}", flush=True)
    results = []
    for n in [int(x) for x in a.sizes.split(",") if x]:
        r = world_leg(n, a.ticks, a.warmup, a.profile)
        r["card"] = gpu
        print(json.dumps(r), flush=True)
        results.append(r)
    if not a.profile:
        for nw in [int(x) for x in a.batches.split(",") if x]:
            r = batch_leg(nw, a.ticks, a.warmup)
            r["card"] = gpu
            print(json.dumps(r), flush=True)
            results.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
