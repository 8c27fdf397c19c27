"""Opt-in measurement of desync capture (BGR_CFG_DESYNC_CAPTURE) and of the P2P desync reports on one GPU; bench.py's
default line is unaffected.

  python scripts/desync_bench.py [--legs capture,p2p] [--rounds 6] [--ticks 200] [--diff-reps 20] [--big 10000000]

1. Ticks: the headline workload (1M particles, SyncTest check distance 8, max_prediction 9; bench.py's build_world and
   request vectors) on two engines, one without and one with capture, fed the same request vectors in alternating
   rounds of --ticks ticks (pipelined submit / collect, two vectors in flight, like bench.py's first leg).  Per round:
   host wall time over the round, which ends in a collect, i.e. a device synchronise.  Checksums of both engines must
   be identical tick for tick.
2. Diff: bgr_desync_diff of a re-saved frame of a capture engine at 1M and at --big entities (a deterministic world:
   no differences, so pass 2 does not run).  The time is the whole synchronous call (pass 1, the host scan of the
   per-tile counts, copies); the bytes are what pass 1 must read, 2 * S * E = two images of bgr_slot_bytes each.
P2P legs (--legs p2p):
3. Ticks: 1M particles on the synthetic P2P trace (BASELINE.md C4: max_prediction 8, random rollback depths), on two
   engines, one without and one with bgr_retain_confirmed(10, 4), in alternating rounds like leg 1.  Checksums must be
   identical tick for tick.
4. Digest: bgr_frame_digest of a retained frame at 1M and at --big entities.  Whole call: host wall time of
   Engine.frame_digest (kernel, word copy, root hash).  Kernel alone: k_frame_digest's device time from torch.profiler.
   Bytes: the kernel reads every word plane and the mask of every row once, S * E = bgr_slot_bytes.
5. Export / remote diff: bgr_frame_export of 8 blocks of a retained frame, and bgr_desync_diff_remote of that blob on a
   second engine with the same registration (no differences: pass 2 does not run).
Prints one JSON line, with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, build_world, pregenerate_ticks  # noqa: E402
from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def run_ticks(eng, ticks, history):
    inflight = 0
    for arr, nreq, _, info, _ in ticks:
        eng.submit_prepared(info, arr, nreq)
        inflight += 1
        if inflight > 2:
            history.extend(eng.collect())
            inflight -= 1
    while inflight:
        history.extend(eng.collect())
        inflight -= 1


def time_diff(eng, reps):
    frames = eng.desync_frames()
    assert frames, "no re-saved frame with a retained first image"
    f = frames[0]
    rep = eng.desync_diff(f, 64)  # warm-up: allocates the scratch
    assert rep is not None and rep.empty
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        eng.desync_diff(f, 64)
        times.append(time.perf_counter() - t0)
    bytes_read = 2 * eng.slot_bytes()
    med = statistics.median(times)
    return {"frame": f, "rows": rep.rows_first, "call_ms_median": med * 1e3, "call_ms_min": min(times) * 1e3,
            "pass1_bytes": bytes_read, "effective_GBps_median": bytes_read / med / 1e9}


def kernel_us(fn, reps, name):
    """Median device time of the kernels called `name` that fn() launches (torch.profiler / CUPTI)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    ts = [getattr(e, "device_time", None) or getattr(e, "cuda_time", 0) for e in prof.events() if name in e.name]
    return statistics.median(ts) if ts else None


def time_digest(eng, reps):
    frames = eng.retained_frames()
    assert frames, "no retained frame"
    f = frames[0]
    h, _ = eng.frame_digest(f)  # warm-up: allocates the scratch
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        eng.frame_digest(f)
        times.append(time.perf_counter() - t0)
    med = statistics.median(times)
    k_us = kernel_us(lambda: eng.frame_digest(f), reps, "k_frame_digest")
    se = eng.slot_bytes()
    return {"frame": f, "rows": h.rows, "n_blocks": h.n_blocks, "digest_bytes": h.n_blocks * (h.n_columns + 1) * 8,
            "call_ms_median": med * 1e3, "call_ms_min": min(times) * 1e3, "kernel_us_median": k_us,
            "bytes_read_S_E": se, "kernel_GBps": (se / (k_us * 1e-6) / 1e9) if k_us else None,
            "call_GBps": se / med / 1e9}


def p2p_legs(args, out):
    n, maxp = 1_000_000, 8
    fill = 12
    ticks = pregenerate_ticks(fill + args.rounds * args.ticks, 0, maxp)  # d == 0: the synthetic P2P trace (C4)
    engines = {"plain": Engine(max_entities=n, max_depth=maxp), "retain": Engine(max_entities=n, max_depth=maxp)}
    engines["retain"].retain_confirmed(10, 4)
    hist = {k: [] for k in engines}
    for k, e in engines.items():
        build_world(e, n, 0, 1)
        run_ticks(e, ticks[:fill], hist[k])
    per_tick = {k: [] for k in engines}
    for r in range(args.rounds):
        chunk = ticks[fill + r * args.ticks: fill + (r + 1) * args.ticks]
        for k in (["plain", "retain"] if r % 2 == 0 else ["retain", "plain"]):
            t0 = time.perf_counter()
            run_ticks(engines[k], chunk, hist[k])
            per_tick[k].append((time.perf_counter() - t0) / len(chunk) * 1e6)
    assert hist["plain"] == hist["retain"], "retention changed a checksum"
    out["p2p_ticks"] = {k: {"us_per_tick_rounds": [round(x, 2) for x in v], "us_per_tick_median": statistics.median(v)}
                        for k, v in per_tick.items()}
    out["p2p_ticks"]["retain_over_plain"] = (out["p2p_ticks"]["retain"]["us_per_tick_median"] /
                                             out["p2p_ticks"]["plain"]["us_per_tick_median"])
    ret = engines["retain"]
    out["digest_1m"] = time_digest(ret, args.diff_reps)
    f = ret.retained_frames()[0]
    blocks = list(range(0, 8 * 97, 97))  # 8 blocks spread over the image
    times = []
    for _ in range(args.diff_reps):
        t0 = time.perf_counter()
        blob = ret.export_blocks(f, blocks)
        times.append(time.perf_counter() - t0)
    engines.pop("plain").close()
    peer = Engine(max_entities=n, max_depth=maxp)  # the other peer: same registration, same trace
    peer.retain_confirmed(10, 4)
    build_world(peer, n, 0, 1)
    run_ticks(peer, ticks, [])
    dtimes = []
    assert f in peer.retained_frames() or f in peer.snapshot_frames()
    rep = peer.diff_remote(f, blob, 64)
    assert rep is not None and rep.empty
    for _ in range(args.diff_reps):
        t0 = time.perf_counter()
        peer.diff_remote(f, blob, 64)
        dtimes.append(time.perf_counter() - t0)
    out["export_8_blocks"] = {"bytes": len(blob), "call_ms_median": statistics.median(times) * 1e3}
    out["diff_remote_8_blocks"] = {"call_ms_median": statistics.median(dtimes) * 1e3, "call_ms_min": min(dtimes) * 1e3}
    peer.close()
    ret.close()
    big = Engine(max_entities=args.big, max_depth=maxp)
    big.retain_confirmed(1, 2)
    build_world(big, args.big, 0, 2)
    run_ticks(big, pregenerate_ticks(fill, 0, maxp), [])
    out["digest_big"] = time_digest(big, args.diff_reps)
    big.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="capture,p2p")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--diff-reps", type=int, default=20)
    ap.add_argument("--big", type=int, default=10_000_000)
    args = ap.parse_args()
    n, d, maxp = WORKLOADS["stress_1m_d8"]
    out = {"gpu": gpu_info(), "workload": {"entities": n, "check_distance": d, "max_prediction": maxp}}
    legs = args.legs.split(",")
    if "p2p" in legs:
        p2p_legs(args, out)
    if "capture" not in legs:
        out["gpu_after"] = gpu_info()
        print(json.dumps(out))
        return

    fill = maxp + 2
    ticks = pregenerate_ticks(fill + args.rounds * args.ticks, d, maxp)
    engines = {"plain": Engine(max_entities=n, max_depth=maxp), "capture": Engine(max_entities=n, max_depth=maxp,
                                                                                   flags=capi.BGR_CFG_DESYNC_CAPTURE)}
    hist = {k: [] for k in engines}
    for k, e in engines.items():
        build_world(e, n, d, 1)
        run_ticks(e, ticks[:fill], hist[k])
    per_tick = {k: [] for k in engines}
    for r in range(args.rounds):
        chunk = ticks[fill + r * args.ticks: fill + (r + 1) * args.ticks]
        order = ["plain", "capture"] if r % 2 == 0 else ["capture", "plain"]
        for k in order:
            t0 = time.perf_counter()
            run_ticks(engines[k], chunk, hist[k])
            per_tick[k].append((time.perf_counter() - t0) / len(chunk) * 1e6)
    assert hist["plain"] == hist["capture"], "capture changed a checksum"
    out["ticks"] = {k: {"us_per_tick_rounds": [round(x, 2) for x in v], "us_per_tick_median": statistics.median(v)}
                    for k, v in per_tick.items()}
    out["ticks"]["capture_over_plain"] = out["ticks"]["capture"]["us_per_tick_median"] / out["ticks"]["plain"]["us_per_tick_median"]
    out["diff_1m"] = time_diff(engines["capture"], args.diff_reps)
    for e in engines.values():
        e.close()
    engines.clear()

    big = Engine(max_entities=args.big, max_depth=maxp, flags=capi.BGR_CFG_DESYNC_CAPTURE)
    build_world(big, args.big, d, 2)
    run_ticks(big, pregenerate_ticks(fill + 4, d, maxp), [])
    out["diff_big"] = time_diff(big, args.diff_reps)
    big.close()
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
