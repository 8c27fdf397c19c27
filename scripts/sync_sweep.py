#!/usr/bin/env python
"""Tuning sweep of the SYNCHRONOUS path (one bgr_handle_requests per tick, compiled caller): per variant of the
BGR_TUNE_* knobs, the e2e tick time, the device-side kernel duration (bgr_trace_enable) and the pipelined tick time.
Usage: python scripts/sync_sweep.py [workload ...] > sync_sweep.json"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def one(workload, env, K=300):
    import numpy as np
    import torch
    from bevy_ggrs_b200.engine import Engine
    for k in list(os.environ):
        if k.startswith("BGR_TUNE_"):
            del os.environ[k]
    os.environ.update({k: str(v) for k, v in env.items()})
    n, d, maxp = bench.WORKLOADS[workload]
    eng = Engine(max_entities=n, max_depth=maxp, fps=60)
    bench.build_world(eng, n, d, bench.SEED)
    stream = torch.cuda.ExternalStream(eng.stream())
    fill = max(d, maxp) + 2
    ticks = bench.pregenerate_ticks(fill + 5 + 2 * K, d, maxp)
    caller = bench.load_caller()
    warm = bench.CallerBatch(ticks[:fill + 5])
    warm.run(caller, eng)
    eng.trace_enable(K + 8)
    b = bench.CallerBatch(ticks[fill + 5: fill + 5 + K])
    torch.cuda.synchronize()
    hp0 = eng.host_profile()
    s = b.run(caller, eng)
    hp1 = eng.host_profile()
    host = {k: (hp1[k] - hp0[k]) / K / 1e3 for k in ("compile_ns", "launch_ns", "wait_ns", "fold_ns")}
    tr = eng.trace_read(K + 8)
    eng.trace_enable(0)
    # pipelined
    pt = ticks[fill + 5 + K:]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    inflight = 0
    for arr, nreq, _, info, _ in pt:
        eng.submit_prepared(info, arr, nreq)
        inflight += 1
        if inflight > 2:
            eng.collect(); inflight -= 1
    while inflight:
        eng.collect(); inflight -= 1
    e1.record(stream)
    torch.cuda.synchronize()
    res = {"workload": workload, "env": env, "sync_us_per_tick": s / K * 1e6, "sync_p50_us": float(np.median(b.per_tick) * 1e6),
           "sync_p10_us": float(np.percentile(b.per_tick, 10) * 1e6),
           "kernel": bench.trace_stats(tr), "pipelined_us_per_tick": e0.elapsed_time(e1) * 1e3 / len(pt),
           "fused": eng.last_path_fused(), "host_us": host}
    eng.close()
    return res


def main():
    workloads = sys.argv[1:] or ["stress_1m_d8", "stress_100k_d8"]
    variants = [{}, {"BGR_TUNE_DYNAMIC": 0}, {"BGR_TUNE_PREFETCH": 0}, {"BGR_TUNE_BPS": 2}, {"BGR_TUNE_BPS": 1},
                {"BGR_TUNE_POLL": 0}]
    extra = os.environ.get("SWEEP_EXTRA")
    if extra:
        variants = [{}] + json.loads(extra)
    out = []
    for w in workloads:
        for v in variants:
            try:
                r = one(w, v)
            except Exception as exc:
                r = {"workload": w, "env": v, "error": repr(exc)}
            out.append(r)
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
