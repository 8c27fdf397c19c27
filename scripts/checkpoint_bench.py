"""World checkpoint cost on the stress world (1M and 10M rows after 200 SyncTest ticks): blob size against the stored
image S*E, kernel time of encoding (k_ckpt_measure + k_ckpt_scan + k_ckpt_pack) and decoding (k_ckpt_unpack) from
torch.profiler's CUDA activity over repeated calls, as GB/s of 2*S*E read plus the payload written and as a share of the
H100 SXM's 3.35 TB/s, and whole bgr_checkpoint_save / bgr_checkpoint_restore calls into pageable and page-locked
buffers.  Prints one JSON line per size, with the card's name and power limit read in the same run.

    python scripts/checkpoint_bench.py [--rows 1048576 10485760] [--reps 10]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevy_ggrs_b200.engine import Engine  # noqa: E402
from bevy_ggrs_b200.session import SyncTestSession  # noqa: E402
from bevy_ggrs_b200.stress import SLOT_BYTES_PER_ENTITY, populate, register_particles, synth_particles  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
ENCODE = ("k_ckpt_measure", "k_ckpt_scan", "k_ckpt_pack")
DECODE = ("k_ckpt_unpack",)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def world(rows: int) -> Engine:
    eng = Engine(max_entities=rows, max_depth=9)
    cols = register_particles(eng)
    eng.build()
    populate(eng, cols, *synth_particles(rows, 1, 400, 800))
    sess = SyncTestSession(1, 2, 8)
    for _ in range(200):
        sess.add_local_input(0, 0)
        for f, c in eng.handle_requests(sess.info(), sess.advance_frame()):
            sess.save_cell(f, c)
    return eng


def kernel_ns(fn, reps: int, names) -> float:
    """Mean device time per call of the kernels whose names contain one of ``names``.  The kernels run inside one
    library call, between the digest and the copies, so events recorded from outside the call cannot bracket them;
    the profiler's CUDA activity records each kernel's own start and end on the device."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total = 0.0
    for ka in prof.key_averages():
        if any(n in ka.key for n in names):
            total += ka.self_device_time_total   # a kernel row: its own device time, nothing nested
    return total * 1e3 / reps   # us -> ns


def timed(fn, reps: int) -> float:
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def bench(rows: int, reps: int) -> dict:
    eng = world(rows)
    lib = eng._lib
    frame = eng.snapshot_frames()[0]
    blob = eng.checkpoint(frame)
    n = len(blob)
    size, found = C.c_size_t(), C.c_int32()
    pageable = np.empty(n, np.uint8)
    pinned = eng.host_alloc(n, 1)

    def save(dst):
        eng._check(lib.bgr_checkpoint_save(eng._h, frame, dst.ctypes.data, dst.size, C.byref(size), C.byref(found)))

    def restore(src):
        eng._check(lib.bgr_checkpoint_restore(eng._h, src.ctypes.data, n))
    save(pinned)
    assert pinned.tobytes() == blob
    stored = rows * SLOT_BYTES_PER_ENTITY
    enc_ns = kernel_ns(lambda: save(pinned), reps, ENCODE)
    dec_ns = kernel_ns(lambda: restore(pinned), reps, DECODE)
    payload = n - 104 - 8 * (-(-rows // 512) + 1)
    enc_bytes = 2 * stored + payload   # measure and pack each read the image, pack writes the payload
    dec_bytes = payload + stored       # unpack reads the payload and writes the scratch image
    out = {
        "rows": rows, **card(),
        "blob_bytes": n, "stored_bytes": stored, "ratio": round(stored / n, 3),
        "encode_kernels_us": round(enc_ns / 1e3, 1),
        "encode_GBps": round(enc_bytes / enc_ns, 1), "encode_share_of_3.35TBps": round(enc_bytes / enc_ns * 1e9 / HBM_BYTES_PER_S, 3),
        "decode_kernels_us": round(dec_ns / 1e3, 1),
        "decode_GBps": round(dec_bytes / dec_ns, 1), "decode_share_of_3.35TBps": round(dec_bytes / dec_ns * 1e9 / HBM_BYTES_PER_S, 3),
        "save_call_ms_pageable": round(timed(lambda: save(pageable), reps) * 1e3, 2),
        "save_call_ms_pinned": round(timed(lambda: save(pinned), reps) * 1e3, 2),
        "restore_call_ms_pageable": round(timed(lambda: restore(pageable), reps) * 1e3, 2),
        "restore_call_ms_pinned": round(timed(lambda: restore(pinned), reps) * 1e3, 2),
    }
    eng.close()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[1 << 20, 10 * (1 << 20)])
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    for rows in a.rows:
        print(json.dumps(bench(rows, a.reps)), flush=True)


if __name__ == "__main__":
    main()
