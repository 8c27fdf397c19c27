"""App replays against engine replays: host wall time of ONE App.replay call (the engine's replay plus the App's
FrameCount resource stepped through every frame on the host, its checksum parts XORed in) versus ONE Engine.replay call
of the same log on a twin, alternating, on box_game (2 entities, FrameCount checksummed as box_game_p2p.rs registers it)
x 3 600 frames (a minute at 60 fps) at the desync-detection interval of 10.

Workloads: 1 world in Python and in C++ (scripts/app_replay_bench.cpp, compiled into a temporary directory), and
replay_batch versus EngineBatch.replay at 16, 256 and 1 024 worlds in Python.  Prints one JSON line per workload with
the median ms per call and the card's name and power limit read in the same run.

    python scripts/app_replay_bench.py [--reps 5] [--only single,cpp,batch] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import Engine, EngineBatch  # noqa: E402
from bevy_ggrs_b200.plugin import App, GgrsSchedule, ResourceSystem, System, replay_batch  # noqa: E402

FRAMES, INTERVAL = 3600, 10


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def increase_frame_system(res):  # box_game.rs:146-148
    res["FrameCount"][:] = struct.pack("<I", (struct.unpack("<I", res["FrameCount"])[0] + 1) & 0xFFFFFFFF)


def box_app(seed, stream=None) -> App:
    app = App(Engine(max_entities=2, max_depth=4, stream=stream))
    vel = app.rollback_component_with_copy("Velocity", 12)
    tf = app.rollback_component_with_clone("Transform", 40)
    app.checksum_component(tf, 0, 12, assert_finite=True)
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_BOX_MOVE, [tf, vel]))
    app.rollback_resource_with_copy("FrameCount", bytes(4)).checksum_resource_with_hash("FrameCount")
    app.add_systems(GgrsSchedule, ResourceSystem(increase_frame_system))
    app.finish()
    app.world.spawn(2)
    t = np.zeros((2, 10), np.float32)
    t[:, 0:3] = np.random.default_rng(seed).uniform(-2, 2, (2, 3)); t[:, 6] = 1.0; t[:, 7:10] = 1.0
    app.world.write_component(tf, 0, t)
    return app


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def bench_single(reps):
    a, b = box_app(0), box_app(0)
    rng = np.random.default_rng(1)
    t_app, t_eng = [], []
    for rep in range(reps + 1):
        log = rng.integers(0, 16, (FRAMES, 2), dtype=np.uint8)
        t1, ca = timed(lambda: a.replay(log, INTERVAL))
        t2, cb = timed(lambda: b.world.replay(log, INTERVAL))
        assert [f for f, _ in ca] == [f for f, _ in cb] and ca != cb
        if rep:
            t_app.append(t1)
            t_eng.append(t2)
    return {"workload": "box_game_1", "frames": FRAMES, "interval": INTERVAL,
            "app_replay_ms": 1e3 * statistics.median(t_app), "engine_replay_ms": 1e3 * statistics.median(t_eng)}


def bench_batch(n_worlds, reps):
    import torch
    stream = torch.cuda.Stream().cuda_stream
    apps = [box_app(i, stream) for i in range(n_worlds)]
    twins = [box_app(i, stream) for i in range(n_worlds)]
    a, b = EngineBatch([x.world for x in apps]), EngineBatch([x.world for x in twins])
    rng = np.random.default_rng(0)
    t_app, t_eng = [], []
    for rep in range(reps + 1):
        log = rng.integers(0, 16, (FRAMES, 2), dtype=np.uint8)
        t1, ra = timed(lambda: replay_batch([(x, log, INTERVAL) for x in apps], a))
        t2, rb = timed(lambda: b.replay([(w, log, INTERVAL) for w in range(n_worlds)]))
        assert all(st == capi.BGR_OK for st, _ in rb) and len(ra) == n_worlds
        if rep:
            t_app.append(t1)
            t_eng.append(t2)
    return {"workload": f"box_game_batch_{n_worlds}", "frames": FRAMES, "interval": INTERVAL,
            "resource_system_calls": n_worlds * FRAMES,
            "app_replay_ms": 1e3 * statistics.median(t_app), "engine_replay_ms": 1e3 * statistics.median(t_eng)}


def bench_cpp(reps):
    import __graft_entry__ as g
    lib = g.build_engine()
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "app_replay_bench")
        r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-o", out,
                            os.path.join(ROOT, "scripts", "app_replay_bench.cpp"), "-L" + os.path.dirname(lib),
                            "-lbevy_ggrs_b200", "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        if r.returncode:
            raise RuntimeError(r.stdout + r.stderr)
        r = subprocess.run([out, str(FRAMES), str(INTERVAL), str(reps)], capture_output=True, text=True)
        if r.returncode:
            raise RuntimeError(r.stdout + r.stderr)
        return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="single,cpp,batch")
    ap.add_argument("--out")
    a = ap.parse_args()
    only = set(a.only.split(","))
    info = card()
    runs = []
    if "single" in only:
        runs.append(lambda: bench_single(a.reps))
    if "cpp" in only:
        runs.append(lambda: bench_cpp(a.reps))
    if "batch" in only:
        runs += [lambda n=n: bench_batch(n, a.reps if n < 1024 else min(a.reps, 2)) for n in (16, 256, 1024)]
    rows = []
    for fn in runs:
        r = fn()
        r.update(info)
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
