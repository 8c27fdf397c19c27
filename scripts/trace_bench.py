"""Replay traces against the two ways a caller gets the same per-frame data without them, in one process on twin engines,
alternating every repetition: host wall time of ONE trace replay call (bgr_replay_trace / bgr_batch_replay_trace), of a
plain replay of the same log (bgr_replay / bgr_batch_replay), and of the two status-quo paths:
  - "step": the log split at every sample frame, each piece replayed (batched across the worlds), then per world
    bgr_row_count, bgr_read_alive, and bgr_read_component + bgr_has_component per field;
  - "keyframes": bgr_batch_replay_keyframes with K = T, then every blob decoded on the host (tests/checkpoint_codec.py,
    the numpy restatement of the checkpoint format) and the records cut out of it.
Both status-quo paths are one host round trip or more per sample and world, so they run on the first STATUS_QUO_WORLDS
worlds over the first STATUS_QUO_FRAMES frames of the log, and are reported per world and frame next to the trace call's
per world and frame.  The records of both must equal the trace call's on every repetition.

Workloads: box_game batches of 1, 16, 256 and 1 024 worlds x 3 600 frames tracing every row's Transform translation and
Velocity at T = 1 and T = 10; one spawning particles world (2 000 rows, a spawn every 60 frames) tracing rows
[0, 4 000) at T = 10; the 100k-row stress world tracing 1 000 rows at T = 10 over 600 frames.  Checksums at the examples'
interval of 10.  Prints one JSON line per workload, with the card's name, power limit and max SM clock read in the same
run.  `--profile` instead takes device times from torch.profiler in a run of its own (tracing slows the host): one trace
call and one plain replay call per workload after a warm-up call, every kernel and copy summed by name.

    python scripts/trace_bench.py [--reps 3] [--only box_game,particles,stress] [--profile] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import checkpoint_codec as cc  # noqa: E402
from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.engine import EngineBatch  # noqa: E402
from keyframe_bench import OneWorld, card, particles_world, timed  # noqa: E402
from replay_bench import box_world  # noqa: E402

K_CHECKSUM = 10
STATUS_QUO_WORLDS = 4
STATUS_QUO_FRAMES = 600
# Transform's translation and Velocity: the columns are Transform then Velocity for the particles worlds, Velocity then
# Transform for box_game
BOX_FIELDS = [(1, 0, 12), (0, 0, 12)]
PARTICLE_FIELDS = [(0, 0, 12), (1, 0, 12)]


class OneTrace(OneWorld):
    def replay_trace(self, calls, fields):
        return [(capi.BGR_OK, *self.engines[0].replay_trace(x, k, tt, fields, a, nr)) for _, x, k, tt, a, nr in calls]


def read_records(e, fields, first, n_rows):
    """The records of rows [first, first + n_rows) read back with the per-row entry points."""
    rb = 8 + sum(ln for _, _, ln in fields)
    out = np.zeros((n_rows, rb), np.uint8)
    out[:, 0:4] = np.arange(first, first + n_rows, dtype="<u4").view(np.uint8).reshape(-1, 4)
    m = max(0, min(first + n_rows, e.row_count()) - first)
    if m:
        state = (e.read_alive(first, m) != 0).astype("<u4")
        at = 8
        for k, (c, off, ln) in enumerate(fields):
            has = e.has_component(c, first, m) != 0
            state |= has.astype("<u4") << (1 + k)
            v = e.read_component(c, first, m)[:, off:off + ln].copy()
            v[~has] = 0
            out[:m, at:at + ln] = v
            at += ln
        out[:m, 4:8] = state.view(np.uint8).reshape(-1, 4)
    return out


def blob_records(blob, e, fields, first, n_rows):
    """The records cut out of a checkpoint blob (no optional columns in these workloads: present = exists)."""
    h, planes, mask = cc.decode(blob)
    plane0 = np.cumsum([0] + [b // 4 for b in e.elem_bytes])
    rb = 8 + sum(ln for _, _, ln in fields)
    out = np.zeros((n_rows, rb), np.uint8)
    rows = np.arange(first, first + n_rows)
    out[:, 0:4] = rows.astype("<u4").view(np.uint8).reshape(-1, 4)
    ok = rows < h["rows"]
    t, lane = rows[ok] // 512, rows[ok] % 512
    alive = np.zeros(n_rows, bool)
    alive[ok] = (mask[t, lane] & 1) != 0
    state = alive.astype("<u4")
    at = 8
    for k, (c, off, ln) in enumerate(fields):
        state |= alive.astype("<u4") << (1 + k)
        for w in range(ln // 4):
            v = np.zeros(n_rows, "<u4")
            v[ok] = planes[t, plane0[c] + off // 4 + w, lane]
            v[~alive] = 0
            out[:, at:at + 4] = v.view(np.uint8).reshape(-1, 4)
            at += 4
    out[:, 4:8] = state.view(np.uint8).reshape(-1, 4)
    return out


def step_path(group, worlds, log, tt, fields, first, n_rows):
    f0 = group.engines[worlds[0]].rollback_frame_count()
    recs = [[] for _ in worlds]
    at = 0
    for j in range(len(log)):
        if (f0 + j) % tt:
            continue
        if j > at:
            group.replay([(w, log[at:j], K_CHECKSUM) for w in worlds])
            at = j
        for i, w in enumerate(worlds):
            recs[i].append(read_records(group.engines[w], fields, first, n_rows))
    if at < len(log):
        group.replay([(w, log[at:], K_CHECKSUM) for w in worlds])
    return [np.array(r, np.uint8) for r in recs]


def keyframe_path(group, worlds, log, tt, fields, first, n_rows):
    res = group.replay_keyframes([(w, log, K_CHECKSUM, tt) for w in worlds])
    return [np.array([blob_records(b, group.engines[w], fields, first, n_rows) for _, b in kfs], np.uint8)
            for w, (_, _, kfs) in zip(worlds, res)]


def bench(name, make, n_worlds, frames, tt, fields, first, n_rows, reps, spawn_every=0, batched=True):
    import torch
    stream = torch.cuda.Stream().cuda_stream
    group = (lambda es: EngineBatch(es)) if batched else (lambda es: OneTrace(es[0]))
    sq_n = min(n_worlds, STATUS_QUO_WORLDS)
    trb, plain = (group([make(i, stream) for i in range(n_worlds)]) for _ in range(2))
    step, kfp = (group([make(i, stream) for i in range(sq_n)]) for _ in range(2))
    sq_worlds = list(range(sq_n))
    sq_frames = min(frames, STATUS_QUO_FRAMES)
    rng = np.random.default_rng(0)
    t_tr, t_plain, t_step, t_kf = [], [], [], []
    for rep in range(reps + 1):
        log = rng.integers(0, 16, (frames, 2), dtype=np.uint8)
        if spawn_every:
            log[::spawn_every, 0] |= capi.BGR_INPUT_SPAWN
        t1, ra = timed(lambda: trb.replay_trace([(w, log, K_CHECKSUM, tt, first, n_rows) for w in range(n_worlds)], fields))
        t2, rb = timed(lambda: plain.replay([(w, log, K_CHECKSUM) for w in range(n_worlds)]))
        t3, rc = timed(lambda: step_path(step, sq_worlds, log[:sq_frames], tt, fields, first, n_rows))
        t4, rd = timed(lambda: keyframe_path(kfp, sq_worlds, log[:sq_frames], tt, fields, first, n_rows))
        for g in (step, kfp):  # on to the end of the log, so that every group starts the next repetition at one frame
            g.replay([(w, log[sq_frames:], K_CHECKSUM) for w in sq_worlds])
        assert [r[1] for r in ra] == [cs for _, cs in rb], "trace replay and plain replay disagree"
        assert trb.engines[0].last_kernel().replay
        n_sq = len(rc[0])
        for i in sq_worlds:
            assert np.array_equal(ra[i][3][:n_sq], rc[i]), "the trace and the step path differ"
            assert np.array_equal(ra[i][3][:n_sq], rd[i]), "the trace and the keyframe path differ"
        if rep:
            t_tr.append(t1); t_plain.append(t2); t_step.append(t3); t_kf.append(t4)
        n_samples = len(ra[0][2])
        rec_bytes = sum(r[3].nbytes for r in ra)
    med = lambda xs: 1e3 * statistics.median(xs)  # noqa: E731
    per = lambda t, w, f: med(t) / (w * f)  # noqa: E731
    return {"workload": name, "worlds": n_worlds, "rows": trb.engines[0].row_count(), "frames": frames, "trace_interval": tt,
            "traced_rows": n_rows, "samples_per_world": n_samples, "record_bytes": rec_bytes,
            "trace_replay_ms": med(t_tr), "plain_replay_ms": med(t_plain),
            "trace_cost": statistics.median(t_tr) / statistics.median(t_plain),
            "trace_ms_per_world_frame": per(t_tr, n_worlds, frames),
            "status_quo_worlds": sq_n, "status_quo_frames": sq_frames,
            "step_path_ms": med(t_step), "step_path_ms_per_world_frame": per(t_step, sq_n, sq_frames),
            "keyframe_path_ms": med(t_kf), "keyframe_path_ms_per_world_frame": per(t_kf, sq_n, sq_frames)}


def profile_call(name, make, n_worlds, frames, tt, fields, first, n_rows, spawn_every=0, batched=True):
    """Device time of one trace call and one plain replay call, by kernel and copy name (microseconds)."""
    import torch
    from torch.profiler import ProfilerActivity
    stream = torch.cuda.Stream().cuda_stream
    group = (lambda es: EngineBatch(es)) if batched else (lambda es: OneTrace(es[0]))
    trb, plain = (group([make(i, stream) for i in range(n_worlds)]) for _ in range(2))
    rng = np.random.default_rng(0)
    out = {"workload": name, "worlds": n_worlds, "frames": frames, "trace_interval": tt}
    for rep in range(2):  # the first call compiles the generated kernel and sizes the buffers
        log = rng.integers(0, 16, (frames, 2), dtype=np.uint8)
        if spawn_every:
            log[::spawn_every, 0] |= capi.BGR_INPUT_SPAWN
        for tag, fn in (("trace", lambda: trb.replay_trace([(w, log, K_CHECKSUM, tt, first, n_rows) for w in range(n_worlds)], fields)),
                        ("plain", lambda: plain.replay([(w, log, K_CHECKSUM) for w in range(n_worlds)]))):
            if not rep:
                fn()
                continue
            with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            times = {}
            for e in prof.key_averages():
                if e.device_time_total > 0:
                    times[e.key[:60]] = round(e.device_time_total, 1)
            out[tag + "_device_us"] = times
            out[tag + "_device_us_total"] = round(sum(times.values()), 1)
    return out


def cases(only):
    """(name, make, worlds, frames, T, fields, first_row, n_rows, spawn_every, batched)"""
    out = []
    if "box_game" in only:
        for n in (1, 16, 256, 1024):
            for tt in (1, 10):
                out.append((f"box_game_{n}_t{tt}", lambda i, s: box_world(i, s), n, 3600, tt, BOX_FIELDS, 0, 2, 0, True))
    if "particles" in only:
        out.append(("particles_2000_t10", lambda i, s: particles_world(2000, 5, (60, 300), s), 1, 3600, 10, PARTICLE_FIELDS,
                    0, 4000, 60, False))
    if "stress" in only:
        out.append(("stress_100000_rows1000_t10", lambda i, s: particles_world(100_000, 0, (10**6, 2 * 10**6), s), 1, 600, 10,
                    PARTICLE_FIELDS, 50_000, 1000, 0, False))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="box_game,particles,stress")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    info = card()
    rows = []
    for name, make, n, frames, tt, fields, first, nr, spawn_every, batched in cases(args.only.split(",")):
        if args.profile:
            r = profile_call(name, make, n, frames, tt, fields, first, nr, spawn_every, batched)
        else:
            r = bench(name, make, n, frames, tt, fields, first, nr, args.reps, spawn_every, batched)
        r = dict(r, **info)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
