"""-m gpu: destroying an engine releases everything it allocated.

One round builds, exercises and destroys engines that between them touch every resource an engine allocates lazily or
only under some configuration: downloads, change feeds (one on a growable engine that then grows), host-edit staging,
the desync diff, frame digest, export and remote-diff scratch, the launch trace, and the tile and work-item flags of a
fixed and a growable engine.  After several rounds this process's device memory must equal what it was after the first
round: comparing against the first round leaves out one-time costs (module loads, the JIT cache).  The figure is the
process's own, read from NVML, because the GPU may be shared.  Engines use the ctypes wrapper, so no caching allocator
sits in between.

The file also runs as a plain script, e.g. under a leak checker:
    compute-sanitizer --tool memcheck --leak-check full python tests/test_gpu_engine_lifetime.py
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bevy_ggrs_b200 import capi  # noqa: E402
from bevy_ggrs_b200.capi import BgrError  # noqa: E402
from bevy_ggrs_b200.engine import EDIT_DTYPE, Engine  # noqa: E402
from bevy_ggrs_b200.session import P2PTraceSession, SyncTestSession  # noqa: E402
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
GROW = capi.BGR_CFG_GROWABLE
ROUNDS = 4


def process_device_bytes():
    """Device memory NVML attributes to this process, or None (and why) when NVML cannot see it."""
    try:
        import pynvml
    except ImportError:
        return None, "pynvml is not installed"
    try:
        pynvml.nvmlInit()
    except pynvml.NVMLError as ex:
        return None, f"NVML is unavailable: {ex}"
    try:
        total, seen = 0, False
        for i in range(pynvml.nvmlDeviceGetCount()):
            for p in pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(i)):
                if p.pid == os.getpid():
                    seen = True
                    total += p.usedGpuMemory or 0
        if not seen:
            return None, "NVML lists no compute process with this PID (e.g. a separate PID namespace)"
        return total, None
    finally:
        pynvml.nvmlShutdown()


def _tick(w, sess, inputs):
    for h, x in enumerate(inputs):
        sess.add_local_input(h, x)
    return w.handle_requests(sess.info(), sess.advance_frame())


def _particles(w, n, rate=64):
    cols = register_particles(w, spawn_rate=rate, spawn_ttl=200)
    w.build()
    populate(w, cols, *synth_particles(n, seed=3, ttl_lo=50, ttl_hi=300))
    return cols


def _scores(w, n):
    score = w.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)
    health = w.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE)
    for c in (score, health):
        w.checksum_component(c, 0, 4)
    w.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    w.build()
    first = w.spawn(n)
    w.write_component(score, first, np.arange(n, dtype=np.uint32))
    w.write_component(health, first, np.full(n, 500, np.uint32))
    return score, health


def _exercise_particles(flags, cap, n):
    """The bundle (tile flags, content stamps) with downloads, a feed, host edits, the trace and queued submits; a
    growable engine grows behind its feed."""
    w = Engine(max_entities=cap, max_depth=8, flags=flags)
    t, v, l = _particles(w, n)
    w.trace_enable(64)
    fields = [(t, 0, 12), (v, 0, 12), (l, 0, 8)]
    feed = w.feed_create(fields)
    buf = w.feed_alloc(feed, 4 * cap)
    dst = w.host_alloc(n, 12)
    sess = P2PTraceSession(2, 8, 2, seed=1)
    for k in range(12):
        _tick(w, sess, (capi.BGR_INPUT_SPAWN if k % 3 == 0 else 0, 0))
        w.feed_wait(w.feed_begin(feed, buf, 4 * cap))
        w.download_wait(w.download_begin(v, 0, 12, 0, n, dst))
        if k == 6:
            edits = np.zeros(2, EDIT_DTYPE)
            edits["kind"] = capi.BGR_EDIT_SPAWN
            edits["count"] = (2000, 3000) if flags & GROW else (10, 20)
            w.apply_edits(edits)
            w.despawn(1)
    for _ in range(4):  # queued request vectors: overlapping launches through the tile flags
        for h in range(2):
            sess.add_local_input(h, 0)
        w.submit_requests(sess.info(), sess.advance_frame())
    for _ in range(4):
        w.collect()
    w.trace_read(64)
    if flags & GROW:
        assert w.capacity()[0] > cap
    w.close()


def _exercise_desync():
    """Desync capture: the diff scratch, the frame digest and the export of a frame."""
    w = Engine(max_entities=4096, max_depth=8, flags=capi.BGR_CFG_DESYNC_CAPTURE)
    _scores(w, 3000)
    sess = SyncTestSession(2, 7, 8, input_delay=2)
    for _ in range(16):
        _tick(w, sess, (0, 0))
    frames = w.snapshot_frames()
    assert frames
    for f in frames[:3]:
        w.desync_diff(f)
        d = w.frame_digest(f)
        if d is not None:
            w.export_blocks(f, list(range(d[0].n_blocks)))
    w.close()


def _exercise_remote_diff():
    """P2P desync reports: retained frames, digests, and a remote diff against another engine's export."""
    engines = []
    for seed in (5, 6):
        w = Engine(max_entities=4096, max_depth=8)
        w.retain_confirmed(4, 2)
        _scores(w, 3000)
        sess = P2PTraceSession(2, 8, seed=seed, p_clean=0.3)
        for _ in range(24):
            _tick(w, sess, (0, 0))
        engines.append(w)
    a, b = engines
    common = sorted(set(a.snapshot_frames() + a.retained_frames()) & set(b.snapshot_frames() + b.retained_frames()))
    assert common
    for f in common[:2]:
        d = b.frame_digest(f)
        blob = b.export_blocks(f, list(range(d[0].n_blocks)))
        a.diff_remote(f, blob)
        a.frame_digest(f)
    for w in engines:
        w.close()


def _exercise_generated_kernel(flags, cap):
    """The generated kernel with per-work-item dependencies (work-item flags) on queued submits."""
    saved = {k: os.environ.get(k) for k in ("BGR_TUNE_JIT", "BGR_TUNE_JIT_TILEDEP")}
    os.environ["BGR_TUNE_JIT"] = "2"
    os.environ["BGR_TUNE_JIT_TILEDEP"] = "1"
    try:
        w = Engine(max_entities=cap, max_depth=8, flags=flags)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    _scores(w, cap // 2)
    sess = P2PTraceSession(2, 8, 2, seed=2)
    queued = 0
    for k in range(10):
        for h in range(2):
            sess.add_local_input(h, 0)
        w.submit_requests(sess.info(), sess.advance_frame())
        queued += 1
        if k == 4 and flags & GROW:
            w.reserve(4 * cap)
        if queued > 3:
            w.collect()
            queued -= 1
    for _ in range(queued):
        w.collect()
    w.close()


def one_round():
    _exercise_particles(0, 8192, 6000)
    _exercise_particles(GROW, 4096, 3000)
    _exercise_desync()
    _exercise_remote_diff()
    _exercise_generated_kernel(0, 20000)
    _exercise_generated_kernel(GROW, 20000)


def refused_build():
    """A growable engine whose max_entities exceeds its ceiling: bgr_build refuses, then the engine is destroyed."""
    e = Engine(max_entities=1 << 22, max_depth=32, flags=GROW | capi.BGR_CFG_DESYNC_CAPTURE)
    for i in range(16):
        e.rollback_component(f"Wide{i}", 1024)
    with pytest.raises(BgrError) as ei:
        e.build()
    assert ei.value.status == capi.BGR_ERR_CAPACITY
    e.close()


def test_destroying_engines_releases_their_device_memory():
    one_round()
    after_first, why = process_device_bytes()
    for _ in range(ROUNDS - 1):
        one_round()
    after_last, _ = process_device_bytes()
    if after_first is None:
        pytest.skip(f"device memory of this process not measured: {why}")
    assert after_last == after_first, f"{after_last - after_first} bytes of device memory not released"


def test_destroying_an_engine_whose_build_was_refused():
    refused_build()  # once first: one-time costs
    before, why = process_device_bytes()
    refused_build()
    after, _ = process_device_bytes()
    if before is None:
        pytest.skip(f"device memory of this process not measured: {why}")
    assert after == before


if __name__ == "__main__":
    for _ in range(ROUNDS):
        one_round()
    refused_build()
    print("engine lifetime rounds done:", process_device_bytes())
