"""Checkpoint deltas on the H100 (bgr_checkpoint_save_delta / bgr_checkpoint_restore_delta): the GPU delta equals the
numpy restatement (checkpoint_delta_codec.py) applied to the two frames' full checkpoints, byte for byte, and is the
same on a twin engine whose dead rows hold other bytes; an engine restored from base plus delta equals one restored from
the target's full checkpoint (digests, checkpoints, reads, the ring) and continues like it, and like the oracle restored
from that checkpoint; every refusal leaves the live world and the ring unchanged.  On the interpreter, the generated
kernel with whole tiles and with 128-row items, the particles bundle and BGR_CFG_FORCE_STEPWISE; the App mirrors in
Python and C++ continue a match restored from base plus delta."""
import os
import subprocess
import sys

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, SAVE, P2PTraceSession, Request
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
import checkpoint_codec as cc
import checkpoint_delta_codec as dc
from interleave_driver import NOSESS, FlagsOracle
from test_gpu_checkpoint import (P2P_INFO, _frame_count_app, drive, observe, particles_engine, presence_engine,
                                 run_script, script)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPT = capi.BGR_STRATEGY_OPTIONAL

# kernel -> (environment, engine flags); the generic program runs the presence world, the bundle the particles world
KERNELS = {
    "interpreter": ({"BGR_TUNE_JIT": "0"}, 0),
    "jit_whole_tiles": ({"BGR_TUNE_JIT": "2", "BGR_TUNE_JIT_ITEM": "512"}, 0),
    "jit_quarter_tiles": ({"BGR_TUNE_JIT": "2"}, 0),
    "particles_bundle": ({}, 0),
    "stepwise": ({}, capi.BGR_CFG_FORCE_STEPWISE),
}


def make(kernel, n=1400, garbage=False):
    """A world for `kernel`, driven the same way each time.  ``garbage``: the dead rows hold other bytes."""
    env, flags = KERNELS[kernel]
    if kernel in ("particles_bundle", "stepwise"):
        e, cols = particles_engine(n, flags=flags)
        populate(e, cols, *synth_particles(n, 2, 5, 80, z_fraction=0.2))
        for r in range(7, n, 61):
            if garbage:
                e.write_component(cols[1], r, np.full((1, 3), 7.5, np.float32))
            e.despawn(r)
        drive(e, 30, seed=3, spawn_every=3)
    else:
        e = presence_engine(n, env=env)
        for r in range(11, n, 71):
            if garbage:
                e.write_component(2, r, np.full((1, 3), 0xABCDEF, np.uint32))
            e.despawn(r)
        drive(e, 30, seed=3)
    return e


def reference_delta(eng, frame, base_frame):
    """The numpy delta of the two frames' full checkpoints (each checked by the numpy decoder)."""
    full, base = eng.checkpoint(frame), eng.checkpoint(base_frame)
    th, tp, tm = cc.decode(full)
    bh, bp, bm = cc.decode(base)
    ref = dc.encode((tp, tm), (bp, bm), layout=th["layout"], frame=frame, rows=th["rows"], base_frame=base_frame,
                    base_rows=bh["rows"], n_columns=th["n_columns"], fps=th["fps"], active=th["active"],
                    elapsed_ns=th["elapsed_ns"], rng=th["rng"], digest_root=th["digest_root"], base_root=bh["digest_root"])
    return full, base, ref


def pairs(eng):
    """(target, base): a later target, a later base, base == target."""
    q, ret = eng.snapshot_frames(), eng.retained_frames()
    held = sorted(set(q) | set(ret))
    assert len(held) >= 3
    return [(held[-1], held[0]), (held[0], held[-1]), (held[len(held) // 2], held[len(held) // 2])]


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_delta_equals_the_restatement_and_restores_the_target(kernel):
    a, twin = make(kernel), make(kernel, garbage=True)
    for f, g in pairs(a):
        full, base, ref = reference_delta(a, f, g)
        delta = a.checkpoint_delta(f, g)
        assert delta == ref, (f, g)
        assert twin.checkpoint_delta(f, g) == delta, (f, g)   # dead rows' bytes are not part of a delta
        if f == g:   # every vector CONST zero
            assert not any(delta[120 + 8 * (dc.unpack_header(delta)["n_blocks"] + 1):])
        x, y = make(kernel), make(kernel)
        x.restore_delta(base, delta)
        y.restore(full)
        assert x.snapshot_frames() == y.snapshot_frames() == [f]
        assert x.checkpoint(f) == full
        assert observe(x, 3) == observe(y, 3)
        vecs = script(f, 16, seed=f)
        assert run_script(x, vecs) == run_script(y, vecs)
        assert observe(x, 3) == observe(y, 3)
    # rows differ between the frames of the spawning particles world
    if kernel in ("particles_bundle", "stepwise"):
        rows = {cc.unpack_header(a.checkpoint(f))["rows"] for f, _ in pairs(a)}
        assert len(rows) > 1


def test_growable_spawning_world():
    a, cols = particles_engine(600, cap=1024, flags=capi.BGR_CFG_GROWABLE)
    populate(a, cols, *synth_particles(600, 4, 5, 80, z_fraction=0.2))
    drive(a, 60, seed=5, spawn_every=2)
    held = sorted(set(a.snapshot_frames()) | set(a.retained_frames()))
    f, g = held[-1], held[0]
    full, base, ref = reference_delta(a, f, g)
    assert cc.unpack_header(full)["rows"] > cc.unpack_header(base)["rows"]
    for t, b in ((f, g), (g, f)):
        full_t, base_b, ref_tb = reference_delta(a, t, b)
        assert a.checkpoint_delta(t, b) == ref_tb
        x, _ = particles_engine(100, cap=512, flags=capi.BGR_CFG_GROWABLE, retain=None)
        y, _ = particles_engine(100, cap=512, flags=capi.BGR_CFG_GROWABLE, retain=None)
        x.restore_delta(base_b, a.checkpoint_delta(t, b))
        y.restore(full_t)
        assert observe(x, 3) == observe(y, 3) and x.capacity()[0] >= cc.unpack_header(full_t)["rows"]
        vecs = script(t, 12, seed=t)
        assert run_script(x, vecs) == run_script(y, vecs)
        assert observe(x, 3) == observe(y, 3)


def _presence_oracle(n):
    o = FlagsOracle(max_entities=n + 64, max_depth=9)
    score = o.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | OPT)
    health = o.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | OPT)
    tag = o.rollback_component("Tag", 12)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        o.checksum_component(c, 0, ln)
    o.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    o.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    o.build()
    return o


def test_presence_flips_continue_like_the_oracle():
    a = presence_engine(1400, env=KERNELS["interpreter"][0])
    sess = P2PTraceSession(2, 8, seed=3, p_clean=0.3)

    def ticks(k):
        for _ in range(k):
            for h in range(sess.num_players()):
                sess.add_local_input(h, 0)
            for fr, c in a.handle_requests(sess.info(), sess.advance_frame()):
                sess.save_cell(fr, c)
    ticks(30)
    score, health = 0, 1
    f0 = a.snapshot_frames()[0]   # the newest
    alive = a.read_alive(0, 600)
    for r in range(20, 600, 13):   # presence flips between the frames
        if not alive[r]:
            continue
        if a.has_component(score, r, 1)[0]:
            a.remove_component(score, r)
        else:
            a.insert_component(score, r, np.uint32(5))
        if a.has_component(health, r, 1)[0]:
            a.remove_component(health, r)
    ticks(3)
    f = a.snapshot_frames()[0]
    assert f != f0 and f0 in a.snapshot_frames() + a.retained_frames()
    full, base, ref = reference_delta(a, f, f0)
    delta = a.checkpoint_delta(f, f0)
    assert delta == ref
    x = presence_engine(1400)
    x.restore_delta(base, delta)
    o = _presence_oracle(1400)
    o.restore(full)
    x.set_depth(8)
    o.set_depth(8)
    rng = np.random.default_rng(4)
    for i in range(12):
        g = x.rollback_frame_count()
        reqs = [Request(SAVE, g), Request(ADVANCE, 0, [int(rng.integers(0, 4))])]
        assert x.handle_requests(NOSESS, reqs) == o.handle_requests(NOSESS, reqs), f"vector {i}"
    rows = x.row_count()
    assert rows == o.row_count() and x.active_count() == o.active_count()
    for c in range(3):
        has = x.has_component(c, 0, rows).astype(bool)
        v, ohas = o.read_component_alive(c, 0, rows)
        assert np.array_equal(has, np.asarray(ohas).astype(bool)), c


# ---- refusals ----
def _state(e):
    return observe(e, len(e.elem_bytes)), e.retained_frames()


def _refused(e, base, delta, status, what=""):
    before = _state(e)
    with pytest.raises(BgrError) as ei:
        e.restore_delta(base, delta)
    assert ei.value.status == status, (what, str(ei.value))
    assert _state(e) == before, what


def test_refusals_leave_the_engine_unchanged():
    a = make("jit_quarter_tiles")
    held = sorted(set(a.snapshot_frames()) | set(a.retained_frames()))
    f, g = held[-1], held[0]
    full, base, delta = reference_delta(a, f, g)
    assert a.checkpoint_delta(f, g) == delta
    b = presence_engine(1400)
    drive(b, 9, seed=7)
    inv = capi.BGR_ERR_INVALID_ARGUMENT
    _refused(b, a.checkpoint(held[1]), delta, inv, "another frame's checkpoint as the base")
    _refused(b, full, delta, inv, "the target's checkpoint as the base")
    _refused(b, base, full, inv, "a full checkpoint as the delta")
    h = dc.unpack_header(delta)
    for field, val in (("magic", 1), ("version", 2), ("layout", h["layout"] ^ 1), ("rows", h["rows"] - 1),
                       ("base_frame", h["base_frame"] + 1), ("base_rows", h["base_rows"] - 1), ("words", h["words"] + 1),
                       ("n_blocks", h["n_blocks"] + 1), ("n_columns", 4), ("fps", 30), ("active", h["active"] + 1),
                       ("digest_root", h["digest_root"] ^ 1), ("base_root", h["base_root"] ^ 1),
                       ("payload_bytes", h["payload_bytes"] + 4)):
        _refused(b, base, dc.pack_header({**h, field: val}) + delta[120:], inv, field)
    _refused(b, base, delta[:-4], inv, "truncated")
    _refused(b, base, delta + bytes(4), inv, "overlong")
    _refused(b, base, delta[:100], inv, "shorter than its header")
    _refused(b, base[:-4], delta, inv, "a truncated base")
    prefix = 120 + 8 * (h["n_blocks"] + 1)
    words = h["words"]   # 5: six kind bytes and two of padding
    for at, val, what in ((0, 3, "a kind byte > 2"), (words + 1, 1, "non-zero padding")):
        bad = bytearray(delta)
        bad[prefix + at] = val
        _refused(b, base, bytes(bad), inv, what)
    # targets that are not canonical, coded by the restatement against the same base
    _, bp, bm = cc.decode(base)
    th, tp, tm = cc.decode(full)
    fields = {k: h[k] for k in dc.HEADER_FIELDS if k not in ("magic", "version", "words", "n_blocks", "payload_bytes")}
    tp, tm = dc.widen(tp, tm, h["n_blocks"])
    dead = int(np.nonzero((tm[0] & 1) == 0)[0][0])
    live = int(np.nonzero(tm[0] == 1)[0][0])
    lacks = int(np.nonzero(tm[0] == 3)[0][0])   # alive, Score absent
    cases = []
    p = tp.copy(); p[0, 2, dead] = 9
    cases.append(("a word of a row that does not exist", p, tm))
    m = tm.copy(); m[0, live] |= 0x80
    cases.append(("an unknown presence bit", tp, m))
    p = tp.copy(); p[0, 0, lacks] = 9
    cases.append(("a word of a column the row lacks", p, tm))
    if h["rows"] < h["n_blocks"] * cc.BLOCK:
        m = tm.copy(); m[-1, cc.BLOCK - 1] = 1
        cases.append(("a row past the target's rows", tp, m))
    for what, p, m in cases:
        _refused(b, base, dc.encode((p, m), (bp, bm), **fields), inv, what)
    # un-collected submits, then the world moves on like its twin
    b.submit_requests(P2P_INFO, [Request(ADVANCE, 0, [0, 0], [0, 0])])
    with pytest.raises(BgrError) as ei:
        b.restore_delta(base, delta)
    assert ei.value.status == capi.BGR_ERR_STATE
    b.collect()
    b.restore_delta(base, delta)   # the same pair restores once the submits are collected
    assert b.checkpoint(f) == full
    # frames that are not held: nothing runs
    assert a.checkpoint_delta(10**6, g) is None and a.checkpoint_delta(f, 10**6) is None
    sharded = Engine(max_entities=2048, max_depth=9, flags=capi.BGR_CFG_SHARDED)
    register_particles(sharded)
    sharded.build()
    for call in (lambda: sharded.restore_delta(base, delta), lambda: sharded.checkpoint_delta(0, 0)):
        with pytest.raises(BgrError) as ei:
            call()
        assert ei.value.status == capi.BGR_ERR_UNSUPPORTED


def test_refuses_bits_past_a_sub_word_element():
    def mk():
        e = Engine(max_entities=1200, max_depth=9)
        odd = e.rollback_component("Odd", 5, capi.BGR_STRATEGY_COPY)
        e.checksum_component(odd, 0, 5)
        e.build()
        e.set_depth(8)
        e.spawn(1000)
        e.write_component(odd, 0, np.random.default_rng(3).integers(0, 256, (1000, 5), dtype=np.uint8))
        return e
    eng, other = mk(), mk()
    for _ in range(3):
        f = eng.rollback_frame_count()
        eng.handle_requests(NOSESS, [Request(SAVE, f), Request(ADVANCE, 0, [0])])
    g, f = eng.snapshot_frames()[0], eng.snapshot_frames()[-1]
    full, base, delta = reference_delta(eng, f, g)
    h = dc.unpack_header(delta)
    _, bp, bm = cc.decode(base)
    _, tp, tm = cc.decode(full)
    tp[1, 1, 700 - 512] |= np.uint32(1 << 8)   # a bit past byte 5 of the column, on a live row
    fields = {k: h[k] for k in dc.HEADER_FIELDS if k not in ("magic", "version", "words", "n_blocks", "payload_bytes")}
    _refused(other, base, dc.encode((tp, tm), (bp, bm), **fields), capi.BGR_ERR_INVALID_ARGUMENT, "stray bit")
    other.restore_delta(base, delta)
    assert other.checkpoint(f) == full


# ---- the App mirrors ----
def test_python_app_restored_from_base_plus_delta_continues():
    import copy
    from bevy_ggrs_b200.plugin import Session
    from bevy_ggrs_b200.session import SyncTestSession
    d = 3
    sa, mis = SyncTestSession(1, d, 9), []
    a = _frame_count_app(sa, mis)
    for _ in range(20):
        a.step()
    while (sa.current_frame - d) % 4:
        a.step()
    fb = sa.current_frame - d
    base = a.checkpoint(fb)
    for _ in range(5):
        a.step()
    f = sa.current_frame - d
    assert fb in a.world.retained_frames() or fb in a.world.snapshot_frames()
    delta, full = a.checkpoint_delta(f, fb), a.checkpoint(f)
    with pytest.raises(BgrError) as ei:   # the App holds no resources of the base frame any more
        a.checkpoint_delta(fb, f)
    assert ei.value.status == capi.BGR_ERR_NO_SNAPSHOT
    b = _frame_count_app(SyncTestSession(1, d, 9), mis)
    c = _frame_count_app(SyncTestSession(1, d, 9), mis)
    b.step()
    before = (b.world.snapshot_frames(), dict(b.resources))
    for bb, bd in ((base, delta[:-1]), (base, delta + b"\0"), (base[:-1], delta), (full, delta)):
        with pytest.raises(BgrError) as ei:
            b.restore_checkpoint_delta(bb, bd)
        assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT
    assert (b.world.snapshot_frames(), dict(b.resources)) == before
    b.restore_checkpoint_delta(base, delta)
    c.restore_checkpoint(full)
    assert b.checkpoint(f) == full
    b.insert_resource(Session.SyncTest(copy.deepcopy(sa)))
    c.insert_resource(Session.SyncTest(copy.deepcopy(sa)))
    for _ in range(20):
        a.step()
        b.step()
        c.step()
        assert a.last_checksums == b.last_checksums == c.last_checksums
    assert not mis and a.resources == b.resources == c.resources


def test_cpp_app_restored_from_base_plus_delta_continues(tmp_path):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    lib = g.build_engine()
    out = str(tmp_path / "test_checkpoint_delta")
    src = os.path.join(ROOT, "tests", "cpp", "test_checkpoint_delta.cpp")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-ffp-contract=off", "-o", out, src,
                        "-L" + os.path.dirname(lib), "-lbevy_ggrs_b200", "-Wl,-rpath," + os.path.dirname(lib)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "checkpoint delta test passed" in r.stdout
