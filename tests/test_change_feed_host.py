"""CPU checks of the change feed: its ABI agrees across the header, ctypes and the Rust declarations, and the numpy
model (change_feed_model.py) that the GPU tests hold the engine to reproduces oracle worlds with exactly the differing
rows, under every cap."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request
from change_feed_model import FeedModel, Replica, host_edits, world_of
from oracle_backend import OracleWorld

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)


def test_feed_abi_agrees_across_header_ctypes_and_rust():
    hdr = open(os.path.join(ROOT, "include", "bevy_ggrs_b200.h")).read()
    rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200_sys", "src", "change_feed.rs")).read()
    consts = {k: int(v) for k, v in re.findall(r"#define (BGR_MAX_FEED\w*) (\d+)u", hdr)}
    assert consts == {"BGR_MAX_FEEDS": 8, "BGR_MAX_FEED_FIELDS": 8}
    for k, v in consts.items():
        assert getattr(capi, k) == v
        assert re.search(r"pub const %s: u32 = %d;" % (k, v), rs), k
    assert C.sizeof(capi.bgr_feed_field) == 12 and C.sizeof(capi.bgr_feed_info) == 16
    for struct in ("bgr_feed_field", "bgr_feed_info"):
        c_body = re.search(r"typedef struct %s \{(.*?)\}" % struct, hdr, re.S).group(1)
        c_fields = re.findall(r"(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", c_body).replace("uint32_t", ""))
        rs_body = rs[rs.index("pub struct " + struct):]
        rs_fields = re.findall(r"pub (\w+): u32,", rs_body[:rs_body.index("}")])
        assert c_fields == rs_fields == [f for f, _ in getattr(capi, struct)._fields_], struct


def _world(seed, n=700):
    """An oracle world with one optional column and systems that write one field of each, and despawn."""
    rng = np.random.default_rng(seed)
    w = OracleWorld()
    a = w.rollback_component("A", 12, capi.BGR_STRATEGY_COPY)
    b = w.rollback_component("B", 8, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)
    w.add_system(capi.BGR_SYS_U32_ADD, [a], [4, 1])
    w.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [b], [0, 3])
    w.build()
    w.spawn(n)
    w.write_component(a, 0, rng.integers(0, 256, (n, 12), dtype=np.uint8))
    bv = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    bv.view(np.uint32)[:, 0] = rng.integers(1, 60, n, dtype=np.uint32)
    w.write_component(b, 0, bv)
    for r in rng.choice(n, n // 5, replace=False):
        w.remove_component(b, int(r))
    return w, a, b, rng


def test_model_records_rebuild_oracle_worlds_through_rollbacks():
    w, a, b, rng = _world(1)
    fields = [(a, 0, 4), (a, 4, 8), (b, 0, 8)]
    model = FeedModel(fields, 4096)
    rep = Replica(len(fields), [4, 8, 8], 4096)
    prev, fc = None, 0
    for f in range(30):
        w.handle_requests(NOSESS, [Request(SAVE, fc), Request(ADVANCE, fc, [0])])
        fc += 1
        if f % 7 == 6:  # resurrect rows that the ticks since despawned, and un-spawn the rows spawned since
            fc -= 3
            w.handle_requests(NOSESS, [Request(LOAD, fc)])
        if f % 5 == 2:
            host_edits([w], rng, b, a, 12)
        world = world_of(w, [a, b])
        diff = model.differing(world)
        recs, info = model.report(world, 1 << 20)
        assert info.pending == 0 and np.array_equal(recs["row"], diff)
        if prev is not None:  # the records are exactly the rows whose (state, bytes) differ from the last report
            s0, b0 = prev
            s1, b1 = model.current(world)
            want = np.nonzero((s0 != s1) | np.any([(x != y).any(axis=1) for x, y in zip(b0, b1)], axis=0))[0]
            assert np.array_equal(recs["row"], want)
        prev = model.current(world)
        rep.apply(recs)
        assert rep.matches(model, world)
        assert info.record_bytes == 8 + 4 + 8 + 8
    assert w.row_count() > 700 and w.active_count() < w.row_count()


@pytest.mark.parametrize("cap", [0, 1, 7, 31, 32, 33, 511, 512, 513, 10_000])
def test_model_capped_reports_concatenate_to_one_uncapped_report(cap):
    w, a, b, _ = _world(3, n=1500)
    fields = [(a, 8, 4), (b, 0, 4)]
    world = world_of(w, [a, b])
    full, finfo = FeedModel(fields, 2048).report(world, 1 << 20)
    m = FeedModel(fields, 2048)
    got, rounds = [], 0
    while True:
        recs, info = m.report(world, cap)
        assert info.n_records == min(cap, info.n_records + info.pending)
        got.append(recs)
        rounds += 1
        if info.pending == 0 or cap == 0:
            break
    if cap == 0:
        assert info.pending == finfo.n_records and len(got[0]) == 0
        return
    cat = np.concatenate(got)
    assert cat.tobytes() == full.tobytes()
    assert rounds == max(1, -(-finfo.n_records // cap))
    assert m.report(world, cap)[1].n_records == 0
