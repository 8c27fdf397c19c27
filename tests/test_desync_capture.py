"""Desync capture without a GPU: the ring's witness bookkeeping (bgr_ring_create_capture, the same SlotRing class the
engine runs) and the oracle's restatement of capture + diff driven through the plugin mirror."""
import ctypes as C
import inspect

import numpy as np
import pytest

import test_ring_kats as kats
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.desync import NO_INDEX
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, SyncTestSession
from desync_util import (LARGE_ROWS, N_ROWS, counter_absent_rows, counter_app, counter_values_by_save, despawn_app,
                         health_rows, run_to_first_mismatch)
from oracle_desync import CaptureOracleWorld
from ring_adapters import EngineRing


class CaptureRing(EngineRing):
    """bgr_ring_* of a ring created with desync capture; the payload per slot stands for the HBM image."""

    def __init__(self, depth=None, n_slots=64):
        self.lib = capi.load_library()
        self.cap = n_slots
        self.h = C.c_void_p(self.lib.bgr_ring_create_capture(n_slots))
        self.payload = {}
        if depth is not None:
            self.set_depth(depth)

    def push_slot(self, frame, value):
        slot = C.c_uint32()
        assert self.lib.bgr_ring_push(self.h, frame, C.byref(slot)) == 0, self._err()
        self.payload[slot.value] = value
        return slot.value

    def first(self, frame):
        slot, found = C.c_uint32(), C.c_int32()
        self.lib.bgr_ring_first(self.h, frame, C.byref(slot), C.byref(found))
        return slot.value if found.value else None

    def slots_in_use(self):
        n = C.c_uint32()
        self.lib.bgr_ring_slots_in_use(self.h, C.byref(n))
        return n.value


class PlainRing(EngineRing):
    def __init__(self, depth, n_slots):
        self.lib = capi.load_library()
        self.cap = n_slots
        self.h = C.c_void_p(self.lib.bgr_ring_create(n_slots))
        self.payload = {}
        self.set_depth(depth)


REFERENCE_KATS = [n for n, f in vars(kats).items()
                  if n.startswith("test_") and callable(f) and "snap_with_depth" in inspect.signature(f).parameters]


def test_all_reference_ring_kats_are_collected():
    assert len(REFERENCE_KATS) >= 11


@pytest.mark.parametrize("name", REFERENCE_KATS)
def test_reference_ring_kats_hold_on_a_capture_ring(name):
    getattr(kats, name)(lambda depth: CaptureRing(depth))


def _synctest_requests(d, maxp, ticks):
    sess = SyncTestSession(1, d, maxp)
    for _ in range(ticks):
        sess.add_local_input(0, 0)
        reqs = sess.advance_frame()
        for r in reqs:
            if r.kind == SAVE:
                sess.save_cell(r.frame, 0)
        yield reqs


@pytest.mark.parametrize("d", range(1, 8))
def test_synctest_witness_bookkeeping(d):
    """The engine's per-request ring calls (compile_requests: sync_depth, confirm, push / rollback) over SyncTest
    request streams, on a plain ring of max_depth slots and a capture ring of 2 * max_depth."""
    for maxp in range(d + 1, 9):
        plain, cap = PlainRing(maxp, maxp), CaptureRing(maxp, 2 * maxp)
        frame_count, confirmed, n_push, most = 0, 0, 0, 0
        first_slot = {}
        for reqs in _synctest_requests(d, maxp, 40):
            for r in reqs:
                cf = frame_count - d
                if cf >= 0:
                    confirmed = cf
                if r.kind == SAVE:
                    for ring in (plain, cap):
                        ring.set_depth(maxp)
                        ring.confirm(confirmed)
                    first_slot = {f: s for f, s in first_slot.items() if f >= confirmed}
                    pinned = {cap.first(f) for f in first_slot} - {None}
                    value = (frame_count, n_push)
                    n_push += 1
                    plain.push(frame_count, value)
                    slot = cap.push_slot(frame_count, value)
                    assert slot not in pinned, ("a pinned slot was handed out", d, maxp, r)
                    first_slot.setdefault(frame_count, slot)
                    most = max(most, cap.slots_in_use())
                elif r.kind == LOAD:
                    frame_count = r.frame
                    plain.rollback(r.frame)
                    cap.rollback(r.frame)
                    assert plain.get() == cap.get()
                else:
                    frame_count += 1
                for f in range(max(0, frame_count - 12), frame_count + 2):
                    assert plain.peek(f) == cap.peek(f), (d, maxp, f)
                for f, s in first_slot.items():
                    assert cap.first(f) == s, (d, maxp, f)
                    assert cap.payload[s][0] == f
        # the bound of ring.hpp, reached exactly: 2(d+1) <= 2 * max_depth (d = 1 re-saves no frame: 2 slots)
        assert most == (2 * (d + 1) if d >= 2 else 2) and most <= 2 * maxp, (d, maxp, most)


def test_shortage_releases_the_oldest_witness_instead_of_failing():
    ring = CaptureRing(4, n_slots=4)
    slots = [ring.push_slot(f, f) for f in range(4)]
    ring.rollback(0)                      # frames 1..3 leave the queue; their first images stay pinned
    assert [ring.first(f) for f in range(4)] == slots and ring.slots_in_use() == 4
    s = ring.push_slot(1, 10)             # no free slot: witnesses go, oldest first, until one is free
    assert ring.first(0) is None and ring.first(1) == s
    assert ring.first(2) == slots[2] and ring.first(3) == slots[3]
    assert ring.peek(0) == 0 and ring.peek(1) == 10
    plain = PlainRing(4, 4)
    for f in range(4):
        plain.push(f, f)
    plain.rollback(0)
    plain.push(1, 10)
    assert [plain.peek(f) for f in range(4)] == [ring.peek(f) for f in range(4)]


# ---- the oracle's capture and diff, through plugin.App ----
@pytest.mark.parametrize("n", [N_ROWS, LARGE_ROWS])
def test_oracle_report_names_the_counter_column_and_word(n):
    app, score, counter = counter_app(CaptureOracleWorld(), n_rows=n)
    ev, reports, log = run_to_first_mismatch(app, max_records=2 * n)
    values = counter_values_by_save(log)
    assert app.world.desync_frames()
    for f in ev.mismatched_frames:
        rep = reports[f]
        assert rep is not None and rep.frame == f
        recs = rep.records
        present_rows = [r for r in range(n) if r not in counter_absent_rows(n)]
        first, latest = values[f][0], values[f][-1]
        assert first != latest
        assert list(recs["row"]) == present_rows
        assert set(recs["column"]) == {counter} and set(recs["word"]) == {1}
        assert set(recs["first"]) == {first} and set(recs["latest"]) == {latest}
        assert rep.columns[counter].rows == len(present_rows) == rep.columns[counter].rows_in_checksum
        assert rep.columns[score].rows == 0 and rep.by_name["Counter"].presence == 0
        assert rep.rows_differing == rep.words_differing == len(present_rows) and rep.existence_differing == 0
        assert rep.host_state_differs == 0 and rep.rows_first == rep.rows_latest == n
        # the retained first image is what the first simulation saved
        data, alive = app.world.peek_first(f, counter, 0, n)
        assert list(np.nonzero(alive)[0]) == present_rows
        assert set(data.view("<u4")[alive.astype(bool), 1]) == {first}


@pytest.mark.parametrize("n", [N_ROWS, LARGE_ROWS])
def test_oracle_report_shows_a_row_that_died_only_in_the_first_simulation(n):
    app, marker, health = despawn_app(CaptureOracleWorld(), n_rows=n)
    ev, reports, _ = run_to_first_mismatch(app, max_records=4 * n)
    assert 2 in ev.mismatched_frames
    rep = reports[2]
    ex = rep.records[rep.records["column"] == NO_INDEX]
    assert list(ex["row"]) == health_rows(n)
    assert set(ex["word"]) == {NO_INDEX}
    assert set(ex["first"]) == {0} and set(ex["latest"]) == {1}  # dead, then alive with Health present
    assert rep.existence_differing == len(health_rows(n))
    assert rep.columns[marker].rows == 0


def test_capture_ring_refuses_nothing_the_plain_ring_accepts_on_deep_p2p_rollbacks():
    from bevy_ggrs_b200.session import P2PTraceSession
    maxp = 8
    sess = P2PTraceSession(2, maxp, seed=7, p_clean=0.2)
    plain, cap = PlainRing(maxp, maxp), CaptureRing(maxp, 2 * maxp)
    frame_count = 0
    for _ in range(200):
        sess.add_local_input(0, 0)
        reqs = sess.advance_frame()
        confirmed = sess.confirmed_frame()
        for r in reqs:
            if r.kind == SAVE:
                for ring in (plain, cap):
                    ring.set_depth(maxp)
                    ring.confirm(confirmed)
                plain.push(frame_count, frame_count)
                cap.push(frame_count, frame_count)
            elif r.kind == LOAD:
                frame_count = r.frame
                plain.rollback(r.frame)
                cap.rollback(r.frame)
            else:
                frame_count += 1
        for f in range(frame_count - 10, frame_count + 1):
            assert plain.peek(f) == cap.peek(f)


def test_engine_create_refuses_capture_beyond_32_slots_and_on_sharded_engines():
    """Checked before any device is touched, so this holds on a CPU-only box too."""
    from bevy_ggrs_b200.capi import BgrError
    from bevy_ggrs_b200.engine import Engine
    cap = capi.BGR_CFG_DESYNC_CAPTURE
    with pytest.raises(BgrError) as ei:
        Engine(max_entities=16, max_depth=33, flags=cap)
    assert ei.value.status == capi.BGR_ERR_INVALID_ARGUMENT and "max_depth <= 32" in str(ei.value)
    with pytest.raises(BgrError) as ei:
        Engine(max_entities=16, max_depth=8, flags=cap | capi.BGR_CFG_SHARDED)
    assert ei.value.status == capi.BGR_ERR_UNSUPPORTED
