"""Worlds whose SyncTest re-simulation diverges on purpose, for the desync capture tests (oracle and GPU).

counter world  (tests/synctest.rs:83-125): Score (4 B, +1 per frame, deterministic, not checksummed) and Counter
               (8 B, optional, checksummed) into whose word 1 BGR_SYS_U32_STORE_CALL_COUNT writes a host-side call
               counter that is not rolled back.  Counter is removed at Startup from the rows r with r % 6 in (2, 5).
despawn world  Marker (4 B) and Health (4 B, optional, checksummed): the call counter is stored into Health, then
               BGR_SYS_U32_SATSUB_DESPAWN subtracts 1 and despawns at 0.  Health is inserted into the rows r with
               r % 6 in (1, 3) before the Save of frame 1: the first simulation of frame 1 -> 2 stores 1 and the rows
               die; the re-simulation stores a larger count and they survive.
               mixed=True adds a second counter system on Counter's word 0 and removes Counter from the rows r with
               r % 6 == 0 before the Save of frame 2 (the re-simulation from frame 1 still has it): frame 2 then has
               rows with two word records, rows with a presence record and rows with none.
Both take the row count: 6 rows fit one warp; LARGE_ROWS puts records in many warps of three tiles (512 rows each).

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.plugin import (App, GgrsPlugin, GgrsSchedule, LocalInputs, ReadInputs, Session, Startup,
                                   SyncTestMismatch, System)
from bevy_ggrs_b200.session import ADVANCE, SAVE, SyncTestSession

N_ROWS = 6
LARGE_ROWS = 1400


def counter_absent_rows(n_rows: int = N_ROWS) -> List[int]:
    return [r for r in range(n_rows) if r % 6 in (2, 5)]


def health_rows(n_rows: int = N_ROWS) -> List[int]:
    return [r for r in range(n_rows) if r % 6 in (1, 3)]


def _recording(backend, log: List[list]):
    """Log every request vector the backend executes (the test derives the call counter from them on its own)."""
    inner = backend.handle_requests

    def handle_requests(info, requests):
        reqs = list(requests)
        log.append(reqs)
        return inner(info, reqs)
    backend.handle_requests = handle_requests


def counter_app(backend, check_distance: int = 2, max_prediction: int = 8, n_rows: int = N_ROWS, mixed: bool = False):
    app = App(backend)
    app.insert_resource(Session.SyncTest(SyncTestSession(1, check_distance, max_prediction)))
    app.add_plugins(GgrsPlugin())
    score = app.rollback_component_with_copy("Score", 4)
    counter = app.rollback_optional_component_with_copy("Counter", 8)

    def read_inputs(a):
        if mixed and a.ticks == 2:  # before the Save of frame 2
            for r in range(0, n_rows, 6):
                a.world.remove_component(counter, r)
        a.insert_resource(LocalInputs({h: 0 for h in a.local_players.handles}))
    app.add_systems(ReadInputs, read_inputs)
    app.checksum_component_with_hash(counter)
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_U32_ADD, [score], [0, 1]))
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_U32_STORE_CALL_COUNT, [counter], [4]))
    if mixed:
        app.add_systems(GgrsSchedule, System(capi.BGR_SYS_U32_STORE_CALL_COUNT, [counter], [0]))

    def setup(a):
        first = a.world.spawn(n_rows)
        a.world.write_component(score, first, np.zeros(n_rows, np.uint32))
        for r in counter_absent_rows(n_rows):
            a.world.remove_component(counter, first + r)
    app.add_systems(Startup, setup)
    return app, score, counter


def despawn_app(backend, check_distance: int = 3, max_prediction: int = 8, n_rows: int = N_ROWS):
    app = App(backend)
    app.insert_resource(Session.SyncTest(SyncTestSession(1, check_distance, max_prediction)))
    app.add_plugins(GgrsPlugin())
    marker = app.rollback_component_with_copy("Marker", 4)
    health = app.rollback_optional_component_with_copy("Health", 4)
    app.checksum_component_with_hash(health)
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_U32_STORE_CALL_COUNT, [health], [0]))
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1]))

    def setup(a):
        first = a.world.spawn(n_rows)
        a.world.write_component(marker, first, np.arange(n_rows, dtype=np.uint32))
        for r in range(n_rows):
            a.world.remove_component(health, first + r)

    def read_inputs(a):
        if a.ticks == 1:  # before the Save of frame 1
            for r in health_rows(n_rows):
                a.world.insert_component(health, r, np.array([100], np.uint32))
        a.insert_resource(LocalInputs({h: 0 for h in a.local_players.handles}))
    app.add_systems(Startup, setup)
    app.add_systems(ReadInputs, read_inputs)
    return app, marker, health


def run_to_first_mismatch(app, max_updates: int = 20, max_records: int = 64):
    """Update until SyncTestMismatch fires; the observer asks for a report of every mismatched frame.  Returns
    (event, {frame: report}, request vectors executed so far)."""
    log: List[list] = []
    app._finish()
    _recording(app.world, log)
    seen = []

    def on_mismatch(ev: SyncTestMismatch):
        if not seen:
            seen.append((ev, {f: app.desync_report(f, max_records) for f in ev.mismatched_frames}))
    app.add_observer(SyncTestMismatch, on_mismatch)
    for _ in range(max_updates):
        app.update()
        if seen:
            break
    assert seen, "SyncTestMismatch did not fire"
    ev, reports = seen[0]
    return ev, reports, log


def counter_values_by_save(log: List[list]) -> Dict[int, List[int]]:
    """Value of the call counter in every Save of each frame, in execution order: every Advance stores the number of
    Advances executed before it into every row that has Counter, and a Save keeps what the last Advance stored."""
    n_adv, last, out = 0, 0, {}
    for vec in log:
        for r in vec:
            if r.kind == ADVANCE:
                last, n_adv = n_adv, n_adv + 1
            elif r.kind == SAVE:
                out.setdefault(r.frame, []).append(last)
    return out
