"""Shared drivers for parity tests: run the same seeded workload on the CUDA engine (through the
C ABI) and on the oracle, and compare bit for bit."""
from __future__ import annotations

import numpy as np

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.plugin import (App, GgrsPlugin, LocalInputs, ReadInputs, RollbackFrameRate, Session,
                                   SyncTestMismatch)
from bevy_ggrs_b200.session import P2PTraceSession, SyncTestSession
from bevy_ggrs_b200.stress import populate, register_particles, synth_particles
from oracle_backend import OracleWorld


def input_system(app):
    """tests/common/mod.rs:16-22: zero input for every local player."""
    app.insert_resource(LocalInputs({h: 0 for h in app.local_players.handles}))


def make_particles_app(backend, n_entities, seed, session, ttl_lo, ttl_hi, noop_inputs=False, spawn_rate=0,
                       spawn_ttl=300, startup_burst=False, z_fraction=0.0, checksums=None):
    app = App(backend)
    app.add_plugins(GgrsPlugin())
    app.insert_resource(RollbackFrameRate(60))
    if spawn_rate:
        # INPUT_SPAWN = 1 << 4 held by player 0 on two frames out of five, INPUT_NOOP noise on player 1
        def read(app_):
            app_.insert_resource(LocalInputs({h: ((1 << 4) if (h == 0 and app_.ticks % 5 in (1, 2)) else 0) |
                                              ((1 << 5) if (app_.ticks + h) % 3 == 0 else 0)
                                              for h in app_.local_players.handles}))
        app.add_systems(ReadInputs, read)
    elif noop_inputs:
        # INPUT_NOOP = 1 << 5 on a seeded schedule (particles.rs:75-76): inputs never change the simulation
        def read(app_):
            app_.insert_resource(LocalInputs({h: (1 << 5) if (app_.ticks + h) % 3 == 0 else 0
                                              for h in app_.local_players.handles}))
        app.add_systems(ReadInputs, read)
    else:
        app.add_systems(ReadInputs, input_system)
    cols = register_particles(backend, spawn_rate=spawn_rate, spawn_ttl=spawn_ttl, checksums=checksums)
    app.insert_resource(session)
    mism = []
    app.add_observer(SyncTestMismatch, lambda ev: mism.append(ev))
    app._finish()
    tf, vel, ttl = synth_particles(n_entities, seed, ttl_lo, ttl_hi, z_fraction)
    populate(backend, cols, tf, vel, ttl)
    if startup_burst:
        backend.run_startup_system(capi.BGR_SYS_PARTICLES_SPAWN)  # add_systems(Startup, spawn_particles), particles.rs:232
    return app, cols, mism


def compare_state(eng, orc, cols, n):
    """Live columns + alive mask, bit for bit (dead rows' stale bytes are not observable)."""
    ok = True
    alive_e = eng.read_alive(0, n)
    for c in cols:
        de = eng.read_component(c, 0, n)
        do, alive_o = orc.read_component_alive(c, 0, n)
        if not np.array_equal(alive_e.astype(bool), alive_o.astype(bool)):
            return False
        m = alive_o.astype(bool)
        ok = ok and np.array_equal(de[m], do[m])
    return ok


def run_particles_synctest_pair(n_entities, check_distance, ticks, seed, max_prediction=None, ttl_lo=None,
                                ttl_hi=None, flags=0, tune=None, spawn_rate=0, spawn_ttl=300, startup_burst=False,
                                peek_check=False, z_fraction=0.0, checksums=None):
    """SyncTest on the GPU engine and on the oracle with identical inputs; returns comparison facts.
    checksums(world, transform, velocity): the checksum registration (default: the example's, see register_particles)."""
    maxp = max_prediction or max(8, check_distance + 1)
    ttl_lo = ttl_lo if ttl_lo is not None else 300 + check_distance
    ttl_hi = ttl_hi if ttl_hi is not None else ttl_lo
    cap = n_entities + spawn_rate * (ticks + 2)
    eng = Engine(max_entities=cap, max_depth=maxp, fps=60, flags=flags)
    orc = OracleWorld(fps=60)
    app_e, cols_e, mism_e = make_particles_app(eng, n_entities, seed, Session.SyncTest(
        SyncTestSession(2, check_distance, maxp, input_delay=2)), ttl_lo, ttl_hi, noop_inputs=True,
        spawn_rate=spawn_rate, spawn_ttl=spawn_ttl, startup_burst=startup_burst, z_fraction=z_fraction,
        checksums=checksums)
    app_o, cols_o, mism_o = make_particles_app(orc, n_entities, seed, Session.SyncTest(
        SyncTestSession(2, check_distance, maxp, input_delay=2)), ttl_lo, ttl_hi, noop_inputs=True,
        spawn_rate=spawn_rate, spawn_ttl=spawn_ttl, startup_burst=startup_burst, z_fraction=z_fraction,
        checksums=checksums)
    all_e, all_o = [], []
    launches0 = eng.launch_count()
    for _ in range(ticks):
        app_e.step()
        app_o.step()
        all_e += app_e.last_checksums
        all_o += app_o.last_checksums
    tick_launches = eng.launch_count() - launches0
    fused = eng.last_path_fused()
    kernel = eng.last_kernel()
    peek_equal = True
    if peek_check:  # every live snapshot, every column: same bytes as the oracle's snapshot of that frame
        n_rows = eng.row_count()
        for f in eng.snapshot_frames():
            for c in cols_e:
                pe, po = eng.peek(f, c, 0, n_rows), orc.peek(f, c, 0, n_rows)
                if (pe is None) != (po is None):
                    peek_equal = False
                    continue
                m = po[1].astype(bool)
                peek_equal = peek_equal and np.array_equal(pe[1].astype(bool), m) and np.array_equal(pe[0][m], po[0][m])
    res = {
        "checksums_equal": all_e == all_o and len(all_e) > 0,
        "n_checksums": len(all_e),
        "state_equal": eng.row_count() == orc.row_count() and compare_state(eng, orc, cols_e, eng.row_count()),
        "rows": (eng.row_count(), orc.row_count()),
        "peek_equal": peek_equal,
        "mismatch_events": (len(mism_e), len(mism_o)),
        "fused": fused,
        "kernel": kernel,
        "launches": tick_launches,
        "frames": (eng.rollback_frame_count(), orc.rollback_frame_count()),
        "active": (eng.active_count(), orc.active_count()),
        "ring": (eng.snapshot_frames(), orc.snapshot_frames()),
        "confirmed": (eng.confirmed_frame_count(), orc.confirmed_frame_count()),
        "checksums": all_e,
    }
    eng.close()
    orc.close()
    return res
