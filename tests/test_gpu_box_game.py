"""BASELINE config C1 on the GPU: box_game SyncTest, 2 players, check_distance 8 (max_prediction 9),
input_delay 2 (examples/box_game/box_game_synctest.rs).  Transform / Velocity and the checksum (FrameCount resource
part ^ entity part, box_game_synctest.rs:55) must be bit-identical: move_cube_system's friction factor
`0.0018.powf(dt)` is the C library's powf on both sides (the host evaluates it once per Advance)."""
import struct

import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.plugin import (App, GgrsPlugin, GgrsSchedule, LocalInputs, ReadInputs, ResourceSystem, Session,
                                   Startup, SyncTestMismatch, System)
from bevy_ggrs_b200.session import SyncTestSession
from oracle_backend import ORC_SYS_RESOURCE_U32_ADD, OracleWorld

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]
SEQ = [0b0001, 0b1000, 0b0101, 0, 0b0010, 0b1010, 0b0100, 0b1001]


def _setup(a, tf):
    first = a.world.spawn(2)
    t = np.zeros((2, 10), np.float32)
    r = 5.0 / 4.0
    for h in range(2):
        rot = np.float32(h) / np.float32(2) * np.float32(2.0) * np.float32(np.pi)
        t[h, 0] = r * np.cos(rot); t[h, 1] = 0.1; t[h, 2] = r * np.sin(rot)
        t[h, 6] = 1.0; t[h, 7:10] = 1.0
    a.world.write_component(tf, first, t)


def _app(backend, native_resource):
    app = App(backend)
    app.insert_resource(Session.SyncTest(SyncTestSession(2, 8, 9, input_delay=2)))
    app.add_plugins(GgrsPlugin())
    app.add_systems(ReadInputs, lambda a: a.insert_resource(
        LocalInputs({h: SEQ[(a.ticks + 3 * h) % len(SEQ)] for h in a.local_players.handles})))
    vel = app.rollback_component_with_copy("Velocity", 12)
    tf = app.rollback_component_with_clone("Transform", 40)
    app.add_systems(GgrsSchedule, System(capi.BGR_SYS_BOX_MOVE, [tf, vel]))
    if native_resource:  # the oracle restates resource rollback + checksum itself
        fc = backend.rollback_resource("FrameCount", bytes(4), checksum=True)
        app.add_systems(GgrsSchedule, System(ORC_SYS_RESOURCE_U32_ADD, [], [fc]))
    else:                # product: resources stay host-side in the shim
        app.rollback_resource_with_copy("FrameCount", bytes(4)).checksum_resource_with_hash("FrameCount")

        def increase_frame_system(res):  # box_game.rs:146-148
            res["FrameCount"][:] = struct.pack("<I", (struct.unpack("<I", res["FrameCount"])[0] + 1) & 0xFFFFFFFF)
        app.add_systems(GgrsSchedule, ResourceSystem(increase_frame_system))
    app.add_systems(Startup, lambda a: _setup(a, tf))
    bad = []
    app.add_observer(SyncTestMismatch, lambda ev: bad.append(ev))
    return app, tf, vel, bad


@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
def test_box_game_synctest_c1_gpu_vs_oracle(flags):
    eng, orc = Engine(max_entities=4, max_depth=9, flags=flags), OracleWorld()
    app_e, tf, vel, bad_e = _app(eng, native_resource=False)
    app_o, _, _, bad_o = _app(orc, native_resource=True)
    cs_e, cs_o = [], []
    launches_per_tick = set()
    for i in range(120):
        l0 = eng.launch_count()
        app_e.update(); app_o.update()
        if i >= 10:                                    # after Startup (spawn + upload kernels) and the ring fill
            launches_per_tick.add(eng.launch_count() - l0)
        cs_e += app_e.last_checksums; cs_o += app_o.last_checksums
    assert not bad_e and not bad_o                     # SyncTest self-consistent on both
    assert cs_e == cs_o and len(cs_e) > 500            # FrameCount part ^ entity part: bit-identical
    assert app_e.rollback_frame_count() == app_o.rollback_frame_count() == 119
    assert struct.unpack("<I", app_e.resources["FrameCount"])[0] == 119
    for col in (tf, vel):
        a = eng.read_component(col, 0, 2).view(np.float32)
        b = orc.read_component(col, 0, 2).view(np.float32)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (a, b)
    t = eng.read_component(tf, 0, 2).view(np.float32)
    assert np.all(np.abs(t[:, [0, 2]]) <= 2.4 + 1e-6)   # constrained to the plane
    v = eng.read_component(vel, 0, 2).view(np.float32)
    assert np.all(np.linalg.norm(v, axis=1) <= 3.0 + 1e-5) and np.any(v != 0)
    # default: the generic one-launch program (move_cube_system + snapshots + checksums of a whole tick in ONE launch)
    assert eng.last_path_fused() == (flags == 0)
    assert (launches_per_tick <= {0, 1}) == (flags == 0)


def test_box_game_eight_players_every_handle_reaches_move_cube_system():
    """`inputs[p.handle]` for EVERY handle (box_game.rs:171): BGR_MAX_PLAYERS = 8 inputs cross the ABI and all of them
    steer their cube (round 1 silently gave handles 4..7 input 0)."""
    from bevy_ggrs_b200.session import ADVANCE, SAVE, Request
    eng, orc = Engine(max_entities=8, max_depth=16), OracleWorld()   # no session: nothing prunes the 12 snapshots
    cols = []
    for w in (eng, orc):
        vel = w.rollback_component("Velocity", 12)
        tf = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
        w.add_system(capi.BGR_SYS_BOX_MOVE, [tf, vel])
        w.build()
        first = w.spawn(8)
        t = np.zeros((8, 10), np.float32)
        t[:, 0] = np.linspace(-1.5, 1.5, 8); t[:, 1] = 0.1; t[:, 6] = 1.0; t[:, 7:10] = 1.0
        w.write_component(tf, first, t)
        cols = [tf, vel]
    nosess = (capi.BGR_SESSION_NONE, 0, 0, 0)
    inputs = [0b0001, 0b0010, 0b0100, 0b1000, 0b0101, 0b1010, 0b1001, 0b0110]
    reqs = []
    for f in range(12):
        reqs += [Request(SAVE, f), Request(ADVANCE, f, inputs)]
    assert eng.handle_requests(nosess, reqs) == orc.handle_requests(nosess, reqs)
    v = eng.read_component(cols[1], 0, 8).view(np.float32)
    vo = orc.read_component(cols[1], 0, 8).view(np.float32)
    assert np.array_equal(v.view(np.uint32), vo.view(np.uint32))
    assert np.array_equal(eng.read_component(cols[0], 0, 8), orc.read_component(cols[0], 0, 8))
    assert np.all(np.linalg.norm(v, axis=1) > 0.5)               # all eight cubes were accelerated by their own input
    assert v[4, 0] < 0 and v[4, 2] < 0 and v[7, 0] < 0 and v[7, 2] > 0   # handles 4 and 7: LEFT|UP, LEFT|DOWN
    eng.close(); orc.close()
