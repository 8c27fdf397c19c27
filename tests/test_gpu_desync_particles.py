"""Desync capture on the particles stress world (the one-launch bundle kernel, and the generic program with
BGR_TUNE_BUNDLE=0), one-launch and stepwise: every checksum, every ring snapshot and the launch count are the same with
and without BGR_CFG_DESYNC_CAPTURE."""
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.plugin import Session
from bevy_ggrs_b200.session import SyncTestSession
from parity_util import make_particles_app

pytestmark = pytest.mark.gpu


def _run(n, flags, ticks=30):
    eng = Engine(max_entities=n + 4096, max_depth=9, flags=flags)
    app, cols, mism = make_particles_app(eng, n, seed=11, session=Session.SyncTest(SyncTestSession(2, 6, 8)),
                                         ttl_lo=5, ttl_hi=40, spawn_rate=64)
    checksums = []
    for _ in range(ticks):
        app.step()
        checksums.append(list(app.last_checksums))
    assert not mism
    rows = eng.row_count()
    peeks = {}
    for f in eng.snapshot_frames():
        for c in cols:
            data, alive = eng.peek(f, c, 0, rows)
            peeks[(f, c)] = (data[alive.astype(bool)].tobytes(), alive.tobytes())
    fused = eng.last_path_fused()
    return checksums, eng.snapshot_frames(), peeks, eng.launch_count(), fused, eng.desync_frames() if flags & capi.BGR_CFG_DESYNC_CAPTURE else None


@pytest.mark.parametrize("bundle", ["1", "0"])
@pytest.mark.parametrize("path", [0, capi.BGR_CFG_FORCE_STEPWISE])
@pytest.mark.parametrize("n", [3000, 120_000])
def test_capture_changes_nothing_on_the_particles_world(monkeypatch, bundle, path, n):
    monkeypatch.setenv("BGR_TUNE_BUNDLE", bundle)
    plain = _run(n, path)
    cap = _run(n, path | capi.BGR_CFG_DESYNC_CAPTURE)
    assert plain[:5] == cap[:5]
    assert cap[5], "SyncTest re-saves must leave frames with a retained first image"


def test_deterministic_world_reports_no_difference():
    n = 3000
    eng = Engine(max_entities=n + 4096, max_depth=9, flags=capi.BGR_CFG_DESYNC_CAPTURE)
    app, cols, mism = make_particles_app(eng, n, seed=3, session=Session.SyncTest(SyncTestSession(2, 6, 8)),
                                         ttl_lo=5, ttl_hi=40)
    for _ in range(12):
        app.step()
    frames = eng.desync_frames()
    assert frames
    for f in frames:
        rep = eng.desync_diff(f)
        assert rep.empty and len(rep.records) == 0 and rep.rows_first == rep.rows_latest
