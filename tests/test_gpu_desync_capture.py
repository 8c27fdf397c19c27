"""Desync capture on the H100, generic one-launch program (interpreter and NVRTC kernels, generic_kernel fixture) and
the stepwise path: capture changes nothing observable, and the GPU report equals the oracle's restatement."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.desync import NO_INDEX
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import SyncTestSession
from desync_util import LARGE_ROWS, N_ROWS, counter_app, despawn_app, health_rows, run_to_first_mismatch
from oracle_desync import CaptureOracleWorld

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]
CAP = capi.BGR_CFG_DESYNC_CAPTURE
PATHS = [0, capi.BGR_CFG_FORCE_STEPWISE]


def _observe(eng, n_cols, rows):
    """Everything a caller can read: every ring frame's peek of every column, and the launch count."""
    peeks = {}
    for f in eng.snapshot_frames():
        for c in range(n_cols):
            data, alive = eng.peek(f, c, 0, rows)
            peeks[(f, c)] = (data[alive.astype(bool)].tobytes(), alive.tobytes())
    return eng.snapshot_frames(), peeks, eng.launch_count()


def _presence_world(flags, n=1300, ticks=24):
    eng = Engine(max_entities=n + 8, max_depth=8, flags=flags)
    opt = capi.BGR_STRATEGY_OPTIONAL
    score = eng.rollback_component("Score", 4, capi.BGR_STRATEGY_COPY | opt)
    health = eng.rollback_component("Health", 4, capi.BGR_STRATEGY_CLONE | opt)
    tag = eng.rollback_component("Tag", 12)
    for c, ln in ((score, 4), (tag, 12), (health, 4)):
        eng.checksum_component(c, 0, ln)
    eng.add_system(capi.BGR_SYS_U32_ADD, [score], [0, 1])
    eng.add_system(capi.BGR_SYS_U32_SATSUB_DESPAWN, [health], [0, 1])
    eng.build()
    eng.spawn(n)
    rng = np.random.default_rng(5)
    eng.write_component(score, 0, rng.integers(0, 1000, n, dtype=np.uint32))
    eng.write_component(health, 0, rng.integers(3, 40, n, dtype=np.uint32))
    eng.write_component(tag, 0, rng.integers(0, 2**32, (n, 3), dtype=np.uint32))
    sess = SyncTestSession(1, 3, 8)
    checksums = []
    for t in range(ticks):
        if t % 5 == 2:  # presence changes between ticks: the re-simulations Load around them
            eng.remove_component(score, (37 * t) % n)
            eng.insert_component(health, (53 * t) % n, np.uint32(9))
        sess.add_local_input(0, 0)
        out = eng.handle_requests(sess.info(), sess.advance_frame())
        for f, _ in out:  # edits between ticks are not rolled back: keep the SyncTest request shape, skip its check
            sess.save_cell(f, 0)
        checksums.append(out)
    return checksums, _observe(eng, 3, n)


@pytest.mark.parametrize("path", PATHS)
def test_capture_changes_nothing_on_the_presence_world(path):
    assert _presence_world(path) == _presence_world(path | CAP)


@pytest.mark.parametrize("path", PATHS)
def test_capture_changes_nothing_on_box_game(path):
    from test_gpu_box_game import _app

    def run(flags):
        app, tf, vel, bad = _app(Engine(max_entities=8, max_depth=9, flags=flags), native_resource=False)
        checksums = []
        for _ in range(50):
            app.update()
            checksums.append(list(app.last_checksums))
        assert not bad
        return checksums, _observe(app.world, 2, 2)
    assert run(path) == run(path | CAP)


def _same_report(a, b):
    assert a is not None and b is not None
    assert a.summary_tuple() == b.summary_tuple()
    assert a.columns == b.columns
    assert a.records.dtype == b.records.dtype and np.array_equal(a.records, b.records)


def _check_against_peeks(eng, rep, n_cols):
    """The records equal a numpy comparison of bgr_peek_first and bgr_peek."""
    rows = max(rep.rows_first, rep.rows_latest)
    changed = np.zeros(rows, bool)
    for c in range(n_cols):
        df, af = eng.peek_first(rep.frame, c, 0, rows)
        dl, al = eng.peek(rep.frame, c, 0, rows)
        eb = eng.elem_bytes[c]
        cw = (eb + 3) // 4
        wf, wl = np.zeros((rows, cw * 4), np.uint8), np.zeros((rows, cw * 4), np.uint8)
        wf[:, :eb], wl[:, :eb] = df, dl
        wf, wl = wf.view("<u4"), wl.view("<u4")
        both = (af & al).astype(bool)
        r, w = np.nonzero((wf != wl) & both[:, None])
        got = rep.records[(rep.records["column"] == c) & (rep.records["word"] != NO_INDEX)]
        assert list(zip(got["row"], got["word"], got["first"], got["latest"])) == \
            list(zip(r, w, wf[r, w], wl[r, w])), c
        changed |= af != al
    structural = rep.records[rep.records["word"] == NO_INDEX]
    assert sorted(set(structural["row"])) == list(np.nonzero(changed)[0])


def _caps(records):
    """records_cap values to try: every cap for a short list; otherwise caps inside a warp, and on either side of the
    warp (32, 64 rows) and tile (512, 1024 rows) boundaries, which in the mixed world also split a row's two records,
    and caps at and beyond the total."""
    n = len(records)
    if n <= 8:
        return list(range(n + 2))
    marks = {0, 1, 5, n - 1, n, n + 3}
    for b in (32, 64, 512, 1024):
        k = int((records["row"] < b).sum())
        marks |= {k - 1, k, k + 1}
    return sorted(m for m in marks if m >= 0)


WORLDS = [("counter", N_ROWS), ("despawn", N_ROWS), ("counter", LARGE_ROWS), ("despawn", LARGE_ROWS),
          ("mixed", LARGE_ROWS)]


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("world,n", WORLDS)
def test_gpu_report_equals_the_oracle_report(path, world, n):
    """Worlds of 6 rows (one warp) and of 1400 rows (records in many warps of three tiles: pass 2 gets several tiles
    with non-zero bases, and rows carry 0, 1 or 2 records)."""
    def make(backend):
        if world == "despawn":
            return despawn_app(backend, n_rows=n)[0]
        return counter_app(backend, n_rows=n, mixed=world == "mixed")[0]
    app_g = make(Engine(max_entities=n + 64, max_depth=8, flags=path | CAP))
    app_o = make(CaptureOracleWorld())
    ev_g, rep_g, _ = run_to_first_mismatch(app_g, max_records=4 * n)
    ev_o, rep_o, _ = run_to_first_mismatch(app_o, max_records=4 * n)
    assert (ev_g.current_frame, ev_g.mismatched_frames) == (ev_o.current_frame, ev_o.mismatched_frames)
    eng = app_g.world
    assert eng.desync_frames() == app_o.world.desync_frames() and eng.desync_frames()
    total = 0
    for f in ev_g.mismatched_frames:
        _same_report(rep_g[f], rep_o[f])
        _check_against_peeks(eng, rep_g[f], len(eng.elem_bytes))
        assert rep_g[f].rows_differing > 0
        _same_report(eng.desync_diff(f, 4 * n), rep_g[f])      # two runs, identical output
        recs = rep_g[f].records
        total += len(recs)
        if n == LARGE_ROWS:
            assert len(set(recs["row"] // 512)) == 3 and len(set(recs["row"] // 32)) > 16
        for cap in _caps(recs):                                 # a small cap: exactly the first `cap` records
            small = eng.desync_diff(f, cap)
            assert np.array_equal(small.records, recs[:cap]), cap
            assert small.summary_tuple() == rep_g[f].summary_tuple() and small.columns == rep_g[f].columns
    assert total > 0
    if world == "despawn":
        ex = rep_g[2].records[rep_g[2].records["column"] == NO_INDEX]
        assert list(ex["row"]) == health_rows(n) and set(ex["first"]) == {0} and set(ex["latest"]) == {1}
    if world == "mixed":
        per_row = np.bincount(rep_g[2].records["row"], minlength=n)
        assert set(per_row) == {0, 1, 2} and rep_g[2].columns[1].presence > 0


@pytest.mark.parametrize("path", PATHS)
def test_entry_points_refuse_an_engine_without_capture(path):
    eng = Engine(max_entities=16, max_depth=8, flags=path)
    eng.rollback_component("X", 4)
    eng.build()
    for call in (lambda: eng.desync_frames(), lambda: eng.desync_diff(0), lambda: eng.peek_first(0, 0, 0, 1)):
        with pytest.raises(BgrError) as ei:
            call()
        assert ei.value.status == capi.BGR_ERR_STATE


@pytest.mark.parametrize("path", PATHS)
def test_unknown_frame_is_not_found_and_reset_session_releases_first_images(path):
    app, score, counter = counter_app(Engine(max_entities=64, max_depth=8, flags=path | CAP))
    for _ in range(5):
        app.update()
    eng = app.world
    frames = eng.desync_frames()
    assert frames and eng.desync_diff(10_000) is None and eng.peek_first(10_000, 0, 0, 1) is None
    assert eng.peek_first(frames[0], counter, 0, N_ROWS) is not None
    eng.reset_session()
    assert eng.desync_frames() == [] and eng.desync_diff(frames[0]) is None
