"""World batches replaying (bgr_batch_replay, EngineBatch.replay): worlds with different log lengths, intervals,
start frames and row counts in one call equal each world's own bgr_replay on a twin engine, and a call with one
invalid world executes nothing anywhere."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import EngineBatch

from test_gpu_batch import box_world, presence_world
from test_gpu_generic_spawn import spawn_world
from test_gpu_replay import live, log_for

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("generic_kernel")]
ROWS = [1, 127, 700, 2000, 129, 40]


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


def worlds(make, stream, n):
    members = [make(ROWS[i % len(ROWS)], 4, stream=stream, seed=i) for i in range(n)]
    twins = [make(ROWS[i % len(ROWS)], 4, seed=i) for i in range(n)]
    for i, (m, t) in enumerate(zip(members, twins)):
        m.set_rollback_frame_count(3 * i)
        t.set_rollback_frame_count(3 * i)
    return members, twins


@pytest.mark.parametrize("make", [presence_world, box_world, spawn_world])
def test_batched_replays_equal_each_worlds_own(generic_kernel, stream, make):
    members, twins = worlds(make, stream, 9)
    batch = EngineBatch(members)
    spawn = make is spawn_world
    calls = [(i, log_for(37 * i + 5, 1 + i % 3, seed=i, spawn_every=23 if spawn else 0), [0, 1, 10, 7, 500][i % 5])
             for i in range(9)]
    for rnd in range(2):
        res = batch.replay(calls)
        for (w, log, k), (status, cs) in zip(calls, res):
            assert status == capi.BGR_OK
            assert cs == twins[w].replay(log, k), f"world {w} round {rnd}"
            lk = members[w].last_kernel()
            assert lk.replay == (generic_kernel != "interpreter")
            assert lk.batched == batch.specialised()
    for w, (m, t) in enumerate(zip(members, twins)):
        assert live(m) == live(t), f"world {w}"


def test_one_invalid_world_executes_nothing(stream):
    members, _ = worlds(box_world, stream, 4)
    batch = EngineBatch(members)
    before = [live(m) for m in members]
    good = log_for(50, 2, seed=1)
    for bad in ([(0, good, 10), (1, np.zeros((5, 9), np.uint8), 1), (2, good, 10)],  # n_players > BGR_MAX_PLAYERS
                [(0, good, 10), (3, good, 1), (0, good, 1)],                          # listed twice
                [(0, good, 10), (7, good, 1)]):                                       # no such world
        with pytest.raises(BgrError) as ei:
            batch.replay(bad)
        assert str(ei.value).startswith("world ")
        assert [live(m) for m in members] == before


@pytest.mark.parametrize("make", [box_world, spawn_world])
def test_logs_split_over_several_launches_equal_one_launch(monkeypatch, generic_kernel, stream, make):
    """BGR_TUNE_REPLAY_POINTS=7: each launch takes at most 7 checksum points, so every world's log runs as segments
    that start mid-log (the segment's first checksum frame, its rows and tiles from the spawn prefix); the results
    equal one launch per call."""
    if generic_kernel == "interpreter":
        pytest.skip("BGR_TUNE_JIT=0: replays run in chunks, not in replay launches")
    one, _ = worlds(make, stream, 5)
    monkeypatch.setenv("BGR_TUNE_REPLAY_POINTS", "7")
    split, _ = worlds(make, stream, 5)
    b1, b2 = EngineBatch(one), EngineBatch(split)
    calls = [(i, log_for(60 + 41 * i, 2, seed=i, spawn_every=5 if make is spawn_world else 0), [1, 10, 3, 1, 7][i])
             for i in range(5)]
    launches = [e.launch_count() for e in split]
    assert b1.replay(calls) == b2.replay(calls)
    assert sum(e.launch_count() for e in split) - sum(launches) > 5
    for w, (a, b) in enumerate(zip(one, split)):
        assert b.last_kernel().replay
        assert live(a) == live(b), f"world {w}"
    # a single engine, interval 1: 300 points in launches of 7
    a, b = one[0], split[0]
    log = log_for(300, 2, seed=9)
    assert a.replay(log, 1) == b.replay(log, 1)
    assert live(a) == live(b)
