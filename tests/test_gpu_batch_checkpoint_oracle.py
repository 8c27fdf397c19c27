"""-m gpu: batched checkpoints held to the oracle, independently of the engine's own encoder and decoder: on the random
registrations of test_gpu_replay_oracle.py, the blobs of one bgr_batch_checkpoint_save over members of different row
counts equal what FlagsOracle.checkpoint_of builds with the numpy encoder from the oracle's snapshots, and worlds restored
by one bgr_batch_checkpoint_restore (each from another member's blob) stay equal to FlagsOracle.restore through the
vectors that follow."""
import numpy as np
import pytest

import checkpoint_codec as cc
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine, EngineBatch
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request
from bevy_ggrs_b200.stress import synth_particles
from interleave_driver import FlagsOracle
from test_gpu_replay_oracle import KINDS, assert_state, log_for, registration

pytestmark = pytest.mark.gpu
FRAMES = 24
MAX_ROWS = 1300
# more than 8 systems tick on the stepwise path, whose engines a batch does not take
BATCHABLE = [k for k in KINDS if k != "many_systems"]


@pytest.fixture
def stream():
    torch = pytest.importorskip("torch")
    s = torch.cuda.Stream()
    yield s.cuda_stream
    torch.cuda.synchronize()


def fleet(kind, seed, stream, n_worlds=3):
    rng = np.random.default_rng(0xBA7C + 131 * seed + KINDS.index(kind))
    cap = MAX_ROWS + 3 * FRAMES * 64 + 8   # every member can hold every other member's blob
    s, rate, players = registration(kind, rng)
    members, oracles, cols = [], [], None
    for i in range(n_worlds):
        n = int(rng.integers(100, MAX_ROWS))
        data = s.values(rng, n)
        if rate:
            tf, vel, ttl = synth_particles(n, seed + i, 2, 40)
            data[-3:] = [tf.view(np.uint8).reshape(n, 40), vel.view(np.uint8).reshape(n, 12), ttl.view(np.uint8).reshape(n, 8)]
        for w, out in ((Engine(max_entities=cap, max_depth=4, stream=stream), members), (FlagsOracle(max_entities=cap, max_depth=9), oracles)):
            cols = s.register(w)
            w.build()
            w.spawn(n)
            for c, d in zip(cols, data):
                w.write_component(c, 0, d)
            out.append(w)
    return members, oracles, cols, rate, players, rng


def run(eng, orc, log, f0):
    for j, row in enumerate(log):
        f = f0 + j
        info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))   # confirms the frame before: the oracle's ring never fills
        reqs = [Request(SAVE, f), Request(ADVANCE, 0, [int(v) for v in row])]
        assert eng.handle_requests(info, reqs) == orc.handle_requests(info, reqs), f"frame {f}"


@pytest.mark.parametrize("env", ["default", "jit0"])
@pytest.mark.parametrize("kind", BATCHABLE)
def test_batched_checkpoints_match_the_oracle(monkeypatch, stream, kind, env):
    if env == "jit0":
        monkeypatch.setenv("BGR_TUNE_JIT", "0")
    members, oracles, cols, rate, players, rng = fleet(kind, 1, stream)
    batch = EngineBatch(members)
    for e, o in zip(members, oracles):
        run(e, o, log_for(rng, FRAMES, players, bool(rate)), 0)
    f = FRAMES - 1
    blobs = batch.checkpoint([(w, f) for w in range(len(members))])
    for w, (blob, o) in enumerate(zip(blobs, oracles)):
        h = cc.unpack_header(blob)
        assert blob == o.checkpoint_of(f, h["layout"], h["rng"]), f"world {w}"
    # each world restored from the next one's blob, in one call
    order = [(w, blobs[(w + 1) % len(members)]) for w in range(len(members))]
    batch.restore(order)
    for (w, blob), o in zip(order, oracles):
        o.restore(blob)
    for e, o in zip(members, oracles):
        assert_state(e, o, cols)
        run(e, o, log_for(rng, FRAMES, players, bool(rate)), f)
        assert_state(e, o, cols)
