"""-m gpu: replay keyframes (bgr_replay_keyframes) held to the oracle, independently of the engine's checkpoint encoder:
on the random registrations of test_gpu_replay_oracle.py (sub-word and optional columns, despawn_on_input, the call
counter, spawn_particles, 30-word rows, nine systems), each keyframe blob must equal the one FlagsOracle.checkpoint_of
builds with the numpy encoder (tests/checkpoint_codec.py) from the oracle's own snapshot of that frame, taken by a Save
in the request stream the replay stands for.  The oracle does not hold ParticleRng, so the rng words come from the
engine's blob; tests/cpp/test_replay_keyframes.cpp holds them to the generator.  Then the live worlds must agree."""
import numpy as np
import pytest

import checkpoint_codec as cc
from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, SAVE, Request
from bevy_ggrs_b200.stress import synth_particles
from interleave_driver import FlagsOracle
from test_gpu_replay_oracle import KINDS, assert_state, log_for, registration

pytestmark = pytest.mark.gpu
FRAMES = 120
# (checksum interval, keyframe interval, start frame).  A keyframe at the first frame only from frame 0: the oracle
# restates a snapshot's Time<GgrsTime> as the frame's runtime, which a world moved by bgr_set_rollback_frame_count does
# not have (test_gpu_replay_keyframes.py holds that case to bgr_checkpoint_save on a twin)
CASES = [(10, 10, 0), (0, 1, 0), (7, 25, 5), (10, 60, 0)]


def worlds(kind, seed, n):
    rng = np.random.default_rng(0xC0DE + 131 * seed + KINDS.index(kind))
    s, rate, players = registration(kind, rng)
    data = s.values(rng, n)
    if rate:
        tf, vel, ttl = synth_particles(n, seed, 2, 40)
        data[-3:] = [tf.view(np.uint8).reshape(n, 40), vel.view(np.uint8).reshape(n, 12), ttl.view(np.uint8).reshape(n, 8)]
    removes = [(c, int(r)) for c, o in enumerate(s.optional) if o for r in rng.choice(n, min(n, 9), replace=False)]
    out = []
    cap = n + rate * FRAMES + 8
    for w in (Engine(max_entities=cap, max_depth=4), FlagsOracle(max_entities=cap, max_depth=9)):
        cols = s.register(w)
        w.build()
        w.spawn(n)
        for c, d in zip(cols, data):
            w.write_component(c, 0, d)
        for c, r in removes:
            w.remove_component(cols[c], r)
        out.append(w)
    return out[0], out[1], cols, rate, players, rng


@pytest.mark.parametrize("env", ["default", "jit0"])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("kind", KINDS)
def test_keyframes_match_the_oracle(monkeypatch, kind, case, env):
    if env == "jit0":
        monkeypatch.setenv("BGR_TUNE_JIT", "0")
    k, kk, f0 = CASES[case]
    eng, orc, cols, rate, players, rng = worlds(kind, case, int(np.random.default_rng(case).integers(200, 1300)))
    for w in (eng, orc):
        w.set_rollback_frame_count(f0)
    log = log_for(rng, FRAMES, players, bool(rate))
    _, kfs = eng.replay_keyframes(log, k, kk)
    assert [f for f, _ in kfs] == [f0 + j for j in range(FRAMES) if (f0 + j) % kk == 0]
    for j in range(FRAMES):
        f = f0 + j
        info = (capi.BGR_SESSION_P2P, 7, 0, max(0, f - 1))  # confirms the frame before: the oracle's ring never fills
        if f % kk == 0:
            orc.handle_requests(info, [Request(SAVE, f)])
            blob = dict(kfs)[f]
            h = cc.unpack_header(blob)
            assert blob == orc.checkpoint_of(f, h["layout"], h["rng"]), f"keyframe {f}"
        orc.handle_requests(info, [Request(ADVANCE, 0, [int(v) for v in log[j]])])
    assert_state(eng, orc, cols)
