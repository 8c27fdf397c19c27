"""-m gpu: replay traces (bgr_replay_trace) held to the oracle: on the random registrations of test_gpu_replay_oracle.py
(sub-word and optional columns, despawn_on_input, the call counter, spawn_particles, 30-word rows, nine systems), with a
random field list over the whole-word columns and a random row range, each sample's records must equal the ones read
back from the oracle at that frame, the oracle driven through the request stream the replay stands for.  The default
kernel selection and BGR_TUNE_JIT=0.  Then the checksums and the live worlds must agree."""
import numpy as np
import pytest

from test_gpu_replay_oracle import KINDS, assert_state, log_for, oracle_stream, worlds
from test_gpu_replay_trace import expected

pytestmark = pytest.mark.gpu
FRAMES = 150
# (checksum interval, trace interval, start frame)
CASES = [(10, 1, 0), (0, 7, 5), (10, 60, 3)]


def random_trace(rng, s, cols, cap):
    """A field list over the whole-word columns (at most three fields, a column may repeat) and a row range."""
    whole = [c for c, sz in enumerate(s.sizes) if sz % 4 == 0]
    fields = []
    for _ in range(int(rng.integers(0, 4)) if whole else 0):
        c = int(rng.choice(whole))
        off = 4 * int(rng.integers(0, s.sizes[c] // 4))
        ln = 4 * int(rng.integers(1, (s.sizes[c] - off) // 4 + 1))
        fields.append((cols[c], off, ln))
    first = int(rng.integers(0, cap))
    return fields, first, int(rng.integers(1, cap - first + 1))


@pytest.mark.parametrize("env", ["default", "jit0"])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("kind", KINDS)
def test_trace_matches_the_oracle(monkeypatch, kind, case, env):
    if env == "jit0":
        monkeypatch.setenv("BGR_TUNE_JIT", "0")
    k, tt, f0 = CASES[case]
    eng, orc, cols, s, rate, players, rng = worlds(kind, case, int(np.random.default_rng(case).integers(200, 1500)))
    for w in (eng, orc):
        w.set_rollback_frame_count(f0)
    log = log_for(rng, FRAMES, players, bool(rate))
    cap = eng.capacity()[0]
    fields, first, n_rows = random_trace(rng, s, cols, cap)
    cs, samples, recs = eng.replay_trace(log, k, tt, fields, first, n_rows)
    want_cs, at, q = [], 0, 0
    for j in range(FRAMES):
        if (f0 + j) % tt == 0:
            want_cs += oracle_stream(orc, f0 + at, log[at:j], k)
            at = j
            assert samples[q] == (f0 + j, orc.row_count())
            assert np.array_equal(recs[q], expected(orc, fields, first, n_rows)), f"sample {f0 + j}"
            q += 1
    want_cs += oracle_stream(orc, f0 + at, log[at:], k)
    assert q == len(samples)
    assert cs == want_cs
    assert_state(eng, orc, cols)
