"""The trace entry point of the generated kernel (k_generic_jit_replay_trace, csrc/generic_program_jit.cuh) compiles
through NVRTC for sm_90a for every registration of test_replay_sources.py, in both instances the engine builds, with no
local-memory spills and no stack: the run-time field map selects record words, never register rows.  Its figures are
pinned, and the four entry points that existed before it keep theirs (recorded below from ptxas of CUDA 12.9), so the
tick, the batched tick, plain replays and keyframe replays are not slowed by traces.  NVRTC needs no GPU."""
import pytest

from test_jit_sources_compile import _prelude
from test_replay_keyframe_sources import _figures
from test_replay_sources import CASES, _compile_log, _kernel_report

# (registers, smem bytes) per registration and (rows, item_rows)
TRACE = {
    ("presence", 4, 512): (116, 5120), ("presence", 2, 128): (88, 5120),
    ("particles", 4, 512): (168, 10240), ("particles", 2, 128): (106, 7680),
    ("box_game", 4, 512): (207, 10240), ("box_game", 2, 128): (142, 7680),
    ("no_systems_no_checksums", 4, 512): (64, 5120), ("no_systems_no_checksums", 2, 128): (64, 5120),
    ("spawning", 4, 512): (168, 10240), ("spawning", 2, 128): (112, 7680),
}
# k_generic_jit, k_generic_jit_batch, k_generic_jit_replay, k_generic_jit_replay_kf before traces
BEFORE = {
    ("presence", 4, 512): ((90, 2568), (104, 2564), (118, 5120), (120, 5120)),
    ("presence", 2, 128): ((64, 2568), (76, 2564), (77, 5120), (90, 5120)),
    ("particles", 4, 512): ((114, 2568), (154, 2564), (158, 10240), (166, 10240)),
    ("particles", 2, 128): ((78, 2568), (88, 2564), (103, 7680), (109, 7680)),
    ("box_game", 4, 512): ((142, 2568), (172, 2564), (206, 10240), (214, 10240)),
    ("box_game", 2, 128): ((93, 2568), (108, 2564), (122, 7680), (121, 7680)),
    ("no_systems_no_checksums", 4, 512): ((40, 2568), (48, 2564), (56, 5120), (64, 5120)),
    ("no_systems_no_checksums", 2, 128): ((30, 2568), (40, 2564), (56, 5120), (64, 5120)),
    ("spawning", 4, 512): ((114, 2568), (154, 2564), (158, 10240), (168, 10240)),
    ("spawning", 2, 128): ((80, 2568), (96, 2564), (100, 7680), (119, 7680)),
}
EXISTING = ("k_generic_jit", "k_generic_jit_batch", "k_generic_jit_replay", "k_generic_jit_replay_kf")


@pytest.mark.parametrize("rows,item_rows", [(4, 512), (2, 128)])
@pytest.mark.parametrize("name", list(CASES))
def test_trace_entry_point_compiles_and_the_others_are_unchanged(name, rows, item_rows):
    words, systems, hashes = CASES[name]
    log = _compile_log(_prelude(words, rows, systems, hashes, item_rows))
    tr = _figures(_kernel_report(log, "k_generic_jit_replay_trace"))
    assert tr[:3] == (0, 0, 0), tr
    assert (tr[3], tr[5]) == TRACE[(name, rows, item_rows)]
    assert tr[4] == 1  # one named barrier: the trace stores add none
    for kernel, want in zip(EXISTING, BEFORE[(name, rows, item_rows)]):
        got = _figures(_kernel_report(log, kernel))
        assert got[:3] == (0, 0, 0), (kernel, got)
        assert (got[3], got[5]) == want, kernel
