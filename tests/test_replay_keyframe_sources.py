"""The keyframe entry point of the generated kernel (k_generic_jit_replay_kf, csrc/generic_program_jit.cuh) compiles
through NVRTC for sm_90a for every registration of test_replay_sources.py, in both instances the engine builds, with no
local-memory spills and no stack.  k_generic_jit_replay is the same templated body without the keyframe stores: in the
same compile its registers, barriers and shared memory stay what they were before the keyframe entry point existed
(recorded below from ptxas of CUDA 12.9), so plain replays are not slowed by keyframes.  NVRTC needs no GPU."""
import re

import pytest

from test_jit_sources_compile import _prelude
from test_replay_sources import CASES, _compile_log, _kernel_report

# k_generic_jit_replay before keyframes: (registers, smem bytes) per registration and (rows, item_rows)
PLAIN = {
    ("presence", 4, 512): (118, 5120), ("presence", 2, 128): (77, 5120),
    ("particles", 4, 512): (158, 10240), ("particles", 2, 128): (103, 7680),
    ("box_game", 4, 512): (206, 10240), ("box_game", 2, 128): (122, 7680),
    ("no_systems_no_checksums", 4, 512): (56, 5120), ("no_systems_no_checksums", 2, 128): (56, 5120),
    ("spawning", 4, 512): (158, 10240), ("spawning", 2, 128): (100, 7680),
}


def _figures(rep):
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    stack = re.search(r"(\d+) bytes stack frame", rep)
    used = re.search(r"Used (\d+) registers, used (\d+) barriers, (\d+) bytes smem", rep)
    assert spills and stack and used, rep
    return int(spills.group(1)), int(spills.group(2)), int(stack.group(1)), int(used.group(1)), int(used.group(2)), int(used.group(3))


@pytest.mark.parametrize("rows,item_rows", [(4, 512), (2, 128)])
@pytest.mark.parametrize("name", list(CASES))
def test_keyframe_entry_point_compiles_and_the_plain_one_is_unchanged(name, rows, item_rows):
    words, systems, hashes = CASES[name]
    log = _compile_log(_prelude(words, rows, systems, hashes, item_rows))
    kf = _figures(_kernel_report(log, "k_generic_jit_replay_kf"))
    assert kf[:3] == (0, 0, 0), kf
    plain = _figures(_kernel_report(log, "k_generic_jit_replay"))
    assert plain[:3] == (0, 0, 0), plain
    assert (plain[3], plain[5]) == PLAIN[(name, rows, item_rows)]
    assert plain[4] == kf[4] == 1  # one named barrier: the keyframe stores add none
