"""The replay entry point of the generated kernel (k_generic_jit_replay, csrc/generic_program_jit.cuh) compiles through
NVRTC for sm_90a with the preludes test_jit_sources_compile.py uses plus a spawning registration, in every instance the
engine builds, and ptxas reports no local-memory spills for it.  NVRTC needs no GPU."""
import ctypes as C
import os
import re

import pytest

from test_jit_sources_compile import CSRC, FILES, REGISTRATIONS, _nvrtc, _prelude

# the particles example with spawn_particles (update, despawn, spawn): Transform 0..9, Velocity 10..12, Ttl 13..14
SPAWNING = (15, [("BGR_SYS_PARTICLES_UPDATE", 0, 10, 0, 0), ("BGR_SYS_PARTICLES_DESPAWN", 13, 0, 0, 0),
                 ("BGR_SYS_PARTICLES_SPAWN", 0, 10, 0, 13)],
            [(10, 0, 12, 1, 0, 0), (0, 0, 12, 1, 1, 0)])
CASES = dict(REGISTRATIONS, spawning=SPAWNING)


def _compile_log(prelude):
    nvrtc = _nvrtc()
    contents = [open(os.path.join(CSRC, f), "rb").read() for f in FILES]
    prog = C.c_void_p()
    hs = (C.c_char_p * len(FILES))(*contents)
    ns = (C.c_char_p * len(FILES))(*[f.encode() for f in FILES])
    src = (prelude + '#include "generic_program_jit.cuh"\n').encode()
    assert nvrtc.nvrtcCreateProgram(C.byref(prog), src, b"bgr_generic_jit.cu", len(FILES), hs, ns) == 0
    opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"-fmad=false", b"-lineinfo", b"--ptxas-options=-v"]
    rc = nvrtc.nvrtcCompileProgram(prog, len(opts), (C.c_char_p * len(opts))(*opts))
    n = C.c_size_t()
    nvrtc.nvrtcGetProgramLogSize(prog, C.byref(n))
    log = C.create_string_buffer(n.value)
    nvrtc.nvrtcGetProgramLog(prog, log)
    nvrtc.nvrtcDestroyProgram(C.byref(prog))
    assert rc == 0, log.value.decode()
    return log.value.decode()


def _kernel_report(log, name):
    """ptxas' lines for one entry point: 'Compiling entry function', spill line, 'Used N registers' line."""
    lines = log.splitlines()
    start = next(i for i, l in enumerate(lines) if "Compiling entry function" in l and name + "'" in l)
    block = []
    for l in lines[start + 1:]:
        if "Compiling entry function" in l:
            break
        block.append(l)
    return "\n".join(block)


# the instances the engine builds: whole tiles (4 rows per thread) and 128-row items (2 rows per thread)
@pytest.mark.parametrize("rows,item_rows", [(4, 512), (2, 128)])
@pytest.mark.parametrize("name", list(CASES))
def test_replay_entry_point_compiles_without_spills(name, rows, item_rows):
    words, systems, hashes = CASES[name]
    log = _compile_log(_prelude(words, rows, systems, hashes, item_rows))
    rep = _kernel_report(log, "k_generic_jit_replay")
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert spills, rep
    assert spills.group(1) == "0" and spills.group(2) == "0", rep
    stack = re.search(r"(\d+) bytes stack frame", rep)
    assert stack and stack.group(1) == "0", rep
    assert re.search(r"Used \d+ registers", rep), rep
