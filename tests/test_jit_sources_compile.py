"""The run-time specialisation (csrc/jit.hpp) hands csrc/generic_program_jit.cuh + a generated prelude to NVRTC at bgr_build.
NVRTC needs no GPU, so the sources are compiled HERE for sm_90a with preludes of three registrations: a change to the
shared headers that breaks the NVRTC build (a host include, an un-annotated function) would otherwise only show up as a
silent fallback to the interpreter kernel on the GPU box."""
import ctypes as C
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bevy_ggrs_b200", "csrc")
FILES = ["generic_program_jit.cuh", "generic_program.cuh", "kernels.cuh", "seahash.cuh", "tma_copy.cuh", "rtc_prelude.cuh"]  # jit.hpp's list


def _nvrtc():
    for name in ("libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"):
        try:
            return C.CDLL(name)
        except OSError:
            continue
    pytest.skip("libnvrtc not installed")


def _system_ids():
    import re
    hdr = open(os.path.join(ROOT, "include", "bevy_ggrs_b200.h")).read()
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"(BGR_SYS_[A-Z0-9_]+)\s*=\s*(\d+)", hdr)}


def _prelude(words, rows, systems, hashes, item_rows=512):
    ids = _system_ids()
    lines = [f"#define {k} {v}" for k, v in ids.items()]
    lines += [f"#define BGR_TILE_ROWS 512", f"#define BGR_JIT_WORDS {words}", f"#define BGR_JIT_ROWS {rows}", f"#define BGR_JIT_ITEM_ROWS {item_rows}", "#define BGR_JIT_MINB 2",
              f"#define BGR_JIT_NSYS {len(systems)}", f"#define BGR_JIT_NHASH {len(hashes)}"]
    fmt = lambda t: "{" + ",".join(f"{int(v)}u" for v in t) + "}"
    lines.append("#define BGR_JIT_SYS_LIST " + ", ".join([fmt((ids[s[0]],) + tuple(s[1:])) for s in systems] + ["{0u,0u,0u,0u,0u}"]))
    lines.append("#define BGR_JIT_HASH_LIST " + ", ".join([fmt(h) for h in hashes] + ["{0u,0u,0u,0u,0u,0u}"]))
    return "\n".join(lines) + "\n"


def _compile(prelude):
    nvrtc = _nvrtc()
    contents = [open(os.path.join(CSRC, f), "rb").read() for f in FILES]
    prog = C.c_void_p()
    hs = (C.c_char_p * len(FILES))(*contents)
    ns = (C.c_char_p * len(FILES))(*[f.encode() for f in FILES])
    src = (prelude + '#include "generic_program_jit.cuh"\n').encode()
    assert nvrtc.nvrtcCreateProgram(C.byref(prog), src, b"bgr_generic_jit.cu", len(FILES), hs, ns) == 0
    opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"-fmad=false", b"-lineinfo"]
    rc = nvrtc.nvrtcCompileProgram(prog, len(opts), (C.c_char_p * len(opts))(*opts))
    n = C.c_size_t()
    nvrtc.nvrtcGetProgramLogSize(prog, C.byref(n))
    log = C.create_string_buffer(n.value)
    nvrtc.nvrtcGetProgramLog(prog, log)
    assert rc == 0, log.value.decode()
    nvrtc.nvrtcGetCUBINSize(prog, C.byref(n))
    cubin = C.create_string_buffer(n.value)
    nvrtc.nvrtcGetCUBIN(prog, cubin)
    nvrtc.nvrtcDestroyProgram(C.byref(prog))
    return cubin.raw


# {system, plane0, plane1, need, param} / {first_plane, off, len, finite, slot, absent}
REGISTRATIONS = {
    "presence": (5, [("BGR_SYS_U32_ADD", 0, 0, 2, 1), ("BGR_SYS_U32_SATSUB_DESPAWN", 1, 0, 4, 1)],
                 [(0, 0, 4, 0, 0, 2), (2, 0, 12, 0, 1, 0), (1, 0, 4, 0, 2, 4)]),
    "particles": (15, [("BGR_SYS_PARTICLES_UPDATE", 0, 10, 0, 0), ("BGR_SYS_PARTICLES_DESPAWN", 13, 0, 0, 0)],
                  [(10, 0, 12, 1, 0, 0), (0, 0, 12, 1, 1, 0)]),
    "box_game": (14, [("BGR_SYS_BOX_MOVE", 0, 10, 0, 0), ("BGR_SYS_DESPAWN_ON_INPUT", 13, 0, 2, 0x301), ("BGR_SYS_U32_STORE_CALL_COUNT", 13, 0, 2, 0)],
                 [(0, 0, 40, 0, 0, 0), (10, 4, 8, 0, 1, 0), (13, 0, 4, 0, 2, 2)]),
    "no_systems_no_checksums": (1, [], []),
}


# (4, 512) and (2, 128) are what jit_specialise builds by default; the others are reachable through BGR_TUNE_JIT_ROWS / _ITEM
@pytest.mark.parametrize("rows,item_rows", [(4, 512), (2, 128), (1, 512), (2, 512), (4, 128), (2, 256)])
@pytest.mark.parametrize("name", list(REGISTRATIONS))
def test_generated_kernel_compiles_for_sm_100a(name, rows, item_rows):
    # The name predates the move to Hopper and is kept so the test's id stays stable; it compiles for sm_90a (_compile).
    words, systems, hashes = REGISTRATIONS[name]
    cubin = _compile(_prelude(words, rows, systems, hashes, item_rows))
    assert cubin[:4] == b"\x7fELF" and b"k_generic_jit" in cubin


def test_engine_and_test_agree_on_the_source_list():
    """jit.hpp reads exactly these files next to the shared library."""
    src = open(os.path.join(CSRC, "jit.hpp")).read()
    for f in FILES:
        assert f'"{f}"' in src
        assert os.path.exists(os.path.join(CSRC, f))
