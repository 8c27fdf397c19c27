"""World batches on the CPU: the generated kernel's module exports both entry points (k_generic_jit for one engine,
k_generic_jit_batch for a batch) for the registrations a batch is made of, neither spills, and the C ABI refuses an
empty batch without a GPU."""
import ctypes as C

import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.engine import LastKernel
from test_jit_sources_compile import FILES, CSRC, _nvrtc, _prelude

import os

# {system, plane0, plane1, need, param} / {first_plane, off, len, finite, slot, absent}
REGISTRATIONS = {
    # Score (optional U32_ADD), Health (optional SATSUB_DESPAWN), Tag 12 B: every column checksummed
    "presence": (5, [("BGR_SYS_U32_ADD", 0, 0, 2, 1), ("BGR_SYS_U32_SATSUB_DESPAWN", 1, 0, 4, 1)],
                 [(0, 0, 4, 0, 0, 2), (2, 0, 12, 0, 1, 0), (1, 0, 4, 0, 2, 4)]),
    # box_game: Velocity 12 B, Transform 40 B, move_cube_system, the translation asserting finite
    "box_game": (13, [("BGR_SYS_BOX_MOVE", 3, 0, 0, 0)], [(3, 0, 12, 1, 0, 0), (0, 0, 12, 0, 1, 0)]),
    # the stress schema (Transform, Velocity, Ttl: 15 words) on the generic program
    "stress_15_words": (15, [("BGR_SYS_PARTICLES_UPDATE", 0, 10, 0, 0), ("BGR_SYS_PARTICLES_DESPAWN", 13, 0, 0, 0)],
                        [(10, 0, 12, 1, 0, 0), (0, 0, 12, 1, 1, 0)]),
}


def _compile_verbose(prelude):
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
    assert rc == 0, log.value.decode()
    nvrtc.nvrtcGetCUBINSize(prog, C.byref(n))
    cubin = C.create_string_buffer(n.value)
    nvrtc.nvrtcGetCUBIN(prog, cubin)
    nvrtc.nvrtcDestroyProgram(C.byref(prog))
    return cubin.raw, log.value.decode()


# (2, 128): the batch's default instance; (4, 512): what BGR_TUNE_JIT_ITEM=512 selects
@pytest.mark.parametrize("rows,item_rows", [(2, 128), (4, 512)])
@pytest.mark.parametrize("name", list(REGISTRATIONS))
def test_module_exports_both_entry_points_without_spills(name, rows, item_rows):
    words, systems, hashes = REGISTRATIONS[name]
    cubin, log = _compile_verbose(_prelude(words, rows, systems, hashes, item_rows))
    assert cubin[:4] == b"\x7fELF"
    assert b"k_generic_jit\x00" in cubin and b"k_generic_jit_batch\x00" in cubin
    for kernel in ("k_generic_jit", "k_generic_jit_batch"):
        at = log.index(f"Compiling entry function '{kernel}'")
        block = log[at:log.index("Compiling entry function", at + 1) if "Compiling entry function" in log[at + 1:] else len(log)]
        assert "0 bytes spill stores, 0 bytes spill loads" in block, block


def test_empty_batch_is_refused():
    lib = capi.load_library()
    out = C.c_void_p()
    assert lib.bgr_batch_create(None, 0, C.byref(out)) == capi.BGR_ERR_INVALID_ARGUMENT
    assert not out.value
    assert lib.bgr_batch_handle_requests(None, None, 0, None, None, None, None, 0, None, None) == capi.BGR_ERR_INVALID_ARGUMENT
    lib.bgr_batch_destroy(None)


def test_batched_flag_decodes():
    raw = capi.BGR_KERNEL_GENERIC_NVRTC | (128 << 16) | capi.BGR_KERNEL_BATCHED
    lk = LastKernel.decode(raw)
    assert lk.batched and lk.kind == "generic_nvrtc" and lk.item_rows == 128
    assert not LastKernel.decode(capi.BGR_KERNEL_GENERIC_NVRTC | (128 << 16)).batched
    hdr = open(os.path.join(os.path.dirname(CSRC), "..", "include", "bevy_ggrs_b200.h")).read()
    rs = open(os.path.join(os.path.dirname(CSRC), "..", "rust_shim", "bevy_ggrs_b200_sys", "src", "lib.rs")).read()
    assert "#define BGR_KERNEL_BATCHED (1u << 28)" in hdr and "pub const BGR_KERNEL_BATCHED: u32 = 1 << 28;" in rs
    assert capi.BGR_KERNEL_BATCHED == 1 << 28
