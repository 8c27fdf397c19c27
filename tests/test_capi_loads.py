"""CPU-only checks of the C-ABI library: it loads, exports every symbol the header declares, its
host-only entry points work, and it refuses to run without a GPU instead of falling back."""
import ctypes as C
import os
import re

import pytest

from bevy_ggrs_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_binds_all_prototypes():
    lib = capi.load_library()
    assert lib.bgr_abi_version() == capi.BGR_ABI_VERSION


def test_every_header_symbol_is_exported_and_bound():
    hdr = open(os.path.join(ROOT, "include", "bevy_ggrs_b200.h")).read()
    declared = set(re.findall(r"BGR_API\s+[\w\s\*]+?\b(bgr_\w+)\s*\(", hdr))
    assert len(declared) >= 40
    lib = capi.load_library()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert declared == set(capi.PROTOTYPES), declared ^ set(capi.PROTOTYPES)


def test_struct_layouts_match_the_header():
    assert C.sizeof(capi.bgr_request) == 28
    assert C.sizeof(capi.bgr_session_info) == 16
    assert C.sizeof(capi.bgr_checksum) == 24
    assert C.sizeof(capi.bgr_partial) == 24 + 8 * capi.BGR_MAX_CHECKSUM_COLUMNS
    assert C.sizeof(capi.bgr_config) == 40


def test_last_kernel_kinds_agree_across_header_ctypes_and_rust():
    """bgr_last_kernel's kind values are part of the ABI: the header's #defines, capi.py and the Rust constants agree,
    and Engine.last_kernel() decodes the documented bit layout."""
    from bevy_ggrs_b200.engine import LastKernel
    hdr = open(os.path.join(ROOT, "include", "bevy_ggrs_b200.h")).read()
    rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200_sys", "src", "lib.rs")).read()
    in_hdr = {k: int(v) for k, v in re.findall(r"#define (BGR_KERNEL_\w+) (\d+)u", hdr)}
    in_rs = {k: int(v) for k, v in re.findall(r"pub const (BGR_KERNEL_\w+): u32 = (\d+);", rs)}
    assert len(in_hdr) == 6 and in_hdr == in_rs
    assert all(getattr(capi, k) == v for k, v in in_hdr.items())
    # bundle, VEC 4, MODE 1, 1024-thread tier, passive TMA, whole-tile items
    raw = capi.BGR_KERNEL_BUNDLE | (4 << 4) | (1 << 8) | (2 << 10) | (1 << 12) | (512 << 16)
    assert LastKernel.decode(raw) == LastKernel("bundle", 4, 1, 2, True, 512, raw)
    assert LastKernel.decode(capi.BGR_KERNEL_GENERIC_NVRTC | (128 << 16)).item_rows == 128
    assert LastKernel.decode(capi.BGR_KERNEL_STEPWISE_FLAT).kind == "stepwise_flat"


def test_ggrs_time_delta_bits_matches_oracle(oracle_lib):
    lib = capi.load_library()
    for fps in (30, 60, 144):
        for frame in range(1, 400):
            assert lib.bgr_ggrs_time_delta_bits(fps, frame) == oracle_lib.orc_ggrs_time_delta_bits(fps, frame)


def test_fold_partials_matches_golden_composition():
    """checksum = entity_part ^ part(col0) ^ part(col1) with SURVEY §8c vectors."""
    lib = capi.load_library()
    p = capi.bgr_partial()
    p.frame, p.n_columns, p.active, p.total = 7, 1, 2, 2
    p.xor_[0] = 0x27EA43A38B7BD31A  # per-entity hash of translation (1,2,3), order 0
    cs = capi.bgr_checksum()
    assert lib.bgr_fold_partials(C.byref(p), C.byref(cs)) == 0
    assert cs.hi == 0 and cs.frame == 7
    assert cs.lo == 0x92B817690FA6BA0D ^ 0xC91E3FA134760483
    p.n_columns = 0
    lib.bgr_fold_partials(C.byref(p), C.byref(cs))
    assert cs.lo == 0x92B817690FA6BA0D


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="GPU present")
def test_no_gpu_fails_loudly_no_cpu_fallback():
    from bevy_ggrs_b200.engine import Engine
    with pytest.raises(capi.BgrError) as ei:
        Engine(max_entities=16)
    assert ei.value.status == capi.BGR_ERR_CUDA
    assert "no CPU fallback" in str(ei.value)


def test_rust_ffi_source_declares_every_engine_symbol():
    """rust_shim/ is source only (no rustc here), but it must not rot: every engine entry point of the header
    (the bgr_ring_* host-test hooks aside) has an `extern "C"` declaration and the #[repr(C)] structs keep the
    field order of the C structs."""
    hdr = open(os.path.join(ROOT, "include", "bevy_ggrs_b200.h")).read()
    rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200_sys", "src", "lib.rs")).read()
    declared = set(re.findall(r"BGR_API\s+[\w\s\*]+?\b(bgr_\w+)\s*\(", hdr))
    have = set(re.findall(r"pub fn (bgr_\w+)", rs))
    assert {d for d in declared if not d.startswith("bgr_ring_")} <= have
    for struct, fields in (("bgr_request", ["kind", "frame", "n_players", "inputs", "status"]),
                           ("bgr_config", ["abi_version", "device", "max_entities", "max_depth", "fps", "flags", "order_base", "stream"]),
                           ("bgr_checksum", ["frame", "has_checksum", "lo", "hi"])):
        body = rs[rs.index("pub struct " + struct):]
        body = body[:body.index("}")]
        assert re.findall(r"pub (\w+):", body) == fields


def test_rust_ffi_repr_c_structs_have_the_c_layout():
    """Without rustc the -sys crate cannot be compiled, but its #[repr(C)] structs can still be checked: parse every
    struct, lay it out with the C rules (natural alignment) and compare field order, offsets and total size with the
    ctypes mirror of the header (capi.py) — which test_struct_layouts_match_the_header pins to the header's sizes."""
    rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200_sys", "src", "lib.rs")).read()
    consts = {k: int(v, 0) for k, v in re.findall(r"pub const (\w+): \w+ = (0x[0-9a-fA-F]+|\d+);", rs)}
    prim = {"u8": 1, "i8": 1, "u16": 2, "i16": 2, "u32": 4, "i32": 4, "f32": 4, "u64": 8, "i64": 8, "usize": 8,
            "*mut c_void": 8, "*const c_void": 8}

    def size_align(ty):
        ty = ty.strip()
        m = re.fullmatch(r"\[(\w+); (\w+)\]", ty)
        if m:
            n = consts[m.group(2)] if not m.group(2).isdigit() else int(m.group(2))
            return prim[m.group(1)] * n, prim[m.group(1)]
        return prim[ty], prim[ty]

    mirrors = {"bgr_request": capi.bgr_request, "bgr_session_info": capi.bgr_session_info, "bgr_checksum": capi.bgr_checksum,
               "bgr_partial": capi.bgr_partial, "bgr_config": capi.bgr_config}
    found = 0
    for m in re.finditer(r"#\[repr\(C\)\]\s*(?:#\[derive\([^)]*\)\]\s*)?pub struct (\w+) \{(.*?)\}", rs, re.S):
        name, body = m.group(1), m.group(2)
        fields = re.findall(r"pub (\w+): ([^,\n]+),", body)
        off, max_align, layout = 0, 1, []
        for fname, ty in fields:
            sz, al = size_align(ty)
            off = (off + al - 1) // al * al
            layout.append((fname, off, sz))
            off += sz
            max_align = max(max_align, al)
        total = (off + max_align - 1) // max_align * max_align
        cst = mirrors[name]
        assert [f for f, _, _ in layout] == [f for f, _ in cst._fields_], name
        for fname, o, sz in layout:
            assert getattr(cst, fname).offset == o and getattr(cst, fname).size == sz, (name, fname)
        assert total == C.sizeof(cst), name
        found += 1
    assert found == len(mirrors)
    assert consts["BGR_MAX_PLAYERS"] == capi.BGR_MAX_PLAYERS and consts["BGR_MAX_REQUESTS"] == capi.BGR_MAX_REQUESTS
    assert consts["BGR_MAX_CHECKSUM_COLUMNS"] == capi.BGR_MAX_CHECKSUM_COLUMNS


def test_rust_shim_keeps_the_reference_api_names():
    """The drop-in crate exposes the reference's RollbackApp / GgrsPlugin names (rollback_app.rs:31-133, lib.rs:198-224),
    not renamed `_b200` variants."""
    rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200", "src", "lib.rs")).read()
    for name in ("rollback_component_with_copy", "rollback_component_with_clone", "checksum_component_with_hash",
                 "checksum_component", "rollback_resource_with_copy", "rollback_resource_with_clone", "checksum_resource_with_hash"):
        assert re.search(r"fn %s<" % name, rs), name
    assert "pub struct GgrsPlugin<C: Config>" in rs and "pub trait RollbackApp" in rs
    assert "_b200::<" not in rs and "fn handle_requests<" in rs and "fn run_ggrs_schedules<" in rs
    assert "On<Add, Rollback>" in rs and "bgr_spawn" in rs          # Rollback on_add -> engine row (rollback.rs:40-54)
    for item in ("Rollback", "Session", "GgrsSchedule", "ReadInputs", "LocalInputs", "PlayerInputs", "SyncTestMismatch"):
        assert re.search(r"pub use bevy_ggrs::\{[^}]*\b%s\b" % item, rs, re.S), item
