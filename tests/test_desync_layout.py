"""The desync capture structs have one layout in C (the header, compiled), ctypes (capi.py) and the Rust -sys crate's
#[repr(C)] mirrors (rust_shim/bevy_ggrs_b200_sys/src/desync.rs, laid out with the C rules: no rustc here)."""
import ctypes as C
import os
import re
import subprocess

from bevy_ggrs_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCTS = {"bgr_desync_column": capi.bgr_desync_column, "bgr_desync_record": capi.bgr_desync_record,
           "bgr_desync_summary": capi.bgr_desync_summary}


def _c_layout(tmp_path):
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "bevy_ggrs_b200.h"', 'int main(void) {']
    for name, cst in STRUCTS.items():
        lines.append(f'printf("{name} size %zu\\n", sizeof({name}));')
        for f, _ in cst._fields_:
            lines.append(f'printf("{name} {f} %zu %zu\\n", offsetof({name}, {f}), sizeof((({name}*)0)->{f}));')
    lines += ['printf("flag %u none %u\\n", BGR_CFG_DESYNC_CAPTURE, BGR_DESYNC_NO_INDEX);', 'return 0; }']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    return subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines()


def test_c_and_ctypes_layouts_agree(tmp_path):
    out = _c_layout(tmp_path)
    for line in out:
        parts = line.split()
        if parts[0] == "flag":
            assert int(parts[1]) == capi.BGR_CFG_DESYNC_CAPTURE and int(parts[3]) == capi.BGR_DESYNC_NO_INDEX
        elif parts[1] == "size":
            assert int(parts[2]) == C.sizeof(STRUCTS[parts[0]]), line
        else:
            name, field, off, size = parts[0], parts[1], int(parts[2]), int(parts[3])
            desc = getattr(STRUCTS[name], field)
            assert (desc.offset, desc.size) == (off, size), line
    assert C.sizeof(capi.bgr_desync_column) == 16 and C.sizeof(capi.bgr_desync_record) == 20
    assert C.sizeof(capi.bgr_desync_summary) == 48


def test_rust_repr_c_mirrors_have_the_c_layout():
    rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200_sys", "src", "desync.rs")).read()
    prim = {"u32": 4, "i32": 4, "u64": 8}
    found = 0
    for m in re.finditer(r"#\[repr\(C\)\]\s*(?:#\[derive\([^)]*\)\]\s*)?pub struct (\w+) \{(.*?)\}", rs, re.S):
        name, body = m.group(1), m.group(2)
        fields = re.findall(r"pub (\w+): (\w+),", body)
        off, align, layout = 0, 1, []
        for f, ty in fields:
            sz = prim[ty]
            off = (off + sz - 1) // sz * sz
            layout.append((f, off, sz))
            off += sz
            align = max(align, sz)
        cst = STRUCTS[name]
        assert [f for f, _, _ in layout] == [f for f, _ in cst._fields_], name
        for f, o, sz in layout:
            assert (getattr(cst, f).offset, getattr(cst, f).size) == (o, sz), (name, f)
        assert (off + align - 1) // align * align == C.sizeof(cst), name
        found += 1
    assert found == len(STRUCTS)
    lib_rs = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200_sys", "src", "lib.rs")).read()
    assert "pub use desync::*;" in lib_rs
    assert re.search(r"pub const BGR_CFG_DESYNC_CAPTURE: u32 = %d;" % capi.BGR_CFG_DESYNC_CAPTURE, lib_rs)
    safe = open(os.path.join(ROOT, "rust_shim", "bevy_ggrs_b200", "src", "lib.rs")).read()
    assert "pub fn desync_report(" in safe and "sys::bgr_desync_diff(" in safe
