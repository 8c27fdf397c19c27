"""bgr_trace and bgr_trace_sample (include/bevy_ggrs_b200.h) have the same layout in the header and in capi.py: the
header's sizes and offsets, read by a C program compiled here, against the ctypes structures.  No GPU."""
import ctypes as C
import os
import subprocess

from bevy_ggrs_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = {
    "bgr_trace_sample": ["frame", "rows"],
    "bgr_trace": ["interval", "first_row", "n_rows", "n_fields", "fields", "dst", "dst_cap", "samples", "samples_cap",
                  "reserved"],
}
PINNED = {"bgr_trace_sample": 8, "bgr_trace": 56}


def test_trace_structs_match_the_header(tmp_path):
    src = tmp_path / "layout.c"
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "bevy_ggrs_b200.h"', "int main(void) {"]
    for name, fields in FIELDS.items():
        tag = "struct bgr_trace" if name == "bgr_trace" else name
        lines.append(f'printf("{name} size %zu\\n", sizeof({tag}));')
        for f in fields:
            lines.append(f'printf("{name} {f} %zu\\n", offsetof({tag}, {f}));')
    lines += ["return 0;", "}"]
    src.write_text("\n".join(lines))
    exe = str(tmp_path / "layout")
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    header = {tuple(l.split()[:2]): int(l.split()[2]) for l in got if l}
    for name, fields in FIELDS.items():
        cls = getattr(capi, name)
        assert header[(name, "size")] == C.sizeof(cls) == PINNED[name]
        assert [f for f, *_ in cls._fields_] == fields
        for f in fields:
            assert header[(name, f)] == getattr(cls, f).offset, (name, f)
