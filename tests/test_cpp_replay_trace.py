"""The host plan of bgr_replay_trace (sample frames and row counts, launch splitting under the trace budget, record
offsets, the kernel's field map, and every refusal of a trace's row range and field list) against a frame-by-frame
scan of random logs (tests/cpp/test_replay_trace.cpp).  Host only: the program is compiled with nvcc into a temporary
directory and needs no GPU."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_trace_plan_equals_a_frame_by_frame_scan(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = str(tmp_path / "test_replay_trace")
    src = os.path.join(ROOT, "tests", "cpp", "test_replay_trace.cpp")
    r = subprocess.run([nvcc, "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-o", out, src],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "replay trace plan test passed" in r.stdout
