"""The replay's per-frame op derivation against compile_requests' ADVANCE ops (tests/cpp/test_replay_ops.cpp).  Host
only: the program is compiled with nvcc into a temporary directory and needs no GPU."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_replay_op_equals_the_host_advance(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = str(tmp_path / "test_replay_ops")
    src = os.path.join(ROOT, "tests", "cpp", "test_replay_ops.cpp")
    r = subprocess.run([nvcc, "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-Xcompiler", "-ffp-contract=off", "-o", out, src],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "replay op test passed" in r.stdout
