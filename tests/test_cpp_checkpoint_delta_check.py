"""The host checks of a checkpoint delta's header and offsets (csrc/checkpoint_check.hpp checkpoint_delta_check, run by
bgr_checkpoint_restore_delta before anything is uploaded) against every malformed case with the restore's status and
message, and well-formed deltas written by the test (tests/cpp/test_checkpoint_delta_check.cpp).  Host only: the program
is compiled with nvcc into a temporary directory and needs no GPU."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_checkpoint_delta_host_checks_refuse_every_malformed_delta(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = str(tmp_path / "test_checkpoint_delta_check")
    src = os.path.join(ROOT, "tests", "cpp", "test_checkpoint_delta_check.cpp")
    r = subprocess.run([nvcc, "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-o", out, src],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "checkpoint delta host check test passed" in r.stdout
