"""The host side of a batched edit call (csrc/edit_batch.hpp, run by bgr_batch_apply_edits before anything runs): every
refusal of an entry with its status, message and entry, and the patch layout against hand-computed offsets
(tests/cpp/test_edit_batch.cpp).  Host only: the program is compiled with nvcc into a temporary directory and needs no
GPU."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_batched_edit_host_checks_and_layout(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = str(tmp_path / "test_edit_batch")
    src = os.path.join(ROOT, "tests", "cpp", "test_edit_batch.cpp")
    r = subprocess.run([nvcc, "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-o", out, src],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "edit batch host check test passed" in r.stdout
