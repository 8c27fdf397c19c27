"""The keyframe plan of bgr_replay_keyframes (placement, byte bound, and each blob header's rows, Time<GgrsTime> and
ParticleRng) against a frame-by-frame restatement of the request stream (tests/cpp/test_replay_keyframes.cpp).  Host
only: the program is compiled with nvcc into a temporary directory and needs no GPU."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_keyframe_plan_equals_the_request_stream(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = str(tmp_path / "test_replay_keyframes")
    src = os.path.join(ROOT, "tests", "cpp", "test_replay_keyframes.cpp")
    r = subprocess.run([nvcc, "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-Xcompiler", "-ffp-contract=off", "-o", out, src],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "replay keyframe plan test passed" in r.stdout
