"""World checkpoints through the C++ host mirror (tests/cpp/test_checkpoint.cpp)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _binary():
    """Produced by __graft_entry__.build(); only (re)link the small C++ program here if it is missing."""
    import __graft_entry__ as g
    out = os.path.join(ROOT, "tests", "cpp", "test_checkpoint")
    if os.path.exists(out) and os.path.exists(g.LIB):
        return out
    if not os.path.exists(g.LIB):
        g.build_engine()
    return g.build_host_mirror_tests("test_checkpoint")


def test_checkpoint_mirror_builds_and_refuses_without_gpu():
    r = subprocess.run([_binary(), "--no-gpu"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ("engine started" if os.path.exists("/dev/nvidiactl") else "refused") in r.stdout, r.stdout


@pytest.mark.gpu
def test_app_checkpoint_continues_the_match_in_a_second_app():
    r = subprocess.run([_binary()], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "checkpoint test passed" in r.stdout
