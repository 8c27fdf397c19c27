"""Content ids on their own (bevy_ggrs_b200/csrc/content_ids.hpp, tests/cpp/test_content_ids.cpp): LIFO slot reuse
derives equal ids, a different input, frame time or call count a new one, a spawn a fresh one, and the id table stays
trivially copyable.  Host code only: compiled here with the system C++ compiler, no GPU."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_content_id_derivation(tmp_path):
    exe = str(tmp_path / "test_content_ids")
    src = os.path.join(ROOT, "tests", "cpp", "test_content_ids.cpp")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, src], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "content id tests passed" in r.stdout


def test_host_state_stays_trivially_copyable():
    """The engine copies HostState, content ids included, on every handle_requests call: it must not allocate."""
    src = open(os.path.join(ROOT, "bevy_ggrs_b200", "csrc", "engine.cu")).read()
    assert "static_assert(std::is_trivially_copyable<HostState>::value" in src
    assert "ContentIds<SlotRing::kMaxSlots> cids;" in src
