"""App replays through the C++ host mirror (tests/cpp/test_app_replay.cpp), on the generated kernel, the interpreter
(BGR_TUNE_JIT=0) and BGR_CFG_FORCE_STEPWISE."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def binary(tmp_path_factory):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    lib = g.build_engine()
    out = str(tmp_path_factory.mktemp("app_replay") / "test_app_replay")
    src = os.path.join(ROOT, "tests", "cpp", "test_app_replay.cpp")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-ffp-contract=off", "-o", out, src,
                        "-L" + os.path.dirname(lib), "-lbevy_ggrs_b200", "-Wl,-rpath," + os.path.dirname(lib)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["jit", "interpreter", "stepwise"])
def test_cpp_app_replays_the_p2p_match(binary, path):
    env = dict(os.environ)
    if path != "stepwise":
        env["BGR_TUNE_JIT"] = "0" if path == "interpreter" else "2"
    r = subprocess.run([binary] + (["--stepwise"] if path == "stepwise" else []), capture_output=True, text=True,
                       timeout=600, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "app replay test passed" in r.stdout
