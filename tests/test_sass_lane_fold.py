"""scripts/sass_budget.py on every k_particles_program instance (no GPU needed): the instances that run by default fold
each Save's checksum partials into per-lane shared-memory slots, so their save_fold region holds no warp reduction
(REDUX); the warp-fold instances, which launches take only where the slots would cost a resident block, still reduce
there.  No instance spills."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_default_instances_fold_without_redux_and_nothing_spills():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not installed")
    if not os.path.exists(os.environ.get("NVDISASM", "/usr/local/cuda/bin/nvdisasm")):
        pytest.skip("nvdisasm not installed")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "sass_budget.py"), "--instances", "all"],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    inst = json.loads(r.stdout.strip().splitlines()[-1])["instances"]
    default = [f"k_particles_program<{m},{s},false>" for m in range(3) for s in ("false", "true")]
    warp = [name[:-1] + ",true>" for name in default]
    verify = [f"k_particles_program<{m},{s},true>" for m in range(3) for s in ("false", "true")]
    assert sorted(inst) == sorted(default + warp + verify)
    for name, b in inst.items():
        assert b["spill_stores"] == 0 and b["spill_loads"] == 0, name
        assert b["blocks_per_sm_by_registers"] >= 3, name
    for name in default + verify:
        assert inst[name]["regions"]["save_fold"]["total"] > 0, name
        assert inst[name]["redux"].get("save_fold", 0) == 0, (name, inst[name]["redux"])
    for name in warp:
        assert inst[name]["redux"].get("save_fold", 0) >= 3, (name, inst[name]["redux"])
