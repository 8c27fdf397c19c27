"""scripts/sass_budget.py compiles the engine for sm_90a and attributes the bundle kernel's SASS to source regions; no GPU
needed.  This checks that it runs, finds the six instances the engine launches by default, and that none of them spills
or loses the three resident 256-thread blocks per SM the kernel is tuned for.  It pins no instruction counts."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_sass_budget_runs_and_reports_no_spills():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not installed")
    if not os.path.exists(os.environ.get("NVDISASM", "/usr/local/cuda/bin/nvdisasm")):
        pytest.skip("nvdisasm not installed")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "sass_budget.py")], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    inst = out["instances"]
    assert sorted(inst) == sorted(f"k_particles_program<{m},{s},false>" for m in range(3) for s in ("false", "true"))
    for name, b in inst.items():
        assert b["spill_stores"] == 0 and b["spill_loads"] == 0, name
        assert b["blocks_per_sm_by_registers"] >= 3, name
        assert b["regions"]["save_hash"]["imad"] > 0 and b["regions"]["advance"]["fp32"] > 0, name
        assert b["total"]["all"] == sum(r["total"] for r in b["regions"].values()), name
