"""Static instruction budget of the bundle kernel (k_particles_program), per region and per issue pipe.  Needs no GPU.

Compiles bevy_ggrs_b200/csrc/engine.cu with the engine's own flags (__graft_entry__.NVCC_FLAGS) into a cubin, runs
`nvdisasm -gi`, and attributes every SASS instruction of every k_particles_program instance to the region of the kernel
source it came from.  nvdisasm prints the inline chain of each instruction (`seahash.cuh line 35 inlined at seahash.cuh
line 58 inlined at kernels.cuh line 794`); the outermost kernels.cuh line of the chain is the statement of the kernel
body, and the `budget: <region>` markers in kernels.cuh name the region each statement belongs to (a marker holds
until the next one).  Within each region the count is split by issue pipe:

    imad   IMAD* (IMAD, IMAD.WIDE, IMAD.IADD, IMAD.MOV, ...): the half-rate integer multiply-add pipe
    alu    integer ALU (LOP3, SHF, IADD3, ISETP, SEL, PLOP3, LEA, ...)
    fp32   FADD / FMUL / FFMA / FSETP / FMNMX / FSEL ...
    other  memory, control flow, warp votes and reductions, uniform datapath, conversions

It also reports registers, spills and the 256-thread blocks per SM the register count allows (-Xptxas -v), and the
warp reductions (REDUX) of each region: the default instances reduce a Save's checksum partials in per-lane shared
memory slots, so their save_fold has none.

A static count is not a timing: predicated-off instructions and code the workload never reaches count like the hot
path.  It tells where a change can cut instructions, not what the cut is worth.

    python scripts/sass_budget.py [--instances default|all] [--cubin FILE --ptxas-log FILE]

One JSON line on stdout.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bevy_ggrs_b200", "csrc")
KERNELS = os.path.join(CSRC, "kernels.cuh")
KERNEL = "k_particles_program"
REGIONS = ["prologue", "tile_loop", "load", "advance", "save_track", "save_store", "save_hash", "save_fold", "epilogue"]
PIPES = ["imad", "alu", "fp32", "other"]
ALU = {"LOP3", "LOP", "SHF", "SHL", "SHR", "IADD3", "IADD", "ISETP", "SEL", "PLOP3", "LEA", "VIADD", "VIADDMNMX",
       "VIMNMX", "IMNMX", "IABS", "PRMT", "MOV", "P2R", "R2P", "POPC", "FLO", "BMSK", "BREV", "ICMP", "ISCADD", "SGXT"}
FP32 = {"FADD", "FMUL", "FFMA", "FSETP", "FMNMX", "FSEL", "FSET", "FCHK", "FRND", "FSWZADD"}
REGS_PER_SM, BLOCK = 65536, 256


def _nvcc_flags():
    sys.path.insert(0, ROOT)
    from __graft_entry__ import NVCC_FLAGS
    flags, skip = [], 0
    for f in NVCC_FLAGS:
        if skip:
            skip -= 1
            continue
        if f == "-cudart":  # host-link options: a cubin links nothing
            skip = 1
            continue
        flags.append("-cubin" if f == "-shared" else f)
    return flags


def compile_cubin(out_dir: str):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cubin = os.path.join(out_dir, "engine.cubin")
    r = subprocess.run([nvcc] + _nvcc_flags() + ["-Xptxas", "-v", "-o", cubin, os.path.join(CSRC, "engine.cu")],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return cubin, r.stderr


def ptxas_resources(log: str) -> dict:
    """mangled name -> {registers, spill_stores, spill_loads, stack}"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), {})
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur.update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            cur["registers"] = int(m.group(1))
    return out


def region_map() -> dict:
    """kernels.cuh line -> region, for the lines of k_particles_program's body"""
    lines = open(KERNELS).read().splitlines()
    start = next(i for i, l in enumerate(lines) if re.search(KERNEL + r"\(const __grid_constant__", l))
    out, region = {}, None
    for i in range(start, len(lines)):
        m = re.search(r"budget: (\w+)", lines[i])
        if m:
            region = m.group(1)
            if region not in REGIONS:
                raise ValueError(f"kernels.cuh:{i + 1}: unknown budget region {region!r}")
        if i > start and lines[i].startswith("}"):  # the kernel's closing brace
            break
        out[i + 1] = region
    return out


def pipe_of(opcode: str) -> str:
    base = opcode.split(".")[0]
    if base == "IMAD":
        return "imad"
    if base in ALU:
        return "alu"
    if base in FP32:
        return "fp32"
    return "other"


_LOC = re.compile(r'"([^"]+)", line (\d+)')
_INSN = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)")


def budget(sass: str, lines_to_region: dict) -> tuple[dict, dict]:
    """per-instance {region: {pipe: count}} and {region: REDUX count} from nvdisasm -gi output"""
    out, redux, cur, red, region = {}, {}, None, None, "other"
    for line in sass.splitlines():
        if line.startswith("//---------------------") and ".text." in line:
            name = line.split(".text.", 1)[1].split()[0]
            cur = out.setdefault(name, {r: dict.fromkeys(PIPES, 0) for r in REGIONS + ["other"]}) if KERNEL in name else None
            red = redux.setdefault(name, dict.fromkeys(REGIONS + ["other"], 0)) if KERNEL in name else None
            region = "other"
            continue
        if cur is None:
            continue
        if line.lstrip().startswith("//## File"):
            locs = [(f, int(n)) for f, n in _LOC.findall(line) if f.endswith("kernels.cuh")]
            region = (lines_to_region.get(locs[-1][1]) or "other") if locs else "other"
            continue
        m = _INSN.match(line)
        if m and m.group(1) not in ("NOP",):
            cur[region][pipe_of(m.group(1))] += 1
            red[region] += m.group(1).startswith("REDUX")
    return out, redux


def demangle_params(name: str) -> str:
    """<MODE,STAMPS,VERIFY>, with a fourth argument `true` for the warp-fold instances (WARP_FOLD defaults to false)"""
    m = re.search(KERNEL + r"ILi(\d)ELb([01])ELb([01])E(?:Lb([01])E)?", name)
    args = [m.group(1)] + ["true" if m.group(i) == "1" else "false" for i in (2, 3)] + (["true"] if m.group(4) == "1" else [])
    return f"{KERNEL}<{','.join(args)}>"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--instances", choices=["default", "all"], default="default",
                    help="default: the six instances that run by default (VERIFY=false, lane fold)")
    ap.add_argument("--cubin", help="an engine cubin built already (with --ptxas-log, the -Xptxas -v output)")
    ap.add_argument("--ptxas-log")
    args = ap.parse_args()
    nvdisasm = os.environ.get("NVDISASM", "/usr/local/cuda/bin/nvdisasm")
    with tempfile.TemporaryDirectory() as tmp:
        if args.cubin:
            cubin, log = args.cubin, open(args.ptxas_log).read() if args.ptxas_log else ""
        else:
            cubin, log = compile_cubin(tmp)
        r = subprocess.run([nvdisasm, "-gi", cubin], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvdisasm failed:\n" + r.stderr)
        sass = r.stdout
    res = ptxas_resources(log)
    per, redux = budget(sass, region_map())
    instances = {}
    for name in sorted(per):
        label = demangle_params(name)
        if args.instances == "default" and label.endswith(",true>"):
            continue
        regions = {rg: dict(c, total=sum(c.values())) for rg, c in per[name].items() if sum(c.values())}
        rs = res.get(name, {})
        regs = rs.get("registers")
        instances[label] = {
            "registers": regs, "spill_stores": rs.get("spill_stores"), "spill_loads": rs.get("spill_loads"),
            "blocks_per_sm_by_registers": REGS_PER_SM // (-(-regs // 8) * 8 * BLOCK) if regs else None,
            "total": {p: sum(c[p] for c in per[name].values()) for p in PIPES} | {"all": sum(sum(c.values()) for c in per[name].values())},
            "regions": regions,
            "redux": {rg: c for rg, c in redux[name].items() if c},
        }
    print(json.dumps({"kernel": KERNEL, "instances": instances}))


if __name__ == "__main__":
    main()
