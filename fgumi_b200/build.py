"""In-tree build of libfgumi_b200.so with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libfgumi_b200.so")
SOURCES = ["capi.cu", "host_tables.cpp", "host/caller_host.cpp", "host/bgzf.cpp"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-maxrregcount=112",      # upper bound only; vote_kernel must land at <= 96 (see _check_vote_kernel)
    "-fmad=false",            # no FMA contraction anywhere near the f64 vote (DESIGN.md numerics)
    "-Xcompiler", "-fPIC", "-shared",
    # host code (record parsing / assembly loops): AVX2-class auto-vectorisation; every H100 host has it
    "-Xcompiler", "-march=x86-64-v3", "-Xcompiler", "-ffp-contract=off",
]


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def _check_vote_kernel(ptxas_log: str) -> None:
    """Two 288-thread CTAs fit an SM only up to 96 registers per thread (registers are granted to
    10-warp blocks: 65536 / (2 * 10 * 32) = 102 -> 96), and a spill in the item loop costs ~10 %.
    ptxas' choice is sensitive to small source changes, so say so loudly when it drifts."""
    import re
    m = re.search(r"Function properties for \S*vote_kernelE\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores"
                  r".*\n.*Used (\d+) registers", ptxas_log)
    if not m:
        return
    spills, regs = int(m.group(2)), int(m.group(3))
    if regs > 96 or spills > 16:   # a word or two saved around the whole tile loop is harmless
        sys.stderr.write(f"fgumi_b200 build WARNING: vote_kernel uses {regs} registers with {spills} bytes of "
                         "spill stores; expected <= 96 and <= 16 (occupancy drops to one CTA per SM above 96)\n")


def build(force: bool = False, verbose: bool = False) -> str:
    deps = [os.path.join(dp, f) for dp, _, fs in os.walk(CSRC) for f in fs]
    deps.append(os.path.join(HERE, "..", "include", "fgumi_b200.h"))
    if not force and _newer(OUT, deps):
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-Xptxas", "-v", "-o", OUT] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libfgumi_b200.so")
    _check_vote_kernel(r.stdout + r.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
