"""In-tree build of libfgumi_b200.so with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libfgumi_b200.so")
SOURCES = ["capi.cu", "host_tables.cpp", "host/caller_host.cpp", "host/bgzf.cpp", "host/umi_host.cpp",
           "host/group_host.cpp", "host/sort_host.cpp", "host/dedup_host.cpp", "host/filter_host.cpp",
           "metrics.cu", "host/metrics_host.cpp", "zipper.cu", "host/zipper_host.cpp"]
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


def _check_umi_kernels(ptxas_log: str) -> None:
    """The UMI edge kernels keep a query key and a short scalar state per thread in registers: a spill or a stack
    frame means a source change pushed the comparator into local memory, and fails the build."""
    import re
    found = 0
    for m in re.finditer(r"Function properties for (\S*umi_\w+_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores",
                         ptxas_log):
        found += 1
        if int(m.group(2)) or int(m.group(3)):
            raise RuntimeError(f"fgumi_b200 build: {m.group(1)} has a {m.group(2)}-byte stack frame and spills "
                               f"{m.group(3)} bytes (expected none)")
    if found != 4:
        raise RuntimeError(f"fgumi_b200 build: ptxas reported {found} UMI edge kernels, expected 4")


def _check_sort_kernels(ptxas_log: str) -> None:
    """The sort's key kernels walk a record's CIGAR, aux block and MC string, or stream its read name, in registers,
    and the gather kernel copies with a few words per lane: a stack frame or a spill means a source change pushed the
    key state into local memory, and fails the build."""
    import re
    found = 0
    for m in re.finditer(r"Function properties for (\S*sort_(?:name_key|key|gather)_kernel\S*)\n\s*(\d+) bytes stack "
                         r"frame, (\d+) bytes spill stores", ptxas_log):
        found += 1
        if int(m.group(2)) or int(m.group(3)):
            raise RuntimeError(f"fgumi_b200 build: {m.group(1)} has a {m.group(2)}-byte stack frame and spills "
                               f"{m.group(3)} bytes (expected none)")
    if found != 4:
        raise RuntimeError(f"fgumi_b200 build: ptxas reported {found} sort key / gather kernels, expected 4")


def _check_score_kernel(ptxas_log: str) -> None:
    """The template-score kernel keeps one accumulator and a uint4 per lane: a stack frame or a spill means a source
    change pushed its state into local memory, and fails the build."""
    import re
    m = re.search(r"Function properties for (\S*dedup_score_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                  r"stores", ptxas_log)
    if not m:
        raise RuntimeError("fgumi_b200 build: ptxas reported no dedup_score_kernel")
    if int(m.group(2)) or int(m.group(3)):
        raise RuntimeError(f"fgumi_b200 build: {m.group(1)} has a {m.group(2)}-byte stack frame and spills "
                           f"{m.group(3)} bytes (expected none)")


def _check_filter_kernels(ptxas_log: str) -> None:
    """The record filter's kernels keep a record's walk state and tag references in registers: a stack frame or a spill
    means a source change pushed them into local memory, and fails the build."""
    import re
    found = 0
    for m in re.finditer(r"Function properties for (\S*filter_(?:pass1|decide|sizes|pass2)_kernel\S*)\n\s*(\d+) bytes "
                         r"stack frame, (\d+) bytes spill stores", ptxas_log):
        found += 1
        if int(m.group(2)) or int(m.group(3)):
            raise RuntimeError(f"fgumi_b200 build: {m.group(1)} has a {m.group(2)}-byte stack frame and spills "
                               f"{m.group(3)} bytes (expected none)")
    if found != 4:
        raise RuntimeError(f"fgumi_b200 build: ptxas reported {found} record filter kernels, expected 4")


def _check_metrics_kernels(ptxas_log: str) -> None:
    """The metrics kernels keep a template's walk state and a family's running counts in registers (the per-bucket
    counts live in shared memory): a stack frame or a spill means a source change pushed them into local memory, and
    fails the build."""
    import re
    found = 0
    for m in re.finditer(r"Function properties for (\S*metrics_\w+_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes "
                         r"spill stores", ptxas_log):
        found += 1
        if int(m.group(2)) or int(m.group(3)):
            raise RuntimeError(f"fgumi_b200 build: {m.group(1)} has a {m.group(2)}-byte stack frame and spills "
                               f"{m.group(3)} bytes (expected none)")
    if found != 6:
        raise RuntimeError(f"fgumi_b200 build: ptxas reported {found} metrics kernels, expected 6")


def _check_zipper_kernels(ptxas_log: str) -> None:
    """The zipper's kernels keep a record's plan (mate fields, tag-edit decisions, tc values) in registers: a stack
    frame or a spill means a source change pushed it into local memory, and fails the build."""
    import re
    found = 0
    for m in re.finditer(r"Function properties for (\S*zipper_(?:sizes|write)_kernel\S*)\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores", ptxas_log):
        found += 1
        if int(m.group(2)) or int(m.group(3)):
            raise RuntimeError(f"fgumi_b200 build: {m.group(1)} has a {m.group(2)}-byte stack frame and spills "
                               f"{m.group(3)} bytes (expected none)")
    if found != 2:
        raise RuntimeError(f"fgumi_b200 build: ptxas reported {found} zipper kernels, expected 2")


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
    _check_umi_kernels(r.stdout + r.stderr)
    _check_sort_kernels(r.stdout + r.stderr)
    _check_score_kernel(r.stdout + r.stderr)
    _check_filter_kernels(r.stdout + r.stderr)
    _check_metrics_kernels(r.stdout + r.stderr)
    _check_zipper_kernels(r.stdout + r.stderr)
    return OUT


def build_variant(out: str, defines, verbose: bool = False) -> str:
    """Build the library with extra preprocessor definitions (e.g. {"FGB_PIPE_TRACE": 1}) to `out`, always from
    scratch: diagnostic and A/B builds loaded through FGUMI_B200_LIB.  The in-tree library is left alone."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    defs = [f"-D{k}={v}" for k, v in dict(defines).items()]
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    cmd = [nvcc] + NVCC_FLAGS + defs + ["-Xptxas", "-v", "-o", out] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed building {out}")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
