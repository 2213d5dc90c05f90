"""Time fgb_umi_assign on the GPU (H100) over three `fgumi group`-shaped workloads, and sweep the all-pairs /
enumeration crossover.  Prints the card name and power limit of the same run and one JSON line per measurement.

  mapped      ~1 M position groups of 1-200 templates (log-uniform), 8-12 bp UMIs, adjacency k = 1, mapped rules
  amplicon    one deep call of ~1e5 unique UMIs (12 bp), adjacency k = 1, mapped rules
  unmapped    one `--allow-unmapped` call of 1-4 M unique 12-mers, adjacency k = 1 and k = 2, unmapped rules
  --crossover the same unmapped call shape at 1e3..1e5 unique keys, each form forced (FGB_UMI_ENUM_MIN_KEYS)

Times: `call` is the whole fgb_umi_assign (host clock around the synchronous call, median of --reps); the library's
own split of the same calls (fgb_umi_last_timing, medians): `prepare_ms` the host's key tables, `kernels_ms` the edge
kernels with the CUB sort / scan (CUDA events on the library's stream), `device_phase_ms` the whole device phase on the
host clock (staging, copies, kernels), `resolve_ms` the host's BFS / union-find / numbering.  The crossover is set from
`kernels_ms`.  fgumi's own CPU time cannot be measured here (it is not
built), so nothing is compared against it.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def umis_from_codes(codes: np.ndarray, lens: np.ndarray):
    """Fixed-width code array (bases as 0..3, padded) + per-UMI length -> (blob, umi_off)."""
    acgt = np.frombuffer(b"ACGT", np.uint8)
    mask = np.arange(codes.shape[1])[None, :] < lens[:, None]
    blob = acgt[codes][mask]
    off = np.zeros(len(lens) + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    return np.ascontiguousarray(blob), off


def mapped_workload(n_groups, seed=1):
    rng = np.random.default_rng(seed)
    T = np.exp(rng.uniform(0, np.log(200), n_groups)).astype(np.int64).clip(1, 200)   # templates per group
    L = rng.integers(8, 13, n_groups)
    M = np.maximum(1, T // 4)                                                         # molecules per group
    n = int(T.sum())
    g_of = np.repeat(np.arange(n_groups), T)
    mol = (rng.random(n) * M[g_of]).astype(np.int64)
    # a true UMI per (group, molecule): hash the pair into 12 bases, then 1 % per-base errors
    key = (g_of * 1_000_003 + mol * 7919 + seed) % (1 << 40)
    base = np.empty((n, 12), np.uint8)
    h = key.copy()
    for p in range(12):
        h = (h * 6364136223846793005 + 1442695040888963407) & ((1 << 62) - 1)
        base[:, p] = (h >> 33) & 3
    err = rng.random((n, 12)) < 0.01
    base = np.where(err, (base + rng.integers(1, 4, (n, 12))) % 4, base).astype(np.uint8)
    blob, umi_off = umis_from_codes(base, L[g_of])
    call_off = np.zeros(n_groups + 1, np.uint64)
    call_off[1:] = np.cumsum(T)
    group_off = np.arange(n_groups + 1, dtype=np.uint64)
    return blob, umi_off, call_off, group_off


def one_call(n_unique, L, seed, reads_per_key=1.5):
    rng = np.random.default_rng(seed)
    codes = np.unique(rng.integers(0, 4 ** L, int(n_unique * 1.02), dtype=np.int64))[:n_unique]
    reps = 1 + rng.poisson(reads_per_key - 1, len(codes))
    codes = np.repeat(codes, reps)
    codes = codes[rng.permutation(len(codes))]
    digits = ((codes[:, None] >> (2 * np.arange(L))[None, :]) & 3).astype(np.uint8)
    blob, umi_off = umis_from_codes(digits, np.full(len(codes), L))
    return blob, umi_off, np.array([0, len(codes)], np.uint64), np.array([0, 1], np.uint64)


def measure(fg, name, strategy, k, rules, data, reps, threads, extra=None):
    a = fg.UmiAssigner(0, strategy, k, rules, n_threads=threads)
    try:
        a.assign_packed(*data)                          # warm-up: module load, buffers, CUB temp storage
        ts, parts = [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            r = a.assign_packed(*data)
            ts.append(time.perf_counter() - t0)
            parts.append(a.last_timing())
    finally:
        a.close()
    med = {key: float(np.median([p[key] for p in parts])) for key in parts[0]}
    row = {"workload": name, "strategy": strategy, "edits": k, "rules": rules, "umis": len(data[1]) - 1,
           "calls": len(data[2]) - 1, "groups": len(data[3]) - 1, "mi": int(r.mi_counts.sum()),
           "call_s_median": float(np.median(ts)), "call_s_min": float(min(ts)), **med, "host_threads": threads}
    if extra:
        row.update(extra)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--unmapped", type=str, default="1000000,4000000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--crossover", action="store_true")
    ap.add_argument("--skip", type=str, default="")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import fgumi_b200 as fg
    print(f"card: {card()}", flush=True)
    skip = set(args.skip.split(","))
    if "mapped" not in skip:
        measure(fg, "mapped", "adjacency", 1, "mapped", mapped_workload(args.groups), args.reps, args.threads)
    if "amplicon" not in skip:
        measure(fg, "amplicon", "adjacency", 1, "mapped", one_call(100_000, 12, 3, reads_per_key=5), args.reps,
                args.threads)
    if "unmapped" not in skip:
        for n in [int(x) for x in args.unmapped.split(",") if x]:
            for k in (1, 2):
                measure(fg, "unmapped", "adjacency", k, "unmapped", one_call(n, 12, n + k), args.reps, args.threads)
    if args.crossover:
        for k in (1, 2):
            for n in (1000, 2000, 4000, 8000, 16000, 32000, 64000, 128000):
                data = one_call(n, 12, 5 + n)
                for form, env in (("all-pairs", str(1 << 40)), ("enumeration", "0")):
                    if form == "all-pairs" and n > 64000 and k == 1:
                        continue
                    os.environ["FGB_UMI_ENUM_MIN_KEYS"] = env
                    measure(fg, "crossover", "adjacency", k, "unmapped", data, args.reps, args.threads,
                            extra={"form": form, "unique": n})
        os.environ.pop("FGB_UMI_ENUM_MIN_KEYS", None)


if __name__ == "__main__":
    main()
