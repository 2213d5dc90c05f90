"""Records/s of `fgumi group` from raw records (fgb_grouper_add_groups + fgb_grouper_flush) on one GPU.

Two workloads from synth.mapped_templates: mapped-like (many small position groups, adjacency k=1) and amplicon-like
(a few position groups of thousands of molecules, adjacency k=1 with the unmapped rules, so large calls take the
enumeration form).  For 1 and 16 host threads: host prepare (add_groups), the flush's device phase with the edge
kernels' CUDA-event time, the host rules, the emit and the rest of the flush (batch layout, the copy of the stream into
Python), and records/s over add + flush.  The card's name and power
limit are read in the same run.  One JSON line per row on stdout.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the number is still reported; the card is then unknown
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sites", type=int, default=200_000, help="position groups of the mapped-like workload")
    ap.add_argument("--amplicons", type=int, default=8, help="position groups of the amplicon-like workload")
    ap.add_argument("--amplicon-molecules", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import group, synth
    info = card()
    work = {
        "mapped": (synth.mapped_templates(a.sites, molecules=2, mean_family=2.0, umi_error_rate=0.01, seed=1),
                   dict(strategy="adjacency", edits=1)),
        "amplicon": (synth.mapped_templates(a.amplicons, molecules=a.amplicon_molecules, mean_family=3.0,
                                            umi_error_rate=0.01, seed=2),
                     dict(strategy="adjacency", edits=1, allow_unmapped=True)),
    }
    for name, ((hdr, b, off), opts) in work.items():
        keep, begin = group.group_by_position(b, off, hdr)
        kb, koff = group.compact(b, off, keep)
        n_rec = len(koff) - 1
        ref = None
        for threads in (1, 16):
            best = None
            for _ in range(a.repeats + 1):   # the first round warms the device and the allocations
                gr = group.ReadGrouper(0, n_threads=threads, **opts)
                t0 = time.perf_counter()
                gr.add_groups(kb, koff, begin)
                t1 = time.perf_counter()
                out = gr.flush()
                t2 = time.perf_counter()
                tm = gr.last_timing()
                gr.close()
                if ref is None:
                    ref = out
                assert out == ref, "output differs between thread counts"
                flush_ms = 1e3 * (t2 - t1)
                # what the flush's named parts leave out: laying out the UMI batch before the assignment and the copy
                # of the output stream into a Python bytes object
                other = flush_ms - sum(tm[k] for k in ("prepare_ms", "device_phase_ms", "resolve_ms", "emit_ms"))
                row = dict(workload=name, threads=threads, records=n_rec, position_groups=len(begin) - 1,
                           add_groups_ms=1e3 * (t1 - t0), flush_ms=flush_ms, **tm, other_ms=other,
                           records_per_s=n_rec / (t2 - t0), card=info)
                if best is None or row["records_per_s"] > best["records_per_s"]:
                    best = row
            print(json.dumps(best), flush=True)


if __name__ == "__main__":
    main()
