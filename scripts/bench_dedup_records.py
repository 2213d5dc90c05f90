"""Records/s of `fgumi dedup` from raw records (fgb_deduper_add_groups + fgb_deduper_flush) on one GPU, next to
`fgumi group` (fgb_grouper_*) on the same input.

Two workloads from synth.mapped_templates: mapped-like (many small position groups, adjacency k=1, with secondary and
supplementary records) and one large `--no-umi` pileup (a single position of many templates).  The duplicate rate is
the knob of the first: each molecule's family size is 1 + Poisson(mean - 1) with mean = 1 / (1 - rate), so about that
share of templates are duplicates.  For 1 and 16 host threads: records/s over add + flush, every phase of
Deduper.last_timing (the assignment's four, the score phase as the host saw it and its kernel by CUDA events, the
selection and emit), and the same input through ReadGrouper (its records/s and the dedup / group time ratio).  The
score phase runs on its own thread beside the assignment; whether it stays hidden is not assumed: `other_ms`, the part
of the flush outside the assignment and the emit, holds any wait for the scores (besides the batch layout, the thread
start and the copy of the stream into Python).  The card's name and power limit are read in the same run.
One JSON line per row on stdout.
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


def run(make, bodies, rec_off, begin, repeats):
    """Best of `repeats` (after one warm-up round): (add s, flush s, output, last_timing, metrics)."""
    best = None
    for _ in range(repeats + 1):
        x = make()
        t0 = time.perf_counter()
        x.add_groups(bodies, rec_off, begin)
        t1 = time.perf_counter()
        out = x.flush()
        t2 = time.perf_counter()
        tm, m = x.last_timing(), x.metrics()
        x.close()
        if best is None or t2 - t0 < best[0] + best[1]:
            best = (t1 - t0, t2 - t1, out, tm, m)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sites", type=int, default=200_000, help="position groups of the mapped-like workload")
    ap.add_argument("--duplicate-rate", type=float, default=0.6, help="share of duplicate templates (mapped-like)")
    ap.add_argument("--pileup", type=int, default=200_000, help="templates of the no-UMI pileup")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import dedup, group, synth
    info = card()
    mean = 1.0 / (1.0 - a.duplicate_rate)
    work = {
        "mapped": (synth.mapped_templates(a.sites, molecules=2, mean_family=mean, umi_error_rate=0.01,
                                          secondary_rate=0.05, read_length=100, seed=1),
                   dict(strategy="adjacency", edits=1), dict(strategy="adjacency", edits=1)),
        "no_umi_pileup": (synth.mapped_templates(1, molecules=1, mean_family=float(a.pileup), read_length=100, seed=2),
                          dict(strategy="identity", edits=0, no_umi=True),
                          dict(strategy="identity", edits=0, no_umi=True)),
    }
    for name, ((hdr, b, off), dopts, gopts) in work.items():
        _, dbegin = dedup.group_by_position(b, off, hdr)
        keep, gbegin = group.group_by_position(b, off, hdr)
        kb, koff = group.compact(b, off, keep)
        n_rec = len(off) - 1
        ref = None
        for threads in (1, 16):
            add, flush, out, tm, m = run(lambda: dedup.Deduper(0, n_threads=threads, **dopts), b, off, dbegin,
                                         a.repeats)
            if ref is None:
                ref = out
            assert out == ref, "output differs between thread counts"
            gadd, gflush, _, _, _ = run(lambda: group.ReadGrouper(0, n_threads=threads, **gopts), kb, koff, gbegin,
                                       a.repeats)
            assign_ms = sum(tm[k] for k in ("prepare_ms", "device_phase_ms", "resolve_ms"))
            other = 1e3 * flush - assign_ms - tm["emit_ms"]   # batch layout, thread start / join, Python copy
            row = dict(workload=name, threads=threads, records=n_rec, position_groups=len(dbegin) - 1,
                       add_groups_ms=1e3 * add, flush_ms=1e3 * flush, **tm, assignment_ms=assign_ms, other_ms=other,
                       records_per_s=n_rec / (add + flush), duplicate_rate=m["duplicate_rate"],
                       group_records=len(koff) - 1, group_records_per_s=(len(koff) - 1) / (gadd + gflush),
                       group_ms=1e3 * (gadd + gflush), dedup_over_group=(add + flush) / (gadd + gflush), card=info)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
