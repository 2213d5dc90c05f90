"""Records/s of `fgumi duplex-metrics` / `simplex-metrics` from raw records (fgb_metrics_*) on one GPU, beside the
`fgumi group` run that makes its input.

The mapped-like workload of bench_group_records.py (synth.mapped_templates, many small position groups, paired UMIs)
goes through the repo's group (paired strategy, so MIs carry /A and /B); its output is then fed to the collector in
both modes.  Per mode and thread count: records/s over add_records + finish and each phase (template pass, family
pass, UMI consensus, host work), best of --repeats after a warm-up round, and group's own records/s on the same input.
The card's name and power limit are read in the same run.  One JSON line per row on stdout.
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
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, group, metrics, synth
    info = card()
    hdr, b, off = synth.mapped_templates(a.sites, molecules=2, mean_family=2.0, paired_umis=True, umi_error_rate=0.01,
                                         seed=1)
    keep, begin = group.group_by_position(b, off, hdr)
    kb, koff = group.compact(b, off, keep)
    t0 = time.perf_counter()
    gr = group.ReadGrouper(0, strategy="paired", edits=1, n_threads=16)
    gr.add_groups(kb, koff, begin)
    stream = gr.flush()
    t_group = time.perf_counter() - t0
    bodies, rec_off = bamio.split_stream(stream)
    n = len(rec_off) - 1
    print(json.dumps({"bench": "group", "card": info, "records": len(koff) - 1, "seconds": round(t_group, 4),
                      "records_per_s": round((len(koff) - 1) / t_group)}), flush=True)
    for duplex in (True, False):
        for threads in (1, 16):
            best = None
            for _ in range(a.repeats + 1):   # the first round warms the device and the allocations
                m = metrics.MetricsCollector(hdr, duplex=duplex, device=0, n_threads=threads,
                                             duplex_umi_counts=duplex)
                t0 = time.perf_counter()
                m.add_records(bodies, rec_off)
                m.finish()
                dt = time.perf_counter() - t0
                row = dict(m.last_timing(), seconds=dt)
                m.close()
                if best is None or dt < best["seconds"]:
                    best = row
            print(json.dumps({"bench": "duplex-metrics" if duplex else "simplex-metrics", "card": info,
                              "records": n, "threads": threads, "seconds": round(best["seconds"], 4),
                              "records_per_s": round(n / best["seconds"]),
                              **{k: round(v, 2) for k, v in best.items() if k.endswith("_ms")}}), flush=True)


if __name__ == "__main__":
    main()
