"""Records/s of `fgumi filter --ref` from raw records (fgb_filter_records) on one GPU.

Workload: seeded, mapped 150-base simplex and duplex consensus records (pairs with a few mismatches; in one template
in ten a simplex record has a low-depth stretch that is masked and gets its template rejected) against a synthetic
genome that the script writes as FASTA to a temporary directory.  Reports records/s over the filter call, every phase
of RecordFilter.last_timing, the copy of the two streams into Python bytes, what is left of the call outside both
(other_ms), and the bytes the kernel passes move (records read and written by pass 1 and pass 2) over their CUDA-event
time against the H100's 3.35 TB/s, with the card's name and power limit read in the same run.  One JSON line on stdout.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_TBS = 3.35


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the number is still reported; the card is then unknown
        return f"unknown ({e})"


def workload(n_pairs: int, seed: int, genome_len: int = 20_000_000, length: int = 150):
    """(FASTA bytes, header text, bodies, rec_off): a genome of one contig and n_pairs templates of two records."""
    import struct
    rng = np.random.default_rng(seed)
    genome = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, genome_len)].tobytes()
    fasta = b">chr1\n" + b"\n".join(genome[i:i + 80] for i in range(0, genome_len, 80)) + b"\n"
    header = b"@HD\tVN:1.6\tSO:queryname\n@SQ\tSN:chr1\tLN:%d\n" % genome_len
    code = np.zeros(256, np.uint8)
    for i, c in enumerate(b"=ACMGRSVTWYHKDBN"):
        code[c] = i
    r = random.Random(seed)
    recs = []
    cd = struct.pack("<I", length) + np.full(length, 5, np.int16).tobytes()
    low = np.full(length, 5, np.int16)
    low[:40] = 1   # below min_reads 2: 40 bases masked, more than 20 % no-calls, the template rejected
    cd_low = struct.pack("<I", length) + low.tobytes()
    ce = struct.pack("<I", length) + np.zeros(length, np.int16).tobytes()
    for t in range(n_pairs):
        name = b"read%09d\0" % t
        duplex = t & 1
        for flag in (0x63, 0x93):
            pos = r.randrange(genome_len - 400)
            seq = np.frombuffer(genome[pos:pos + length], np.uint8).copy()
            for _ in range(r.randrange(4)):
                seq[r.randrange(length)] = b"ACGT"[r.randrange(4)]
            cig = struct.pack("<I", length << 4)
            packed = (code[seq[0::2]] << 4) | np.append(code[seq[1::2]], 0)[:len(seq[0::2])]
            quals = rng.integers(20, 41, length, dtype=np.uint8).tobytes()
            aux = b"NMC\x02MDZ150\0"
            depth = cd_low if t % 10 == 4 else cd   # an even t: a simplex template
            if duplex:
                aux += b"aDC\x03bDC\x02cDC\x05adBs" + depth + b"bdBs" + cd + b"aeBs" + ce + b"beBs" + ce
            else:
                aux += b"cDC\x05cdBs" + depth + b"ceBs" + ce
            body = struct.pack("<iiBBHHHIiii", 0, pos, len(name), 60, 0, 1, flag, length, 0, pos, 0)
            recs.append(body + name + cig + packed.astype(np.uint8).tobytes() + quals + aux)
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in recs])
    return fasta, header, np.frombuffer(b"".join(recs), np.uint8), off


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000, help="templates (two records each)")
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import filter as F
    fasta, header, bodies, off = workload(a.pairs, 1)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "genome.fa")
        with open(path, "wb") as f:
            f.write(fasta)
        ref = F.Reference(path)
    rf = F.RecordFilter(n_threads=a.threads, reverse_per_base_tags=True, track_rejects=True, min_reads=(2, 1, 1))
    best = None
    for _ in range(a.repeats + 1):   # one warm-up call, then the best of `repeats`
        t0 = time.perf_counter()
        kept, rej, st = rf.filter(header, bodies, off, ref)
        dt = time.perf_counter() - t0
        if best is None or dt < best[0]:
            best = (dt, rf.last_timing(), st, len(kept) + len(rej), rf.last_copy_s)
    rf.close()
    ref.close()
    dt, tm, st, out_bytes, copy_s = best
    n = len(off) - 1
    in_bytes = int(off[-1])
    kernel_s = (tm["pass1_ms"] + tm["pass2_ms"]) / 1e3
    moved = 2 * in_bytes + in_bytes + out_bytes   # pass 1 reads and writes the records, pass 2 reads and writes
    print(json.dumps({"bench": "filter_records", "card": card(), "records": n, "threads": a.threads,
                      "records_per_s": n / dt, "call_s": dt, **{k: round(v, 3) for k, v in tm.items()},
                      "library_ms": round(sum(tm.values()), 3), "copy_out_ms": round(copy_s * 1e3, 3),
                      "other_ms": round(dt * 1e3 - sum(tm.values()) - copy_s * 1e3, 3),
                      "kernel_bytes": moved, "kernel_tb_per_s": moved / kernel_s / 1e12 if kernel_s else None,
                      "kernel_fraction_of_peak": moved / kernel_s / 1e12 / PEAK_TBS if kernel_s else None,
                      **st}))


if __name__ == "__main__":
    main()
