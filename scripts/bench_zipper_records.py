"""Records/s of `fgumi zipper` from raw records (fgb_zipper_records) on one GPU.

Workload: N seeded aligned pairs (150-base reads, one in twenty with a supplementary record, both strands, AS / XS /
MC / MQ on the mapped side) and their unmapped originals carrying RX and the consensus per-base tags, zipped with the
Consensus reverse and revcomp sets.  Reports records/s over the zip call (input records of both streams), every phase
of Zipper.last_timing, the copy of the output into Python bytes, and the bytes the kernel passes move (both streams
read by the size pass, read again and the output written by the write pass) over their CUDA-event time against the
H100's 3.35 TB/s, with the card's name and power limit read in the same run.  One JSON line on stdout.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_TBS = 3.35


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the number is still reported; the card is then unknown
        return f"unknown ({e})"


_CODE = {c: i for i, c in enumerate(b"=ACMGRSVTWYHKDBN")}
_OPS = "MIDNSHP=X"


def make_record(name, flags, ref_id, pos, mapq=60, cigar=(), seq=b"", tags=()):
    """One raw BAM record (no block_size): cigar as text, tags as (tag, "Z" | "i" | "Bs", value)."""
    import re
    import struct
    ops = [int(n) << 4 | _OPS.index(o) for n, o in re.findall(r"(\d+)(\D)", cigar)] if cigar else []
    rec = bytearray(struct.pack("<iiBBHHHIiii", ref_id, pos, len(name) + 1, mapq, 4680, len(ops), flags, len(seq),
                                -1, -1, 0))
    rec += name + b"\0" + b"".join(struct.pack("<I", o) for o in ops)
    codes = [_CODE[c] for c in seq] + [0]
    rec += bytes(codes[i] << 4 | codes[i + 1] for i in range(0, len(seq), 2)) + bytes([30]) * len(seq)
    for tag, typ, val in tags:
        if typ == "Z":
            rec += tag + b"Z" + val + b"\0"
        elif typ == "i":
            rec += tag + b"i" + struct.pack("<i", val)
        else:
            rec += tag + b"Bs" + struct.pack("<I%dh" % len(val), len(val), *val)
    return bytes(rec)


def workload(n_pairs: int, seed: int, length: int = 150):
    import numpy as np
    r = random.Random(seed)
    rng = np.random.default_rng(seed)
    um, mp = [], []
    seq = rng.choice(list(b"ACGT"), length).astype(np.uint8).tobytes()
    per_base = [(b"cd", "Bs", [5] * length), (b"ce", "Bs", [0] * length), (b"cD", "Z", seq)]
    for t in range(n_pairs):
        name = b"read%09d" % t
        for f in (0x4D, 0x8D):
            um.append(make_record(name=name, flags=f, ref_id=-1, pos=-1, mapq=0, cigar="", seq=seq,
                                  tags=[(b"RX", "Z", b"ACGTACGT-TTGCAACG")] + per_base))
        p1, p2 = r.randrange(10_000_000), r.randrange(10_000_000)
        mp.append(make_record(name=name, flags=0x63, ref_id=0, pos=p1, cigar="%dM" % length, seq=seq,
                              tags=[(b"AS", "i", 140), (b"XS", "i", 20), (b"MC", "Z", b"%dM" % length)]))
        mp.append(make_record(name=name, flags=0x93, ref_id=0, pos=p2, cigar="%dM" % length, seq=seq,
                              tags=[(b"AS", "i", 150), (b"MQ", "i", 60)]))
        if t % 20 == 0:
            mp.append(make_record(name=name, flags=0x841, ref_id=1, pos=p1, cigar="50S100M", seq=seq,
                                  tags=[(b"AS", "i", 90)]))
    return um, mp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=250_000)   # about 1 M records in both streams
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=8)
    a = ap.parse_args()
    import numpy as np
    from fgumi_b200.zipper import Zipper

    def arrays(recs):
        off = np.zeros(len(recs) + 1, np.uint64)
        off[1:] = np.cumsum([len(r) for r in recs])
        return np.frombuffer(b"".join(recs), np.uint8), off
    um, mp = workload(a.pairs, a.seed)
    ub, uo = arrays(um)
    mb, mo = arrays(mp)
    z = Zipper(0, tags_to_reverse=["Consensus"], tags_to_revcomp=["Consensus"], n_threads=a.threads)
    z.zip(ub, uo, mb, mo)   # warm-up: module load, allocations
    best = None
    for _ in range(a.reps):
        t0 = time.perf_counter()
        data, used, stats = z.zip(ub, uo, mb, mo)
        dt = time.perf_counter() - t0
        tm = z.last_timing()
        if best is None or dt < best[0]:
            best = (dt, tm, z.last_copy_s, len(data), stats)
    z.close()
    dt, tm, copy_s, out_bytes, stats = best
    n_in = len(um) + len(mp)
    in_bytes = int(uo[-1]) + int(mo[-1])
    moved = 2 * in_bytes + out_bytes   # size pass reads both streams, write pass reads them and writes the output
    kernel_s = (tm["sizes_ms"] + tm["scan_ms"] + tm["write_ms"]) / 1e3
    print(json.dumps({"card": card(), "records_in": n_in, "records_out": stats["records_out"],
                      "records_per_s": n_in / dt, "call_s": dt, "copy_to_python_s": copy_s,
                      "other_ms": dt * 1e3 - copy_s * 1e3 - sum(tm.values()),
                      **{k: round(v, 3) for k, v in tm.items()}, "kernel_bytes": moved,
                      "kernel_share_of_3.35TBs": moved / kernel_s / (PEAK_TBS * 1e12) if kernel_s > 0 else None}))


if __name__ == "__main__":
    main()
