"""Records/s of `fgumi sort` on one GPU (fgb_sort_records), per phase, and `bamio.sort_file` end to end.

The workload is an aligner's unsorted output: paired 2 x 150 bp templates at random positions on 24 references, mates
adjacent, R1 forward and R2 reverse or the other way round, 1-9 soft-clipped bases, MC and RG on every record and
optionally CB and MI.  It is built by numpy in bulk (one fixed record layout filled column by column), so that the run
reaches tens of millions of records, the size at which users sort.  Rows, one JSON line each:
  - one-run sort, both orders: warm-up, then the best of --repeats: the phases of fgb_sort_last_timing, records/s
    over the call, and the gather kernel's bytes (each output byte read once and written once) over its time, as a
    share of the H100 SXM data-sheet 3.35 TB/s (the gather time includes the scan of the output offsets);
  - the same input forced into --runs runs (device_bytes set from the input size), with the host merge's time;
  - sort_file on a BAM of --file-records records: read / inflate / split (read_bam), device (the sort call) and
    compress (BGZF level 1), as wall seconds;
  - queryname order, lexicographic and natural, in one run and forced into --runs runs, on a second input: the same
    number of records with Illumina-style names A00123:8:HJKLMDSXY:<lane>:<tile>:<x>:<y> in coordinate order, so that
    the names arrive shuffled, with the key words per record and the number of them that vary (from the key words of
    a 100 000-record sample; the device skips the others).  --queryname-only runs these rows alone.
The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HEADER = ("@HD\tVN:1.6\tSO:unsorted\n" + "".join("@SQ\tSN:chr%d\tLN:250000000\n" % (i + 1) for i in range(24)) +
          "@RG\tID:A\tSM:s\tLB:L1\n@RG\tID:B\tSM:s\tLB:L2\n@RG\tID:C\tSM:s\tLB:L1\n"
          "@PG\tID:bwa\tPN:bwa\tCL:bwa mem\n").encode()


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the number is still reported; the card is then unknown
        return f"unknown ({e})"


def make_records(n_templates: int, cb: bool, mi: bool, seed: int = 1):
    """(bodies uint8[...], rec_off uint64[n + 1]) of 2 n_templates records in aligner order."""
    rng = np.random.default_rng(seed)
    L = 150
    name_len = 12                                    # "r%010d" + NUL
    layout = [("fixed", 32), ("name", name_len), ("cigar", 8), ("seq", L // 2), ("qual", L), ("mc", 3 + 7),
              ("rg", 3 + 2)] + ([("cb", 3 + 17)] if cb else []) + ([("mi", 3 + 9)] if mi else [])
    size = sum(w for _, w in layout)
    at, o = {}, 0
    for k, w in layout:
        at[k] = o
        o += w
    n = 2 * n_templates
    rec = np.empty((n, size), np.uint8)
    t = np.arange(n_templates, dtype=np.int64)
    tid = rng.integers(0, 24, n_templates).astype(np.int32)
    pos = rng.integers(0, 249_000_000, n_templates).astype(np.int32)
    insert = rng.integers(150, 600, n_templates).astype(np.int32)
    clip = rng.integers(1, 10, size=(n_templates, 2)).astype(np.int32)
    r1_rev = rng.random(n_templates) < 0.5
    for m in range(2):                               # m = 0: R1, 1: R2; R1 at pos forward unless r1_rev
        rows = slice(m, n, 2)
        rev = r1_rev if m == 0 else ~r1_rev
        left = (m == 0) != r1_rev                    # the forward mate sits at the left end
        p = np.where(left, pos, pos + insert - L)
        mp = np.where(left, pos + insert - L, pos)
        flag = (0x1 | 0x2 | (0x40 if m == 0 else 0x80) | np.where(rev, 0x10, 0x20)).astype(np.uint16)
        fixed = np.zeros(n_templates, dtype=[("tid", "<i4"), ("pos", "<i4"), ("lrn", "u1"), ("mapq", "u1"),
                                             ("bin", "<u2"), ("ncig", "<u2"), ("flag", "<u2"), ("lseq", "<u4"),
                                             ("mtid", "<i4"), ("mpos", "<i4"), ("tlen", "<i4")])
        fixed["tid"], fixed["pos"], fixed["lrn"], fixed["mapq"], fixed["bin"] = tid, p, name_len, 60, 4680
        fixed["ncig"], fixed["flag"], fixed["lseq"], fixed["mtid"], fixed["mpos"] = 2, flag, L, tid, mp
        fixed["tlen"] = np.where(left, insert, -insert)
        rec[rows, 0:32] = fixed.view(np.uint8).reshape(n_templates, 32)
        digits = (t[:, None] // (10 ** np.arange(9, -1, -1))) % 10
        rec[rows, at["name"]] = ord("r")
        rec[rows, at["name"] + 1:at["name"] + 11] = (48 + digits).astype(np.uint8)
        rec[rows, at["name"] + 11] = 0
        c_own, c_mate = clip[:, m], clip[:, 1 - m]
        cig = np.stack([(c_own << 4) | 4, ((L - c_own) << 4) | 0], 1).astype("<u4")
        rec[rows, at["cigar"]:at["cigar"] + 8] = cig.view(np.uint8).reshape(n_templates, 8)
        mc = np.empty((n_templates, 10), np.uint8)   # MC:Z:<c>S<150-c>M of the mate
        mc[:, 0:3] = np.frombuffer(b"MCZ", np.uint8)
        mc[:, 3] = 48 + c_mate
        mc[:, 4] = ord("S")
        rest = L - c_mate
        mc[:, 5], mc[:, 6], mc[:, 7] = 48 + rest // 100, 48 + rest // 10 % 10, 48 + rest % 10
        mc[:, 8], mc[:, 9] = ord("M"), 0
        rec[rows, at["mc"]:at["mc"] + 10] = mc
    pool = rng.integers(0, 256, size=(4096, L // 2 + L), dtype=np.uint8)   # SEQ / QUAL do not enter the keys
    rec[:, at["seq"]:at["seq"] + L // 2 + L] = pool[np.arange(n) % 4096]
    rg = np.frombuffer(b"ABC", np.uint8)[np.repeat(rng.integers(0, 3, n_templates), 2)]
    rec[:, at["rg"]:at["rg"] + 3] = np.frombuffer(b"RGZ", np.uint8)
    rec[:, at["rg"] + 3], rec[:, at["rg"] + 4] = rg, 0
    if cb:
        rec[:, at["cb"]:at["cb"] + 3] = np.frombuffer(b"CBZ", np.uint8)
        cells = rng.integers(0, 4, size=(2000, 16)).astype(np.uint8)
        rec[:, at["cb"] + 3:at["cb"] + 19] = np.frombuffer(b"ACGT", np.uint8)[cells][np.repeat(
            rng.integers(0, 2000, n_templates), 2)]
        rec[:, at["cb"] + 19] = 0
    if mi:
        rec[:, at["mi"]:at["mi"] + 3] = np.frombuffer(b"MIZ", np.uint8)
        mol = np.repeat(t // 3, 2)
        rec[:, at["mi"] + 3:at["mi"] + 11] = (48 + (mol[:, None] // (10 ** np.arange(7, -1, -1))) % 10).astype(np.uint8)
        rec[:, at["mi"] + 11] = 0
    off = np.arange(n + 1, dtype=np.uint64) * np.uint64(size)
    return rec.reshape(-1), off


def make_named_records(n: int, seed: int = 3):
    """(bodies, rec_off) of n records of 2 x 75 bp templates with Illumina-style names (lane 1-4, tile 1101-2678, x
    and y five digits; both mates share the name), R1 and R2 flags and 1 % secondary records, in coordinate order."""
    rng = np.random.default_rng(seed)
    L = 75
    prefix = b"A00123:8:HJKLMDSXY:"
    name_len = len(prefix) + 1 + 1 + 4 + 1 + 5 + 1 + 5 + 1   # fixed-width fields + NUL
    size = 32 + name_len + 4 + (L + 1) // 2 + L
    t = np.arange(n) // 2                                     # template of each record
    n_t = int(t[-1]) + 1
    fields = [rng.integers(1, 5, n_t), rng.integers(1101, 2679, n_t), rng.integers(10000, 32001, n_t),
              rng.integers(10000, 40001, n_t)]
    tid = rng.integers(0, 24, n).astype(np.int32)
    pos = rng.integers(0, 249_000_000, n).astype(np.int32)
    order = np.lexsort((pos, tid))                            # coordinate order: mates apart, names shuffled
    tid, pos, t = tid[order], pos[order], t[order]
    mate = order % 2
    flag = (0x1 | np.where(mate == 0, 0x40, 0x80) | np.where(rng.random(n) < 0.01, 0x100, 0)).astype(np.uint16)
    rec = np.zeros((n, size), np.uint8)
    fixed = np.zeros(n, dtype=[("tid", "<i4"), ("pos", "<i4"), ("lrn", "u1"), ("mapq", "u1"), ("bin", "<u2"),
                               ("ncig", "<u2"), ("flag", "<u2"), ("lseq", "<u4"), ("mtid", "<i4"), ("mpos", "<i4"),
                               ("tlen", "<i4")])
    fixed["tid"], fixed["pos"], fixed["lrn"], fixed["mapq"], fixed["bin"] = tid, pos, name_len, 60, 4680
    fixed["ncig"], fixed["flag"], fixed["lseq"], fixed["mtid"], fixed["mpos"] = 1, flag, L, -1, -1
    rec[:, 0:32] = fixed.view(np.uint8).reshape(n, 32)
    at = 32
    rec[:, at:at + len(prefix)] = np.frombuffer(prefix, np.uint8)
    at += len(prefix)
    for k, width in enumerate((1, 4, 5, 5)):
        v = fields[k][t]
        rec[:, at:at + width] = (48 + (v[:, None] // (10 ** np.arange(width - 1, -1, -1))) % 10).astype(np.uint8)
        at += width
        if k < 3:
            rec[:, at] = ord(":")
            at += 1
    at += 1                                                   # the NUL
    rec[:, at:at + 4] = np.frombuffer(struct.pack("<I", (L << 4) | 0), np.uint8)
    pool = rng.integers(0, 256, size=(4096, size - at - 4), dtype=np.uint8)
    rec[:, at + 4:] = pool[np.arange(n) % 4096]
    off = np.arange(n + 1, dtype=np.uint64) * np.uint64(size)
    return rec.reshape(-1), off


def key_word_counts(sort, bodies, off, order, sample: int = 100_000):
    """(key words per record, key words that vary) over a random sample of the records."""
    n = len(off) - 1
    idx = np.random.default_rng(0).choice(n, min(n, sample), replace=False)
    keys = np.array([sort.name_key(bodies[int(off[i]):int(off[i + 1])].tobytes(), order) for i in idx], np.uint64)
    rec0 = bodies[int(off[0]):int(off[1])]
    lrn = int(rec0[8]) - 1
    words = (lrn * (2 if order == "queryname::natural" else 1) + (1 if order == "queryname::natural" else 0) + 7) // 8
    varying = int(np.count_nonzero(np.bitwise_and.reduce(keys, 0) != np.bitwise_or.reduce(keys, 0)))
    return words + 1, varying


def timed_sort(sort, order, cb, bodies, off, repeats, device_bytes=0):
    s = sort.RecordSorter(0, order, b"CB" if cb else None, device_bytes=device_bytes)
    s.sort(HEADER, bodies, off)                      # warm-up: module load, CUB's kernels, host pages
    best = None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = s.sort(HEADER, bodies, off)
        wall = time.perf_counter() - t0
        if best is None or wall < best[0]:
            best = (wall, s.last_timing(), len(out))
        del out
    s.close()
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=20_000_000)
    ap.add_argument("--file-records", type=int, default=4_000_000)
    ap.add_argument("--runs", type=int, default=4, help="runs of the forced multi-run case")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cb", action="store_true", help="a 16-base CB on every record")
    ap.add_argument("--mi", action="store_true", help="an MI on every record")
    ap.add_argument("--queryname-only", action="store_true", help="only the queryname rows")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, lib, sort
    info = card()
    if not a.queryname_only:
        coordinate_rows(a, bamio, lib, sort, info)
    queryname_rows(a, sort, info)


def queryname_rows(a, sort, info):
    t0 = time.perf_counter()
    bodies, off = make_named_records(a.records)
    n = len(off) - 1
    common = dict(records=n, input_bytes=int(off[-1]), generate_s=time.perf_counter() - t0, card=info)
    for order in ("queryname", "queryname::natural"):
        words, varying = key_word_counts(sort, bodies, off, order)
        budget = (int(off[-1]) * 2 + n * (68 + 8 * words + 4)) // a.runs + 1
        for case, repeats, device_bytes in (("one_run", a.repeats, 0), ("forced_runs", 1, budget)):
            wall, tm, _ = timed_sort(sort, order, False, bodies, off, repeats, device_bytes)
            print(json.dumps(dict(case=case, order=order, device_bytes=device_bytes, wall_s=wall, records_per_s=n / wall,
                                  key_words=words, varying_key_words_in_sample=varying, **tm, **common)), flush=True)


def coordinate_rows(a, bamio, lib, sort, info):
    t0 = time.perf_counter()
    bodies, off = make_records(a.records // 2, a.cb, a.mi)
    n = len(off) - 1
    gen_s = time.perf_counter() - t0
    common = dict(records=n, input_bytes=int(off[-1]), cb=a.cb, mi=a.mi, generate_s=gen_s, card=info)
    for order in ("template-coordinate", "coordinate"):
        wall, tm, out_bytes = timed_sort(sort, order, a.cb, bodies, off, a.repeats)
        gather_bytes = 2 * out_bytes
        print(json.dumps(dict(case="one_run", order=order, wall_s=wall, records_per_s=n / wall, **tm,
                              gather_gb_per_s=gather_bytes / (tm["gather_ms"] * 1e6),
                              gather_share_of_3_35_tb_s=gather_bytes / (tm["gather_ms"] * 1e-3) / 3.35e12,
                              **common)), flush=True)
    budget = int(off[-1]) * 2 // a.runs + n * 120 // a.runs
    wall, tm, _ = timed_sort(sort, "template-coordinate", a.cb, bodies, off, 1, device_bytes=budget)
    print(json.dumps(dict(case="forced_runs", order="template-coordinate", device_bytes=budget, wall_s=wall,
                          records_per_s=n / wall, **tm, **common)), flush=True)
    del bodies
    # sort_file: a BGZF BAM of --file-records records in a temporary directory
    fb, foff = make_records(a.file_records // 2, a.cb, a.mi, seed=2)
    nf = len(foff) - 1
    blocks = np.empty((nf, 4 + int(foff[1])), np.uint8)
    blocks[:, :4] = np.frombuffer(struct.pack("<I", int(foff[1])), np.uint8)
    blocks[:, 4:] = fb.reshape(nf, -1)
    payload = bamio.mapped_bam_header(HEADER) + blocks.tobytes()
    del blocks, fb
    L = lib.load()
    import ctypes as C
    comp = np.empty(L.fgb_bgzf_bound(len(payload)), np.uint8)
    cn = C.c_size_t()
    assert L.fgb_bgzf_compress(payload, len(payload), 1, 16, 1, comp.ctypes.data, len(comp), C.addressof(cn)) == 0
    del payload
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bam"), os.path.join(d, "out.bam")
        comp[:cn.value].tofile(src)
        del comp
        s = sort.RecordSorter(0, "template-coordinate", b"CB" if a.cb else None)
        bamio.sort_file(src, dst, s, n_threads=16)   # warm-up
        best = None
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            tm = bamio.sort_file(src, dst, s, n_threads=16)
            wall = time.perf_counter() - t0
            if best is None or wall < best[0]:
                best = (wall, tm)
        wall, tm = best
        print(json.dumps(dict(case="sort_file", order="template-coordinate", records=nf, wall_s=wall,
                              records_per_s=nf / wall, **tm, card=info)), flush=True)


if __name__ == "__main__":
    main()
