"""Seeded raw records for the sort tests: every kind of record the sort keys treat differently."""
import struct

import numpy as np

from tests.bam_builder import make_record

HEADER = (b"@HD\tVN:1.6\tSO:unsorted\n@SQ\tSN:chr1\tLN:1000000\n"
          b"@RG\tID:A\tSM:s\tLB:libB\n@RG\tID:B\tSM:s\tLB:libA\n@RG\tID:C\tSM:s\n"
          b"@RG\tID:D\tSM:s\tLB:unknown\n@RG\tID:E\tSM:s\tLB:libA\n@PG\tID:bwa\tPN:bwa\n")
MC_VALUES = [b"10M", b"5S10M", b"3H2S10M4S1H", b"10M5S3M2S", b"4M2D3N2=1X6S", b"", b"abc", b"12", b"M5S",
             b"99999999999M", b"2S99999999999S8M", b"0S10M0H", b"\xff\xfe10M", b"10M\xc3"]
MI_Z = [b"123", b"45/A", b"6/B", b"/A", b"", b"12x", b"99999999999999999999999", b"7/C", b"8/", b"0/B", b"//B"]
TIDS = [-1, 0, 1, 2, 65534, 65535, 65536, 70000, 2 ** 31 - 1]
POS = [-1, 0, 1, 99, 100, 101, 5000, 2 ** 31 - 1, -5]


def _cigar(rng):
    ops = []
    if rng.random() < 0.3:
        ops.append("%dH" % rng.integers(1, 6))
    if rng.random() < 0.4:
        ops.append("%dS" % rng.integers(1, 8))
    for _ in range(int(rng.integers(1, 4))):
        ops.append("%d%s" % (rng.integers(1, 30), "MMMIDN=X"[int(rng.integers(0, 8))]))
    if rng.random() < 0.4:
        ops.append("%dS" % rng.integers(1, 8))
    if rng.random() < 0.3:
        ops.append("%dH" % rng.integers(1, 6))
    return "".join(ops)


def _aux(rng, cell_values):
    out = b""
    for _ in range(int(rng.integers(0, 7))):
        k = int(rng.integers(0, 9))
        if k == 0:
            out += b"MCZ" + MC_VALUES[int(rng.integers(0, len(MC_VALUES)))] + b"\0"
        elif k == 1:
            out += b"MCZ" + _cigar(rng).encode() + b"\0"
        elif k == 2:
            out += b"MIZ" + MI_Z[int(rng.integers(0, len(MI_Z)))] + b"\0"
        elif k == 3:
            t = "cCsSiI"[int(rng.integers(0, 6))]
            lo, hi = {"c": (-128, 127), "C": (0, 255), "s": (-32768, 32767), "S": (0, 65535),
                      "i": (-2 ** 31, 2 ** 31 - 1), "I": (0, 2 ** 32 - 1)}[t]
            v = int(rng.integers(lo, hi, endpoint=True))
            out += b"MI" + t.encode() + struct.pack({"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i",
                                                     "I": "<I"}[t], v)
        elif k == 4:
            out += b"RGZ" + [b"A", b"B", b"C", b"D", b"E", b"ZZ", b""][int(rng.integers(0, 7))] + b"\0"
        elif k == 5:
            out += b"CBZ" + cell_values[int(rng.integers(0, len(cell_values)))] + b"\0"
        elif k == 6:
            out += b"XXi" + struct.pack("<i", int(rng.integers(0, 1000)))
        elif k == 7:
            n = int(rng.integers(0, 4))
            out += b"ZBBs" + struct.pack("<I", n) + struct.pack("<%dh" % n, *range(n))
        else:
            out += [b"MIf" + struct.pack("<f", 1.5), b"QQ?xyz", b"MIA7", b"ZZZtrunc"][int(rng.integers(0, 4))]
    return out


def random_records(n: int, seed: int, n_names: int = 0):
    """n records (no block_size prefix).  Names come from a pool of n_names (0: about n / 2), so templates share
    names and planted exact duplicates test stability."""
    rng = np.random.default_rng(seed)
    names = [b"q%d" % i + b"x" * int(rng.integers(0, 12)) for i in range(n_names or max(1, n // 2))]
    cells = [b"AAAA", b"CCGT", b"", b"TTTTTTTT", b"\xff"]
    recs = []
    while len(recs) < n:
        if recs and rng.random() < 0.05:             # an exact duplicate of an earlier record
            recs.append(recs[int(rng.integers(0, len(recs)))])
            continue
        flag = 0
        for bit, p in ((0x1, 0.8), (0x4, 0.15), (0x8, 0.15), (0x10, 0.4), (0x20, 0.4), (0x40, 0.5), (0x80, 0.5),
                       (0x100, 0.05), (0x800, 0.05)):
            if rng.random() < p:
                flag |= bit
        tid = TIDS[int(rng.integers(0, len(TIDS)))] if rng.random() < 0.3 else int(rng.integers(0, 3))
        pos = POS[int(rng.integers(0, len(POS)))] if rng.random() < 0.3 else int(rng.integers(0, 400))
        mtid = TIDS[int(rng.integers(0, len(TIDS)))] if rng.random() < 0.2 else int(rng.integers(0, 3))
        mpos = POS[int(rng.integers(0, len(POS)))] if rng.random() < 0.2 else int(rng.integers(0, 400))
        seq_len = int(rng.integers(0, 12))
        seq = bytes(b"ACGT"[int(x)] for x in rng.integers(0, 4, size=seq_len))
        cig = "" if rng.random() < 0.1 else _cigar(rng)
        r = make_record(name=names[int(rng.integers(0, len(names)))], flags=flag, ref_id=tid, pos=pos,
                        cigar=cig if cig else [], mate_ref_id=mtid, mate_pos=mpos, seq=seq)
        r = bytearray(r + _aux(rng, cells))
        u = rng.random()
        if u < 0.03 and len(r) > 34:                  # aux or fields cut short
            r = r[:int(rng.integers(32, len(r)))]
        elif u < 0.05:                                # a read name that runs past the record
            r[8] = 255
        elif u < 0.07:                                # a CIGAR that runs past the record
            struct.pack_into("<H", r, 12, 60000)
        elif u < 0.08:                                # l_seq past the record: no aux block
            struct.pack_into("<I", r, 16, 10 ** 6)
        recs.append(bytes(r))
    return recs


def pack(recs):
    """(bodies uint8[...], rec_off uint64[n + 1])"""
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in recs]) if recs else []
    return np.frombuffer(b"".join(recs) or b"\0", np.uint8)[:int(off[-1])].copy(), off
