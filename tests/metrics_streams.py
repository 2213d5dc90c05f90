"""Test helper: UMI-grouped paired-end streams for the metrics collector, as `fgumi group` writes them (consecutive
templates of one coordinate group, MI and RX on every record)."""
from __future__ import annotations

import numpy as np

from tests.bam_builder import make_record

HEADER = b"@HD\tVN:1.6\tSO:unsorted\tGO:query\n@SQ\tSN:chr1\tLN:248956422\n@SQ\tSN:chr2\tLN:242193529\n"
PAIRED, PROPER, REV, MREV, FIRST, LAST, SECONDARY, SUPP = 0x1, 0x2, 0x10, 0x20, 0x40, 0x80, 0x100, 0x800


def pair(name: bytes, mi, rx, ref1=0, pos1=100, ref2=None, pos2=300, cigar="20M", r1_tags=None, extra=()):
    """R1 forward at (ref1, pos1), R2 reverse at (ref2, pos2); 1-based positions.  mi / rx None: no tag.  r1_tags
    replaces R1's tags when given."""
    ref2 = ref1 if ref2 is None else ref2
    tags = [(b"RX", "Z", rx)] if rx is not None else []
    if mi is not None:
        tags.append((b"MI", "Z", mi))
    seq = b"A" * 20
    r1 = make_record(name, PAIRED | FIRST | MREV, ref1, pos1 - 1, cigar=cigar, mate_ref_id=ref2, mate_pos=pos2 - 1,
                     seq=seq, tags=tags if r1_tags is None else r1_tags)
    r2 = make_record(name, PAIRED | LAST | REV, ref2, pos2 - 1, cigar=cigar, mate_ref_id=ref1, mate_pos=pos1 - 1,
                     seq=seq, tags=tags)
    return [r1, r2] + list(extra)


def to_arrays(records):
    off = np.zeros(len(records) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in records])
    return np.frombuffer(b"".join(records) or b"\0", np.uint8).copy(), off


def random_stream(seed: int, n_groups: int, max_families: int = 4, max_size: int = 6, suffix_rate: float = 0.9,
                  odd_mi_rate: float = 0.0, umi_len: int = 6, umi_error: float = 0.05, big_family: int = 0):
    """Coordinate groups of random families: /A and /B templates of base MI numbers (or, at odd_mi_rate, odd MIs --
    no suffix, leading zeros, letters), RX "X-Y" swapped on /B with base substitutions.  big_family > 0 adds one
    group with a family of that many templates on each strand."""
    rng = np.random.default_rng(seed)
    recs, mi_num, t = [], 0, 0
    bases = np.array(list(b"ACGT"), np.uint8)

    def umi():
        return bytes(rng.choice(bases, umi_len))

    def noisy(u):
        b = bytearray(u)
        for i in range(len(b)):
            if rng.random() < umi_error:
                b[i] = int(rng.choice(bases))
        return bytes(b)

    sizes = []
    for g in range(n_groups):
        sizes.append([(int(rng.integers(0, max_size + 1)), int(rng.integers(0, max_size + 1)))
                      for _ in range(int(rng.integers(1, max_families + 1)))])
    if big_family:
        sizes.append([(big_family, big_family - 3), (40, 1)])
    for g, fams in enumerate(sizes):
        ref, pos = g % 2, 1000 + 500 * g
        tpls = []
        for a, b in fams:
            mi_num += 1
            x, y = umi(), umi()
            odd = rng.random() < odd_mi_rate
            kind = int(rng.integers(0, 3)) if odd else 0
            base = [b"%d" % mi_num, b"0%d" % mi_num, b"m%d" % mi_num][kind]
            for strand, n in ((b"A", a), (b"B", b)):
                for _ in range(n):
                    if rng.random() >= suffix_rate:
                        mi = base
                    else:
                        mi = base + b"/" + strand
                    rx = noisy(x) + b"-" + noisy(y) if strand == b"A" else noisy(y) + b"-" + noisy(x)
                    tpls.append((mi, rx))
        order = rng.permutation(len(tpls))
        for k in order:
            t += 1
            mi, rx = tpls[k]
            recs += pair(b"q%07d" % t, mi, rx, ref1=ref, pos1=pos, pos2=pos + 200)
    return recs
