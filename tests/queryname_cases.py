"""Seeded read names and records for the queryname sort tests: the name styles users sort (Illumina, SRR, `read%d`),
runs of zeros, digit runs longer than a u64, names of 254 bytes, and bytes the comparators treat apart (NUL, 0xff,
digits next to '/' and ':')."""
import numpy as np

from tests.bam_builder import make_record

ALPHABET = b"019a/:\x00\xff"
# flags of one template's records: R1, R2, R1 secondary (twice: equal keys), R1 supplementary, R2 secondary
TEMPLATE_FLAGS = (0x1 | 0x40, 0x1 | 0x80, 0x1 | 0x40 | 0x100, 0x1 | 0x40 | 0x100, 0x1 | 0x40 | 0x800,
                  0x1 | 0x80 | 0x100)


def _digits(rng, k: int) -> bytes:
    return bytes(int(c) for c in rng.integers(0x30, 0x3A, k))


def random_name(rng) -> bytes:
    style = int(rng.integers(0, 9))
    if style == 0:
        return b"A00123:8:HJKLMDSXY:%d:%d:%d:%d" % (rng.integers(1, 5), rng.integers(1101, 2679),
                                                   rng.integers(1000, 32001), rng.integers(1000, 40001))
    if style == 1:
        return b"SRR%06d.%d" % (rng.integers(0, 1000), rng.integers(0, 10 ** int(rng.integers(1, 8))))
    if style == 2:
        return b"read%d" % rng.integers(0, 3000)
    if style == 3:                                       # runs of zeros, alone and before digits
        return b"r" + b"0" * int(rng.integers(0, 6)) + (b"%d" % rng.integers(0, 30) if rng.random() < 0.7 else b"") + \
            [b"", b"x", b"/1", b":00"][int(rng.integers(0, 4))]
    if style == 4:                                       # digit runs past u64, some with leading zeros
        return b"x" + b"0" * int(rng.integers(0, 3)) + _digits(rng, int(rng.integers(19, 60))) + \
            [b"", b"y", b"7"][int(rng.integers(0, 3))]
    if style == 5:                                       # the longest name a record holds
        return bytes(int(c) for c in rng.choice(np.frombuffer(b"0123456789ab:", np.uint8), 254))
    if style == 6:
        return bytes(int(c) for c in rng.choice(np.frombuffer(ALPHABET, np.uint8), int(rng.integers(0, 13))))
    if style == 7:                                       # a shared prefix, then a short varying tail
        return b"mol%d_read%04d" % (rng.integers(0, 20), rng.integers(0, 30))
    return bytes(int(c) for c in rng.integers(1, 256, int(rng.integers(0, 40))))


def random_names(n: int, seed: int):
    rng = np.random.default_rng(seed)
    return [random_name(rng) for _ in range(n)]


def name_records(names, seed: int, per_name: int = len(TEMPLATE_FLAGS)):
    """Records of every name in `names` with the first `per_name` TEMPLATE_FLAGS, shuffled.  Each record carries its
    index in TLEN, which no key reads, so that every record is byte-unique and an unstable tie changes the output."""
    recs = [(nm, f) for nm in names for f in TEMPLATE_FLAGS[:per_name]]
    order = np.random.default_rng(seed).permutation(len(recs))
    return [make_record(name=recs[j][0], flags=recs[j][1], ref_id=-1, pos=-1, tlen=i, seq=b"ACGT")
            for i, j in enumerate(order)]
