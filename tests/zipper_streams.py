"""Seeded unmapped / mapped stream pairs for the zipper tests: paired and unpaired templates, supplementary and
secondary records, one or both mates unmapped, both strands, templates missing from the mapped side, consensus
per-base tags, pre-existing MQ / MC / ms / AS / XS / tc of every integer type, and tags the unmapped read replaces."""
import random

from tests.bam_builder import make_record

INT_TYPES = ("c", "C", "s", "S", "i", "I")
INT_RANGE = {"c": (-128, 127), "C": (0, 255), "s": (-32768, 32767), "S": (0, 65535), "i": (-2 ** 31, 2 ** 31 - 1),
             "I": (0, 2 ** 32 - 1)}


def _int_tag(rng, tag):
    t = rng.choice(INT_TYPES)
    lo, hi = INT_RANGE[t]
    return (tag, t, rng.choice([lo, hi, 0, rng.randint(lo, hi)]))


def _cigar(rng, L, long_cigar):
    if long_cigar:
        ops = []
        left = L
        while left > 1:
            k = rng.randint(1, min(3, left - 1))
            ops.append("%dM%dI" % (k, 1) if rng.random() < 0.5 else "%dM%dD" % (k, rng.randint(1, 500)))
            left -= k + (1 if ops[-1].endswith("I") else 0)
        return "".join(ops) + "%dM" % max(left, 1)
    return rng.choice(["%dM" % L, "5S%dM" % (L - 5), "%dM3S" % (L - 3), "10H%dM" % L, "%dM2I%dM" % (L // 2, L - L // 2 - 2),
                       "%dM4D%dM" % (L // 2, L - L // 2)])


def _seq(rng, L):
    return bytes(rng.choice(b"ACGTN") for _ in range(L))


def _consensus_tags(rng, L):
    return [(b"cd", "Bs", [rng.randint(0, 30) for _ in range(L)]), (b"ce", "Bs", [rng.randint(0, 3) for _ in range(L)]),
            (b"ad", "Bs", [rng.randint(0, 30) for _ in range(L)]), (b"aD", "Z", _seq(rng, L)),
            (b"bD", "Z", _seq(rng, L).lower()), (b"cD", "Z", _seq(rng, L)), (b"ae", "BC", [rng.randint(0, 3) for _ in range(L)])]


def streams(seed, n_templates=200, L=40, missing=0.1, consensus=False, long_cigar=False, odd_mc=True):
    """(unmapped records, mapped records) in the same name order.  odd_mc: some mapped MC entries are not Z strings
    (an aligner writes Z; `group` downstream refuses any other type)."""
    rng = random.Random(seed)
    um, mp = [], []
    for t in range(n_templates):
        name = b"q%07d" % t
        paired = rng.random() < 0.85
        segs = [0x41, 0x81] if paired else [0]
        urec = []
        for f in segs:
            tags = [(b"RX", "Z", _seq(rng, 8)), (b"QX", "Z", b"IIIIIIII")]
            if rng.random() < 0.3:
                tags.append(_int_tag(rng, b"AS"))
            if rng.random() < 0.2:
                tags.append((b"PG", "Z", b"extract"))
            if rng.random() < 0.2:
                tags.append((b"xy", "i", rng.randint(-5, 5)))
            if rng.random() < 0.15:
                tags.append((b"tc", "Z", b"pre"))
            if rng.random() < 0.15:
                tags.append(_int_tag(rng, b"ms"))
            if consensus:
                tags += _consensus_tags(rng, L)
            rng.shuffle(tags)
            uf = (f | 0x4 | (0x8 if paired else 0)) | (0x200 if rng.random() < 0.1 else 0)
            urec.append(make_record(name=name, flags=uf, ref_id=-1, pos=-1, mapq=0, cigar=[], seq=_seq(rng, L),
                                    tags=tags))
        um += urec
        if rng.random() < missing:
            continue
        recs = []
        for k, f in enumerate(segs):
            unm = rng.random() < 0.12
            rev = rng.random() < 0.5
            cig = _cigar(rng, L, long_cigar)
            tags = []
            for tg in (b"MQ", b"MC", b"ms", b"AS", b"XS", b"tc", b"RX", b"PG", b"NM"):
                if rng.random() < 0.35:
                    if tg == b"MC":   # Z of the mate's text length or another, or a non-Z entry kept in place at 3 bytes
                        t = rng.choice(["Z", "Z", "i", "C", "A"] if odd_mc else ["Z"])
                        tags.append((tg, t, b"%dM" % rng.choice([L, 7, 100]) if t == "Z" else
                                     rng.randint(0, 9) if t == "C" else b"x" if t == "A" else rng.randint(-5, 5)))
                    elif tg in (b"RX", b"PG", b"tc"):
                        tags.append((tg, "Z", b"bwa" if tg == b"PG" else b"OLD"))
                    else:
                        tags.append(_int_tag(rng, tg))
            rng.shuffle(tags)
            ff = f | (0x4 if unm else 0) | (0x10 if rev else 0)
            pos = rng.randint(0, 5000)
            recs.append(make_record(name=name, flags=ff, ref_id=-1 if unm else rng.randint(0, 2), pos=-1 if unm else pos,
                                    mapq=rng.choice([0, 60, 255, 200]), cigar=[] if unm else cig, seq=_seq(rng, L),
                                    tlen=rng.randint(-500, 500), tags=tags))
            for extra in range(rng.choice([0, 0, 1, 2])):
                ef = f | (0x800 if rng.random() < 0.6 else 0x100) | (0x10 if rng.random() < 0.5 else 0)
                recs.append(make_record(name=name, flags=ef, ref_id=rng.randint(0, 2), pos=rng.randint(0, 5000),
                                        mapq=rng.randint(0, 60), cigar=_cigar(rng, L, False), seq=_seq(rng, L),
                                        tags=[_int_tag(rng, b"AS")] if rng.random() < 0.5 else []))
        rng.shuffle(recs)
        mp += recs
    return um, mp
