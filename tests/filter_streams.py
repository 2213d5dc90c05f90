"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Seeded inputs of the record filter (fgb_filter_records / tests/filter_oracle.py): a genome with lower-case stretches
and IUPAC codes written as FASTA, and mapped simplex / duplex consensus records on both strands with mixed CIGARs
(M = X I D N S H P, clips at both ends, pure insertions), read bases = and N, NM of every integer type or absent, MD
of the same or another length or absent, UQ absent, unmapped records with and without the tags, ref_id -1 without
0x4, secondary and supplementary records, templates without a primary and R2-before-R1 pairs."""
from __future__ import annotations

import os
import random
import struct
import sys
from typing import List, Tuple

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.bam_builder import make_record   # noqa: E402

IUPAC = b"RYSWKMBDHVN"


def genome(seed: int, n_contigs: int = 3, length: int = 4000) -> List[Tuple[bytes, bytes]]:
    rng = random.Random(seed)
    out = []
    for c in range(n_contigs):
        s = bytearray(rng.choice(b"ACGT") for _ in range(length))
        for _ in range(length // 200):   # lower-case runs and IUPAC codes
            a = rng.randrange(length - 20)
            s[a:a + 10] = s[a:a + 10].lower()
            s[rng.randrange(length)] = rng.choice(IUPAC)
        out.append((b"chr%d" % (c + 1), bytes(s)))
    out.append((b"empty", b""))
    return out


def fasta(contigs, width: int = 60, crlf: bool = False) -> bytes:
    nl = b"\r\n" if crlf else b"\n"
    out = bytearray()
    for name, seq in contigs:
        out += b">" + name + b" some description" + nl
        for i in range(0, len(seq), width):
            out += seq[i:i + width] + nl
    return bytes(out)


def header(contigs, extra: Tuple[bytes, ...] = ()) -> bytes:
    lines = [b"@HD\tVN:1.6\tSO:unsorted"] + [b"@SQ\tSN:%s\tLN:%d" % (n, max(len(s), 1)) for n, s in contigs]
    lines += [b"@SQ\tSN:%s\tLN:1000" % e for e in extra]
    return b"\n".join(lines) + b"\n"


def _cigar(rng, length):
    """(cigar string, read length consumed, reference span)"""
    kind = rng.randrange(8)
    if kind == 0:
        return "%dM" % length, length, length
    if kind == 1:
        return "%dI" % length, length, 0   # a pure insertion: no reference span
    parts, q, ref = [], 0, 0
    if rng.random() < 0.4:
        parts.append("%dH" % rng.randint(1, 5))
    if rng.random() < 0.5:
        s = rng.randint(1, 10)
        parts.append("%dS" % s)
        q += s
    while q < length - 12:
        op = rng.choice("MMM=XIDNP")
        n = rng.randint(1, min(30, length - q - 10))
        if op in "M=X":
            parts.append("%d%s" % (n, op)); q += n; ref += n
        elif op == "I":
            parts.append("%dI" % n); q += n
        elif op in "DN":
            parts.append("%d%s" % (n, op)); ref += n
        else:
            parts.append("%dP" % n)
    tail = length - q
    if rng.random() < 0.5 and tail > 2:
        parts.append("%dM" % (tail - 2)); parts.append("2S"); ref += tail - 2
    else:
        parts.append("%dM" % tail); ref += tail
    if rng.random() < 0.3:
        parts.append("%dH" % rng.randint(1, 5))
    return "".join(parts), length, ref


def _read(rng, contig: bytes, pos: int, cigar: str, length: int) -> bytearray:
    """bases from the reference along the CIGAR with ~3 % changed, some '=' and N"""
    seq, ro, num = bytearray(), pos, ""
    for ch in cigar:
        if ch.isdigit():
            num += ch
            continue
        n = int(num); num = ""
        if ch in "M=X":
            seq += contig[ro:ro + n].upper(); ro += n
        elif ch in "IS":
            seq += bytes(rng.choice(b"ACGT") for _ in range(n))
        elif ch in "DN":
            ro += n
    for i in range(len(seq)):
        r = rng.random()
        if seq[i] not in b"ACGT" or r < 0.03:
            seq[i] = rng.choice(b"ACGT")
        elif r < 0.04:
            seq[i] = ord("N")
        elif r < 0.045:
            seq[i] = ord("=")
    return seq[:length]


def consensus_tags(rng, length: int, duplex: bool, reverse_extra: bool):
    tags = []
    if duplex:
        ad = [rng.randint(0, 6) for _ in range(length)]
        bd = [rng.randint(0, 6) for _ in range(length)]
        tags += [(b"aD", "C", max(ad)), (b"bD", "C", max(bd)), (b"cD", "C", max(ad) + max(bd)),
                 (b"aE", "f", rng.random() * 0.05), (b"bE", "f", rng.random() * 0.05), (b"cE", "f", rng.random() * 0.05),
                 (b"ad", "Bs", ad), (b"bd", "Bs", bd), (b"ae", "Bs", [rng.randint(0, min(1, x)) for x in ad]),
                 (b"be", "Bs", [rng.randint(0, min(1, x)) for x in bd])]
        tags += [(b"ac", "Z", bytes(rng.choice(b"ACGTacgtN") for _ in range(length))),
                 (b"bc", "Z", bytes(rng.choice(b"ACGTN") for _ in range(length)))]
    else:
        cd = [rng.randint(0, 8) for _ in range(length)]
        tags += [(b"cD", "C", max(cd)), (b"cM", "C", min(cd)), (b"cE", "f", rng.random() * 0.04),
                 (b"cd", "Bs", cd), (b"ce", "Bs", [rng.randint(0, min(2, x)) for x in cd])]
    if reverse_extra:
        tags.append((b"aq", "Z", bytes(rng.randint(35, 70) for _ in range(length))))
    return tags


def _nm_md(rng, tags):
    k = rng.randrange(8)
    if k < 6:
        typ = "cCsSiI"[k]
        tags.append((b"NM", typ, rng.randint(0, 100)))
    m = rng.randrange(3)
    if m == 1:
        tags.append((b"MD", "Z", b"1A0"))
    elif m == 2:
        tags.append((b"MD", "Z", b"%d" % rng.randint(0, 150)))
    if rng.random() < 0.3:
        tags.append((b"UQ", "i", rng.randint(0, 500)))
    rng.shuffle(tags)
    return tags


def records(seed: int, contigs, n_templates: int = 300, length: int = 150, long_every: int = 0,
            long_length: int = 65535) -> List[bytes]:
    """Templates of one to five records in input order: pairs (sometimes R2 first), fragments, secondary and
    supplementary records, unmapped and ref_id -1 records, templates without a primary."""
    rng = random.Random(seed)
    usable = [(i, s) for i, (_, s) in enumerate(contigs) if len(s) > 0]
    out = []
    for t in range(n_templates):
        name = b"q%06d" % t
        shape = rng.randrange(10)
        kinds = ["R1", "R2"] if shape < 6 else ["F"]
        if shape == 6:
            kinds = ["R1", "R2", "SUPP"]
        elif shape == 7:
            kinds = ["R2", "R1", "SEC", "SEC"]
        elif shape == 8:
            kinds = ["SUPP", "SEC"]   # no primary record
        duplex = rng.random() < 0.5
        for kind in kinds:
            L = long_length if long_every and t % long_every == 0 and kind != "SEC" else length
            ci, contig = rng.choice(usable)
            cigar, _, span = _cigar(rng, L)
            if span >= len(contig):
                cigar, span = "%dI" % L, 0
            pos = rng.randrange(0, len(contig) - span) if span else rng.randrange(len(contig))
            flags = {"R1": 0x41, "R2": 0x81, "F": 0, "SUPP": 0x800 | 0x41, "SEC": 0x100 | 0x81}[kind]
            if rng.random() < 0.5:
                flags |= 0x10
            ref_id = ci
            u = rng.random()
            if u < 0.06:   # unmapped, with or without the tags
                flags |= 0x4
                if rng.random() < 0.5:
                    ref_id = -1
            elif u < 0.09:   # ref_id -1 without 0x4
                ref_id = -1
            seq = _read(rng, contig, pos, cigar, L)
            quals = bytes(rng.randint(2, 45) for _ in range(L))
            tags = _nm_md(rng, consensus_tags(rng, L, duplex, rng.random() < 0.3))
            out.append(bytes(make_record(name=name, flags=flags, ref_id=ref_id, pos=pos, cigar=cigar, seq=bytes(seq),
                                         quals=quals, tags=tags)))
    return out


def pack(recs) -> Tuple["np.ndarray", "np.ndarray"]:
    import numpy as np
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in recs])
    return np.frombuffer(b"".join(recs) or b"\0", np.uint8).copy(), off
