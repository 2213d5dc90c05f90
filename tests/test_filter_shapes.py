"""The record filter's tag lookup and MD walk on hand-built records, without a GPU.

- The reference's lookup rules (crates/fgumi-raw-bam/src/tags.rs) as known answers, through the oracle
  (tests/filter_oracle.py over oracle/record_oracle.py) and through the host filter fgb_filter_record, which shares
  its lookup with the device filter: a repeated per-base or per-read tag is read from its first entry
  (find_tag_position, tags.rs:13-34), and a record is duplex when an aD / bD entry is found by name before its value
  is sized (find_tag_type, tags.rs:56-59, in is_duplex_consensus, crates/fgumi-consensus/src/filter.rs:443-446).
- NM / UQ / MD of deterministic records written as literals, so that the oracle the device is compared with
  (tests/test_filter_shapes_gpu.py) is pinned: match runs of one to five digits carried across ops and 32-base
  chunks, mismatches at chunk edges, fully mismatching ops, deletions of every placement and length, IUPAC and
  lower-case reference bases, zero and many CIGAR ops, odd and even read lengths, and reads ending on a contig's
  last base."""
import ctypes as C
import os
import struct
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import filter_oracle as O      # noqa: E402
from tests.bam_builder import cigar_from_string, make_record   # noqa: E402

R = O.R

# ---- the hand-built reference ----------------------------------------------------------------------------------
# chrA repeats a 7-base period, so its bases are easy to read off (base i is PERIOD[i % 7]) while a reference window
# misplaced by any multiple of 32 bases still shows; chrB holds lower case, IUPAC codes and N; chrC is the last
# contig of the genome array.
PERIOD = b"ACGTGCA"
CHR_A = PERIOD * 25000
CHR_B = b"ACGTacgtRYSWKMBDHVNnrn"
CHR_C = b"GATTACA" * 10
CONTIGS = [(b"chrA", CHR_A), (b"chrB", CHR_B), (b"chrC", CHR_C)]
GENOME = dict(CONTIGS)
SQ = [n for n, _ in CONTIGS]
HEADER = b"@HD\tVN:1.6\n" + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n, len(s)) for n, s in CONTIGS)
SWAP = {ord("A"): ord("C"), ord("C"): ord("A"), ord("G"): ord("T"), ord("T"): ord("G")}

# no masking and every gate open: the records come out with only their alignment tags edited
OPEN = dict(min_reads=(0,), max_read_error_rate=(1.0,), max_base_error_rate=(1.0,), max_no_call_fraction=1e9)


def along(ctg: bytes, pos: int, cigar: str, mis=()) -> bytes:
    """The read that matches `ctg` from `pos` along `cigar` (inserted and soft-clipped bases T), with the read bases
    at positions `mis` swapped for another base."""
    seq, ro = bytearray(), pos
    for op in cigar_from_string(cigar):
        t, n = op & 0xF, op >> 4
        if t in (0, 7, 8):
            seq += ctg[ro:ro + n].upper()
            ro += n
        elif t in (1, 4):
            seq += b"T" * n
        elif t in (2, 3):
            ro += n
    for i in mis:
        seq[i] = SWAP.get(seq[i], ord("A"))
    return bytes(seq)


def _runs():
    """Match runs of 1 to 5 digits as one op, split across I, N, P and = / X boundaries, and ended by a mismatch."""
    out = []
    for n in (9, 10, 31, 32, 33, 99, 100, 999, 1000, 9999, 10000, 65535):
        a = n // 2
        md = b"%d" % n
        out += [("run%d" % n, 0, 3, "%dM" % n, (), 0, 0, md),
                ("run%d_M_I_M" % n, 0, 3, "%dM2I%dM" % (a, n - a), (), 2, 0, md),
                ("run%d_M_N_M" % n, 0, 3, "%dM5N%dM" % (a, n - a), (), 0, 0, md),
                ("run%d_M_P_M" % n, 0, 3, "%dM3P%dM" % (a, n - a), (), 0, 0, md),
                ("run%d_eq_X_eq" % n, 0, 3, "%d=1X%d=" % (a, n - a - 1), (), 0, 0, md),
                # the run ends in a mismatch: its digits are written at the mismatch, not at the end
                ("run%d_then_mismatch" % n, 0, 3, "%dM" % (n + 1), (n,), 1, 30,
                 b"%d%c0" % (n, PERIOD[(3 + n) % 7]))]
    return out


# (id, contig, pos, cigar, mismatching read positions or the read itself, NM, UQ, MD); qualities 30
MD_CASES = _runs() + [
    ("mismatch_at_0", 0, 0, "100M", (0,), 1, 30, b"0A99"),
    ("mismatch_at_31", 0, 0, "100M", (31,), 1, 30, b"31T68"),
    ("mismatch_at_32", 0, 0, "100M", (32,), 1, 30, b"32G67"),
    ("mismatch_at_63", 0, 0, "100M", (63,), 1, 30, b"63A36"),
    ("mismatch_at_64", 0, 0, "100M", (64,), 1, 30, b"64C35"),
    ("mismatches_at_chunk_edges", 0, 0, "100M", (0, 31, 32, 63, 64), 5, 150, b"0A30T0G30A0C35"),
    ("all_mismatch_32", 0, 0, "32M", tuple(range(32)), 32, 960,
     b"0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0"),
    ("all_mismatch_33", 0, 0, "33M", tuple(range(33)), 33, 990,
     b"0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0"),
    ("all_mismatch_65", 0, 0, "65M", tuple(range(65)), 65, 1950,
     b"0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A"
     b"0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0"),
    ("all_mismatch_32_X_after_run", 0, 0, "5M32X4M", tuple(range(5, 37)), 32, 960,
     b"5C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C4"),
    ("all_mismatch_33_X_after_run", 0, 0, "5M33X4M", tuple(range(5, 38)), 33, 990,
     b"5C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G4"),
    ("all_mismatch_65_X_after_run", 0, 0, "5M65X4M", tuple(range(5, 70)), 65, 1950,
     b"5C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C"
     b"0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A0A0C0G0T0G0C0A4"),
    ("alternating", 0, 0, "70M", tuple(range(0, 70, 2)), 35, 1050,
     b"0A1G1G1A1C1T1C1A1G1G1A1C1T1C1A1G1G1A1C1T1C1A1G1G1A1C1T1C1A1G1G1A1C1T1C1"),
    ("deletion_first", 0, 7, "3D10M", (), 3, 0, b"0^ACG10"),
    ("deletion_last", 0, 7, "10M3D", (), 3, 0, b"10^TGC0"),
    ("deletion_middle", 0, 7, "5M3D5M", (), 3, 0, b"5^CAA5"),
    ("deletion_before_mismatch", 0, 7, "5M2D5M", (5,), 3, 30, b"5^CA0A4"),
    ("deletion_deletion", 0, 7, "5M2D3D5M", (), 5, 0, b"5^CA0^ACG5"),
    ("deletion_insertion_deletion", 0, 7, "5M2D2I3D5M", (), 7, 0, b"5^CA0^ACG5"),
    ("deletion_skip_deletion", 0, 7, "5M2D4N3D5M", (), 5, 0, b"5^CA0^GCA5"),
    ("deletion31", 0, 7, "10M31D10M", (), 31, 0, b"10^TGCAACGTGCAACGTGCAACGTGCAACGTGC10"),
    ("deletion32", 0, 7, "10M32D10M", (), 32, 0, b"10^TGCAACGTGCAACGTGCAACGTGCAACGTGCA10"),
    ("deletion33", 0, 7, "10M33D10M", (), 33, 0, b"10^TGCAACGTGCAACGTGCAACGTGCAACGTGCAA10"),
    ("deletion100000", 0, 7, "10M100000D10M", (), 100000, 0, b"10^" + CHR_A[17:100017] + b"10"),
    ("iupac_equal", 1, 8, "10M", b"RYSWKMBDHV", 0, 0, b"10"),
    ("iupac_different", 1, 8, "10M", b"YRWSMKDBVH", 10, 300, b"0R0Y0S0W0K0M0B0D0H0V0"),
    ("lower_case_reference", 1, 4, "4M", b"ACGT", 0, 0, b"4"),
    ("lower_case_iupac_reference", 1, 20, "1M", b"R", 0, 0, b"1"),
    ("reference_N_read_N", 1, 18, "2M", b"NN", 2, 60, b"0N0n0"),
    ("reference_N_read_A", 1, 18, "2M", b"AA", 2, 60, b"0N0n0"),
    ("read_equals_sign", 1, 0, "2M", b"=C", 1, 30, b"0A1"),
    ("lseq1", 0, 11, "1M", (0,), 1, 30, b"0G0"),
    ("lseq2", 0, 11, "2M", (1,), 1, 30, b"1C0"),
    ("lseq63", 0, 11, "63M", (62,), 1, 30, b"62T0"),
    ("lseq64", 0, 11, "64M", (63,), 1, 30, b"63G0"),
    ("lseq65", 0, 11, "65M", (64,), 1, 30, b"64C0"),
    ("forty_ops", 0, 2, "1M1I" * 20, (0, 38), 22, 60, b"0G18A0"),
    ("zero_cigar_ops", 0, 5, "", b"ACGTA", 0, 0, b"0"),
    ("ends_on_last_base_of_inner_contig", 0, len(CHR_A) - 20, "20M", (19,), 1, 30, b"19A0"),
    ("ends_on_last_base_of_genome", 2, len(CHR_C) - 20, "20M", (19,), 1, 30, b"19A0"),
]


def md_record(case, name=b"q", flags=0, tags=()) -> bytes:
    cid, c, pos, cigar, read = case[:5]
    seq = read if isinstance(read, bytes) else along(CONTIGS[c][1], pos, cigar, read)
    return make_record(name=name, flags=flags, ref_id=c, pos=pos, cigar=cigar, seq=seq, tags=tags)


def md_records():
    return [md_record(c, name=b"md%03d" % k) for k, c in enumerate(MD_CASES)]


@pytest.mark.parametrize("case", MD_CASES, ids=lambda c: c[0])
def test_md_walk_literals(case):
    r = bytearray(md_record(case))
    O.regenerate(r, 0, SQ, GENOME)
    t = R._aux_tags(R.Rec(bytes(r)).aux())
    assert (t[b"NM"][1], t[b"UQ"][1], t[b"MD"][1]) == case[5:]


def test_uq_sums_the_mismatching_qualities():
    quals = bytes(2 + i % 50 for i in range(100))
    r = bytearray(make_record(name=b"q", ref_id=0, pos=0, cigar="100M", quals=quals,
                              seq=along(CHR_A, 0, "100M", (0, 31, 32, 63, 64))))
    O.regenerate(r, 0, SQ, GENOME)
    t = R._aux_tags(R.Rec(bytes(r)).aux())
    assert (t[b"NM"][1], t[b"UQ"][1]) == (5, 2 + 33 + 34 + 15 + 16)


@pytest.mark.parametrize("c", [0, 2])
def test_one_base_past_the_contig_end(c):
    """The read that ends on a contig's last base, one base longer: fetch_slice fails the call."""
    ctg = CONTIGS[c][1]
    r = make_record(name=b"q", ref_id=c, pos=len(ctg) - 20, cigar="21M", seq=ctg[-20:].upper() + b"A")
    with pytest.raises(O.FilterError, match="exceeds"):
        O.filter_records([r], HEADER, O.Config(**OPEN), GENOME)


# ---- the reference's tag lookup ---------------------------------------------------------------------------------
SEQ = b"ACGTACGTAC"
GOOD = [(b"cd", "Bs", [5] * 10)]
CUT_B = b"Bs" + struct.pack("<I", 100) + b"\x05\x00"         # a B:s array of 100 with one element present

# (id, aux entries, duplex, masked, passes) under LOOKUP_CFG: a simplex record with cd 5 keeps its bases, a duplex one
# without ad / bd has depth 0 everywhere and is masked whole, which its no-call fraction then rejects
LOOKUP_CASES = [
    ("cd_twice_first_deep", GOOD + [(b"cd", "Bs", [0] * 10)], False, 0, True),
    ("cd_twice_first_shallow", [(b"cd", "Bs", [0] * 10)] + GOOD, False, 10, False),
    ("cD_twice_first_low", GOOD + [(b"cD", "C", 0), (b"cD", "C", 5)], False, 0, False),
    ("cD_twice_first_high", GOOD + [(b"cD", "C", 5), (b"cD", "C", 0)], False, 0, True),
    ("ce_twice_first_clean", GOOD + [(b"ce", "BC", [0] * 10), (b"ce", "BC", [5] * 10)], False, 0, True),
    ("aD_unknown_type_last", GOOD + [(b"aD", "raw", b"Q\x05")], True, 10, False),
    ("bD_unknown_type_last", GOOD + [(b"bD", "raw", b"Q\x05")], True, 10, False),
    ("aD_B_array_cut_short", GOOD + [(b"aD", "raw", CUT_B)], True, 10, False),
    ("aD_Z_without_NUL", GOOD + [(b"aD", "raw", b"Z12")], True, 10, False),
    ("aD_after_unknown_type", GOOD + [(b"xx", "raw", b"Q\x00"), (b"aD", "C", 5)], False, 0, True),
    ("aD_after_B_unknown_element", GOOD + [(b"xx", "raw", b"Bq" + struct.pack("<I", 1) + b"\0"), (b"aD", "C", 5)],
     False, 0, True),
    ("aD_after_Z_without_NUL", GOOD + [(b"xx", "raw", b"Z12"), (b"aD", "C", 5)], False, 0, True),
    ("aD_well_formed", GOOD + [(b"aD", "C", 5)], True, 10, False),
]
LOOKUP_CFG = dict(min_reads=(1,), max_read_error_rate=(0.5,), max_base_error_rate=(0.5,), max_no_call_fraction=0.5)


def lookup_record(case, flags=0x4, ref_id=-1, pos=-1) -> bytes:
    return make_record(name=b"k_" + case[0].encode(), flags=flags, ref_id=ref_id, pos=pos,
                       cigar="" if flags & 0x4 else "10M", seq=SEQ, tags=case[1])


@pytest.mark.parametrize("case", LOOKUP_CASES, ids=lambda c: c[0])
def test_oracle_follows_the_reference_lookup(case):
    r = bytearray(lookup_record(case))
    assert R.is_duplex_consensus(R.Rec(bytes(r)).aux()) == case[2]
    masked, ok = O.process_record(r, 0, O.Config(**LOOKUP_CFG), SQ, None)
    assert (masked, ok) == case[3:]


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as g
    g.build()
    import fgumi_b200
    return fgumi_b200


@pytest.mark.parametrize("case", LOOKUP_CASES, ids=lambda c: c[0])
def test_host_filter_follows_the_reference_lookup(fg, case):
    """fgb_filter_record (host code sharing record_filter.h with the device filter): the same masks and decision,
    and the same edited bytes, as the oracle."""
    r = bytearray(lookup_record(case))
    want = bytearray(r)
    masked, ok = O.process_record(want, 0, O.Config(**LOOKUP_CFG), SQ, None)
    kw = dict(LOOKUP_CFG)
    status, got_masked = fg.DuplexConsensusFilter(**kw).apply(r)
    assert (got_masked, status == 0) == (masked, ok) == case[3:]
    assert r == want


def test_aux_tags_stops_where_the_reference_stops():
    """A fixed-size value cut short, an unknown B element type and a Z without its NUL end the walk instead of
    raising; the entries before them stay readable and the first of two entries wins."""
    head = b"cDC\x05cDC\x09"
    assert R._aux_tags(head + b"cEf\x00\x00")[b"cD"] == ("C", 5) and b"cE" not in R._aux_tags(head + b"cEf\x00\x00")
    assert set(R._aux_tags(head + b"xxBq\x01\x00\x00\x00\x00aDC\x01")) == {b"cD"}
    assert set(R._aux_tags(head + b"xxZ12")) == {b"cD"}
    assert set(R._aux_tags(head + b"xxB")) == {b"cD"}
    assert R._has_tag(head + b"aDB", b"aD") and not R._has_tag(head + b"xxB" + b"aDC\x01", b"aD")
    # A and H entries are walked over like any other
    r = make_record(name=b"q", seq=b"AC", tags=[(b"XT", "A", b"U"), (b"XH", "H", b"1AE3"), (b"aD", "C", 2)])
    aux = R.Rec(r).aux()
    assert aux == b"XTAUXHH1AE3\0aDC\x02" and R._has_tag(aux, b"aD")
    assert R._aux_tags(aux) == {b"XT": ("A", b"U"), b"XH": ("H", b"1AE3"), b"aD": ("C", 2)}
