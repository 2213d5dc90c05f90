"""Pins the Python record-level oracle (oracle/record_oracle.py) against the reference's own
known-answer unit tests for the host side of the simplex caller.  Each test names the reference test
it reproduces (fgumi 0.2.0: crates/...).  CPU only."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import record_oracle as R          # noqa: E402
from tests import oracle_lib as O              # noqa: E402
from tests.bam_builder import make_record, encode_op, parse_records   # noqa: E402
import fgumi_b200 as fg                        # noqa: E402

P, F1, F2, REV, MREV = R.PAIRED, R.FIRST_SEGMENT, R.LAST_SEGMENT, R.REVERSE, R.MATE_REVERSE


def vote_fn(rows, opt):
    batch = fg.pack_source_reads([rows], opt.min_reads)
    ob, oq, od, oe, cl = O.simplex_batch(batch, opt.error_rate_pre_umi, opt.error_rate_post_umi,
                                         opt.min_reads, opt.min_consensus_base_quality)
    n = int(cl[0])
    return bytes(ob[:n]), bytes(oq[:n]), list(od[:n]), list(oe[:n])


def make_caller(**kw):
    opt = R.VanillaOptions(**kw)
    return R.VanillaCallerOracle("consensus", "A", opt, vote_fn, O.builder_call)


def frag(name, bases, quals, umi=b"UMI1", **kw):   # create_consensus_test_read, vanilla_caller.rs:2067
    return make_record(name=name, ref_id=0, pos=99, seq=bases, quals=quals,
                       tags=[(b"MI", "Z", umi)], **kw)


# ---- find_quality_trim_point, vanilla_caller.rs:1607-1708 ----
def test_find_quality_trim_point():
    f = R.find_quality_trim_point
    assert f([30] * 5 + [2] * 5, 15) == 5
    assert f([30] * 10, 15) == 10
    assert f([12] * 10, 15) == 0
    assert f([12] * 10, 11) == 10 and f([12] * 10, 12) == 10 and f([12] * 10, 13) == 0
    assert f([30, 30, 30, 2, 5, 2, 3, 20, 2, 6], 15) == 3
    assert f([30, 2] * 5, 15) == 9
    assert f([], 15) == 0 and f([30, 30, 30], 0) == 0


# ---- simplify / prefix, vanilla_caller.rs:1892-2030 ----
def test_simplify_and_prefix():
    M, I, D, S = 0, 1, 2, 4
    assert R.simplify_cigar([encode_op(0, 50)]) == [(M, 50)]
    assert R.simplify_cigar([encode_op(S, 5), encode_op(0, 40), encode_op(S, 5)]) == [(M, 50)]
    assert R.simplify_cigar([encode_op(0, 10), encode_op(I, 2), encode_op(0, 10), encode_op(D, 3),
                             encode_op(0, 5)]) == [(M, 10), (I, 2), (M, 10), (D, 3), (M, 5)]
    assert R.simplify_cigar([encode_op(5, 3), encode_op(S, 2), encode_op(7, 10), encode_op(8, 1),
                             encode_op(0, 4)]) == [(M, 20)]
    assert R.is_cigar_prefix([(M, 50)], [(M, 50)])
    assert R.is_cigar_prefix([(M, 10)], [(M, 20)])
    assert not R.is_cigar_prefix([(M, 20)], [(M, 10)])
    assert not R.is_cigar_prefix([(M, 10), (I, 1)], [(M, 10), (D, 1)])
    assert R.is_cigar_prefix([(M, 10), (D, 2), (M, 5)], [(M, 10), (D, 2), (M, 20)])
    assert not R.is_cigar_prefix([(M, 9), (D, 2), (M, 5)], [(M, 10), (D, 2), (M, 20)])


# ---- create_source_read, vanilla_caller.rs:2861-3450 ----
def sr_of(rec, **opt):
    r = R.Rec(rec)
    return R.create_source_read(r, 0, R.num_bases_extending_past_mate(r), R.VanillaOptions(**opt)), R.num_bases_extending_past_mate(r)


def test_source_read_masks_and_trims():
    sr, _ = sr_of(make_record(seq=b"A" * 10, quals=[2, 30, 19, 21, 18, 20, 0, 30, 2, 30]), min_input_base_quality=20)
    assert bytes(sr.bases) == b"NANANANANA" and list(sr.quals) == [2, 30, 2, 21, 2, 20, 2, 30, 2, 30]   # :2861
    sr, _ = sr_of(make_record(seq=b"A" * 10, quals=[30] * 6 + [2] * 4), min_input_base_quality=20)
    assert bytes(sr.bases) == b"AAAAAA" and list(sr.quals) == [30] * 6                                  # :2898
    sr, _ = sr_of(make_record(seq=b"AAAAAANNNN"), min_input_base_quality=20)
    assert bytes(sr.bases) == b"AAAAAA"                                                                  # :2928
    sr, _ = sr_of(make_record(seq=b"NNNNAAAAAA", flags=REV), min_input_base_quality=20)
    assert bytes(sr.bases) == b"TTTTTT"                                                                  # :2959
    sr, _ = sr_of(make_record(seq=b"A" * 10, quals=[5] * 10), min_input_base_quality=20)
    assert sr is None                                                                                    # :2995


def test_mate_overlap_clips():
    r = make_record(flags=P | F1 | MREV, pos=99, mate_ref_id=0, mate_pos=119, tlen=70, seq=b"A" * 50,
                    tags=[(b"MC", "Z", b"50M")])
    sr, clip = sr_of(r, min_input_base_quality=2)
    assert clip == 0 and len(sr.bases) == 50                                                             # :3098
    r = make_record(flags=P | F1 | MREV, pos=99, mate_ref_id=0, mate_pos=99, tlen=30, seq=b"A" * 50,
                    tags=[(b"MC", "Z", b"30M")])
    sr, clip = sr_of(r, min_input_base_quality=2)
    assert clip == 20 and len(sr.bases) == 30                                                            # :3134
    seq = b"A" * 10 + b"C" * 30 + b"G" * 10
    r1 = make_record(flags=P | F1 | MREV, pos=10, mate_ref_id=0, mate_pos=0, tlen=50, seq=seq,
                     tags=[(b"MC", "Z", b"50M")])
    sr, clip = sr_of(r1, min_input_base_quality=2)
    assert clip == 10 and bytes(sr.bases) == b"A" * 10 + b"C" * 30                                       # :3240
    r2 = make_record(flags=P | F2 | REV, pos=0, mate_ref_id=0, mate_pos=10, tlen=-50, seq=seq,
                     tags=[(b"MC", "Z", b"50M")])
    sr, clip = sr_of(r2, min_input_base_quality=2)
    assert clip == 10 and len(sr.bases) == 40 and bytes(sr.bases) == b"C" * 10 + b"G" * 30
    rm = make_record(flags=P | F1 | REV, pos=544, mate_ref_id=0, mate_pos=492, tlen=-124, seq=b"A" * 142,
                     cigar="47S72M23S", tags=[(b"MC", "Z", b"46S96M")])
    sr, clip = sr_of(rm, min_input_base_quality=2)
    assert len(sr.bases) == 142 and bytes(sr.bases) == b"T" * 142                                        # :3328
    rp = make_record(flags=P | F1 | MREV, pos=492, mate_ref_id=0, mate_pos=544, tlen=124, seq=b"A" * 142,
                     cigar="46S96M", tags=[(b"MC", "Z", b"47S72M23S")])
    sr, clip = sr_of(rp, min_input_base_quality=2)
    assert len(sr.bases) == 142 and bytes(sr.bases) == b"A" * 142                                        # :3370
    rs = make_record(flags=P | F1 | MREV, pos=19, mate_ref_id=0, mate_pos=19, tlen=39,
                     seq=b"AA" + b"C" * 46 + b"GG", cigar="10S35M5S", tags=[(b"MC", "Z", b"12S30M8S")])
    sr, clip = sr_of(rs, min_input_base_quality=2)
    assert clip == 2 and bytes(sr.bases) == b"AA" + b"C" * 46                                            # :3410
    # not an FR pair / no MC tag -> no clip (overlap.rs:65-80)
    assert R.num_bases_extending_past_mate(R.Rec(make_record(seq=b"A" * 10))) == 0
    assert R.num_bases_extending_past_mate(R.Rec(make_record(flags=P | F1 | MREV, pos=99, mate_ref_id=0,
                                                             mate_pos=99, tlen=30, seq=b"A" * 50))) == 0


# ---- filterToMostCommonAlignment, vanilla_caller.rs:2702-2860, 3593-3700 ----
def _srs(cigars, length=50):
    out = []
    for i, c in enumerate(cigars):
        r = R.Rec(make_record(seq=b"A" * length, cigar=c))
        out.append(R.create_source_read(r, i, 0, R.VanillaOptions(min_input_base_quality=2)))
    return out


def test_alignment_filter():
    kept, rej = R.filter_by_alignment(_srs(["50M"] * 10))
    assert len(kept) == 10 and rej == 0                                                                  # :2702
    kept, rej = R.filter_by_alignment(_srs(["10M5D10M5I30M"] * 3 + ["50M"] * 2))                         # majority
    assert [k.original_idx for k in kept] == [0, 1, 2] and rej == 2                                      # :2744
    kept, rej = R.filter_by_alignment(_srs(["25M2D25M"] * 3 + ["50M"] + ["25M1I24M"]))
    assert [k.original_idx for k in kept] == [0, 1, 2] and rej == 2                                      # :3172
    kept, rej = R.filter_by_alignment(_srs(["50M"]))
    assert len(kept) == 1 and rej == 0                                                                   # :2840
    # input order is preserved among survivors (:3646)
    kept, _ = R.filter_by_alignment(_srs(["50M", "20M1I29M", "50M", "50M"]))
    assert [k.original_idx for k in kept] == [0, 2, 3]


# ---- end to end, vanilla_caller.rs:2083-2600, 3773-3920, 4267-4640 ----
def test_two_reads_and_tags():
    c = make_caller(min_reads=1, min_consensus_base_quality=0)
    data, n = c.consensus_reads([frag(b"r1", b"GATTACA", [10] * 7), frag(b"r2", b"GATTACA", [10] * 7)])
    rec, = parse_records(data)
    assert n == 1 and rec["bases"] == b"GATTACA" and all(q > 10 for q in rec["quals"])                   # :2083
    assert rec["name"] == b"consensus:UMI1" and rec["flags"] == 0x4 and rec["ref_id"] == -1
    assert rec["tag_order"] == [b"RG", b"cD", b"cM", b"cE", b"cd", b"ce", b"MI"]                         # :1393-1444
    assert rec["tags"][b"RG"] == b"A" and rec["tags"][b"MI"] == b"UMI1" and rec["bin"] == 4680

    c = make_caller(min_reads=1, min_input_base_quality=2)
    reads = [frag(b"r%d" % i, b"A" * 10, [30] * 10) for i in range(3)] + [frag(b"r4", b"AAAAACAAAA", [30] * 10)]
    rec, = parse_records(c.consensus_reads(reads)[0])
    assert rec["bases"] == b"A" * 10 and rec["tags"][b"cD"] == 4 and rec["tags"][b"cM"] == 4             # :2396
    assert abs(rec["tags"][b"cE"] - 0.025) < 1e-6
    assert rec["tags"][b"cd"] == [4] * 10 and rec["tags"][b"ce"] == [0] * 5 + [1] + [0] * 4

    c = make_caller(min_reads=1, produce_per_base_tags=False)
    rec, = parse_records(c.consensus_reads(reads)[0])
    assert b"cd" not in rec["tags"] and b"ce" not in rec["tags"]                                         # :2574


def test_pairs_orphans_and_stats():
    # a proper pair gives R1 + R2 consensus with the pair flags (:3813)
    def pair(i, umi=b"U"):
        r1 = make_record(name=b"q%d" % i, flags=P | F1 | MREV, pos=100, mate_ref_id=0, mate_pos=300, tlen=250,
                         seq=b"ACGTACGTAC", tags=[(b"MI", "Z", umi), (b"RX", "Z", b"AAC-GGT"), (b"MC", "Z", b"10M")])
        r2 = make_record(name=b"q%d" % i, flags=P | F2 | REV, pos=300, mate_ref_id=0, mate_pos=100, tlen=-250,
                         seq=b"TTGCATTGCA", tags=[(b"MI", "Z", umi), (b"RX", "Z", b"AAC-GGT"), (b"MC", "Z", b"10M")])
        return [r1, r2]
    c = make_caller(min_reads=2, min_consensus_base_quality=2)
    data, n = c.consensus_reads(pair(0) + pair(1))
    recs = parse_records(data)
    assert n == 2 and recs[0]["flags"] == 0x4 | 0x1 | 0x40 | 0x8 and recs[1]["flags"] == 0x4 | 0x1 | 0x80 | 0x8
    assert recs[0]["bases"] == b"ACGTACGTAC" and recs[1]["bases"] == b"TGCAATGCAA"    # R2 is revcomp'd
    assert recs[0]["tags"][b"RX"] == b"AAC-GGT"
    assert c.stats.total_reads == 4 and c.stats.consensus_reads == 2 and c.stats.filtered_reads == 0
    # R1 succeeds, R2 has too few reads -> orphan: both dropped, R1 survivors counted once (:4340)
    c = make_caller(min_reads=2, min_consensus_base_quality=2)
    data, n = c.consensus_reads(pair(0) + [pair(1)[0]])
    assert n == 0 and data == b""
    assert c.stats.rejections == {"InsufficientReads": 1, "OrphanConsensus": 2} and c.stats.filtered_reads == 3
    # secondary / supplementary are filtered first (:1711)
    c = make_caller(min_reads=1, min_consensus_base_quality=2)
    sec = make_record(flags=R.SECONDARY, seq=b"ACGT", tags=[(b"MI", "Z", b"U")])
    data, n = c.consensus_reads([frag(b"a", b"ACGT", [30] * 4, b"U"), sec])
    assert n == 1 and c.stats.rejections == {"SecondaryOrSupplementary": 1}
    # reads without base qualities (all 0xFF) are rejected (:3965)
    c = make_caller(min_reads=1, min_consensus_base_quality=2)
    data, n = c.consensus_reads([frag(b"a", b"ACGT", [0xFF] * 4, b"U")])
    assert n == 0 and c.stats.rejections == {"ZeroLengthAfterTrimming": 1}


def test_rx_consensus_and_cell_barcode():
    c = make_caller(min_reads=1, min_consensus_base_quality=2, cell_tag=b"CB")
    reads = [make_record(name=b"a%d" % i, seq=b"ACGT", tags=[(b"MI", "Z", b"7"), (b"CB", "Z", b"CELL1"),
                                                            (b"RX", "Z", rx)])
             for i, rx in enumerate([b"ACGT-TTTT", b"ACGT-TTTT", b"ACGA-TTTT"])]
    rec, = parse_records(c.consensus_reads(reads)[0])
    assert rec["tags"][b"RX"] == b"ACGT-TTTT" and rec["tags"][b"CB"] == b"CELL1"
    assert rec["tag_order"] == [b"RG", b"cD", b"cM", b"cE", b"cd", b"ce", b"MI", b"CB", b"RX"]


# ---- further ports of the reference's caller tests -------------------------------------------
def test_more_source_read_cases():
    # FF pair: no mate-overlap clip (:3021-3057)
    r = make_record(flags=P | F1, pos=10, mate_ref_id=0, mate_pos=0, tlen=50, seq=b"A" * 50,
                    tags=[(b"MC", "Z", b"50M")])
    sr, clip = sr_of(r, min_input_base_quality=2)
    assert clip == 0 and len(sr.bases) == 50
    # FR pair whose reads carry the same insertion: nothing to clip (:3061-3094)
    r = make_record(flags=P | F1 | MREV, pos=0, mate_ref_id=0, mate_pos=0, tlen=80, seq=b"A" * 100,
                    cigar="40M20I40M", tags=[(b"MC", "Z", b"40M20I40M")])
    sr, clip = sr_of(r, min_input_base_quality=2)
    assert len(sr.bases) == 100
    # quality trim + mask together: "AGC" survives (:3923-3957)
    sr, _ = sr_of(make_record(seq=b"AGCACGACGT", quals=[30, 30, 30, 2, 5, 2, 3, 20, 2, 6]),
                  min_input_base_quality=15, trim=True)
    assert bytes(sr.bases) == b"AGC"


def test_read_can_join_several_cigar_groups():               # :3593-3642
    kept, rej = R.filter_by_alignment(_srs(["50M"] * 2 + ["40M1I9M"] * 3) +
                                      [R.create_source_read(R.Rec(make_record(seq=b"A" * 40, cigar="40M")), 5, 0,
                                                            R.VanillaOptions(min_input_base_quality=2))])
    assert len(kept) == 4 and 5 in [k.original_idx for k in kept]       # the 40M prefix read rides with 40M1I9M


def test_groups_pairs_and_missing_mate_cigar():
    def frag_u(name, umi):
        return frag(name, b"GATTACA", [30] * 7, umi)
    # one consensus per call, two calls for two UMI groups (:3773-3809)
    c = make_caller(min_reads=1, min_input_base_quality=2)
    assert c.consensus_reads([frag_u(b"a", b"G1"), frag_u(b"b", b"G1")])[1] == 1
    assert c.consensus_reads([frag_u(b"c", b"G2"), frag_u(b"d", b"G2")])[1] == 1
    assert c.stats.consensus_reads == 2
    # a pair without MC tags still gives R1 + R2 (:3999-4053)
    r1 = make_record(name=b"READ1", flags=P | F1 | MREV, pos=0, mate_ref_id=0, mate_pos=99, tlen=109, seq=b"A" * 10,
                     tags=[(b"MI", "Z", b"GATTACA")])
    r2 = make_record(name=b"READ1", flags=P | F2 | REV, pos=99, mate_ref_id=0, mate_pos=0, tlen=-109, seq=b"A" * 10,
                     tags=[(b"MI", "Z", b"GATTACA")])
    c = make_caller(min_reads=1, min_input_base_quality=2)
    assert c.consensus_reads([r1, r2])[1] == 2


def test_rx_consensus_uses_surviving_reads_only():           # :4058-4154
    def rd(name, cigar, rx):
        return make_record(name=name, pos=0, seq=b"A" * 10, cigar=cigar, tags=[(b"MI", "Z", b"AAA"), (b"RX", "Z", rx)])
    c = make_caller(min_reads=1, min_input_base_quality=2)
    data, n = c.consensus_reads([rd(b"READ1", "10M", b"TTT"), rd(b"READ2", "5M5D5M", b"ATT"),
                                 rd(b"READ3", "10M", b"TAT"), rd(b"READ4", "4M2I4M", b"TTA")])
    rec, = parse_records(data)
    assert n == 1 and rec["tags"][b"RX"] == b"TNT"          # TTT + TAT; the two minority alignments do not vote


def test_orphan_when_r1_fails_and_r2_succeeds():             # :4500-4640 (mirror of :4340)
    def pair(i):
        r1 = make_record(name=b"q%d" % i, flags=P | F1 | MREV, pos=100, mate_ref_id=0, mate_pos=300, tlen=250,
                         seq=b"ACGTACGTAC", tags=[(b"MI", "Z", b"U"), (b"MC", "Z", b"10M")])
        r2 = make_record(name=b"q%d" % i, flags=P | F2 | REV, pos=300, mate_ref_id=0, mate_pos=100, tlen=-250,
                         seq=b"TTGCATTGCA", tags=[(b"MI", "Z", b"U"), (b"MC", "Z", b"10M")])
        return [r1, r2]
    c = make_caller(min_reads=2, min_consensus_base_quality=2)
    data, n = c.consensus_reads(pair(0) + [pair(1)[1]])          # two R2s, one R1
    assert n == 0 and data == b""
    assert c.stats.rejections == {"InsufficientReads": 1, "OrphanConsensus": 2} and c.stats.filtered_reads == 3


# ---- consensus_umis / SimpleConsensusCaller, simple_umi.rs:257-372 (ports of fgbio's SimpleConsensusCallerTest)
def test_simple_consensus_caller_kats():
    cu = lambda umis: R.consensus_umis(list(umis), lambda pre, post, b, q: O.builder_call(pre, post, b, q)[:2])
    assert cu(["A", "A"]) == "A" and cu(["GATTACA", "GATTACA"]) == "GATTACA"                    # :290-297
    assert cu(["A", "C", "G", "T"]) == "N"                                                       # :300-312 tie
    assert cu(["A", "C", "C", "C"]) == "C" and cu(["C", "C", "C", "A"]) == "C"
    assert cu(["GATTACA"] * 3 + ["NNNNNNN"]) == "GATTACA"                                        # Ns do not vote
    assert cu(["GATT-ACA"] * 3) == "GATT-ACA" and cu(["XGAT", "XGAT"]) == "XGAT" and cu(["GATY", "GATY"]) == "GATY"
    assert cu(["AACC", "CCAA"]) == "NNNN"                                                        # :436-448
    assert cu(["ACGT", "ACGT", "CAGT"]) == "ACGT" and cu(["ACGT"] * 3 + ["ACGG"]) == "ACGT"      # :392-400, :451-462
    assert cu([]) == "" and cu(["ACGT"]) == "ACGT"                                               # :236-245
    for bad in (["A", "AC"], ["GATT-ACA", "GATT-ACA", "GATTAACA"], ["GATT-ACA", "GATT+ACA"]):    # the panics :257-287
        try:
            cu(bad)
        except AssertionError:
            continue
        raise AssertionError("expected a failure for %r" % (bad,))
