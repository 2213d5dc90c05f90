"""Known-answer tests of tests/filter_oracle.py, ported from the reference's own tests so that the oracle -- against which
the device filter is compared byte for byte -- is tied to the reference and not only to a reading of its source:
  crates/fgumi-sam/src/alignment_tags.rs     all 25 tests (NM / UQ / MD regeneration, raw-path checks)
  src/lib/tag_reversal.rs                    all 7 tests (reverse_buf_value per array type, the raw path)
  src/lib/commands/filter.rs                 the non-methylation unit tests not already ported by test_filter.py /
                                             test_duplex_filter.py: template_passes, is_duplex_consensus,
                                             check_filters_raw / check_duplex_filters_raw in count and fraction mode,
                                             process_record_raw without a reference, and the execute tests for tag
                                             regeneration, tag reversal and supplementary records
  tests/integration/test_filter_command.rs   all 6 tests
The reference's option parsing / validation tests have no counterpart here (there is no CLI); its remaining execute
tests repeat these shapes through its thread pools."""
import os
import struct
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import record_oracle as R     # noqa: E402
from tests import filter_oracle as O      # noqa: E402
from tests.bam_builder import make_record   # noqa: E402

CHR1 = b"ACGTACGTACGTACGT"   # alignment_tags.rs create_test_reference
SQ = [b"chr1"]
HDR = b"@HD\tVN:1.6\n@SQ\tSN:chr1\tLN:%d\n"


def tags(r) -> dict:
    return R._aux_tags(R.Rec(bytes(r)).aux())


def regen(seq, quals, cigar, pos=0, genome=None, **kw):
    r = bytearray(make_record(name=b"q", ref_id=0, pos=pos, cigar=cigar, seq=seq, quals=bytes(quals), **kw))
    O.regenerate(r, 0, SQ, genome or {b"chr1": CHR1})
    t = tags(r)
    return t[b"NM"][1], t[b"UQ"][1], t[b"MD"][1]


# ---- alignment_tags.rs ---------------------------------------------------------------------------------------------
CASES = [   # (test, seq, quals, cigar, NM, UQ, MD)
    ("perfect_match", b"ACGT", [30] * 4, "4M", 0, 0, b"4"),
    ("one_mismatch", b"ATGT", [30] * 4, "4M", 1, 30, b"1C2"),
    ("masked_base", b"ANGT", [30, 0, 30, 30], "4M", 1, 0, b"1C2"),
    ("insertion", b"ACTTGT", [30, 30, 25, 25, 30, 30], "2M2I2M", 2, 0, b"4"),
    ("deletion", b"ACAC", [30] * 4, "2M2D2M", 2, 0, b"2^GT2"),
    ("soft_clip", b"TTACGTGG", [20, 20, 30, 30, 30, 30, 20, 20], "2S4M2S", 0, 0, b"4"),
    ("hard_clip", b"ACGT", [30] * 4, "2H4M2H", 0, 0, b"4"),
    ("multiple_mismatches", b"AATT", [30, 25, 20, 35], "4M", 2, 45, b"1C0G1"),
    ("multiple_masked_bases", b"ANNN", [30, 0, 0, 0], "4M", 3, 0, b"1C0G0T0"),
    ("complex_cigar", b"ACTCAC", [30, 30, 25, 30, 30, 30], "2M1I1M1D2M", 3, 30, b"2G0^T2"),
    ("sequence_match_and_mismatch_ops", b"ACTT", [30, 30, 25, 30], "2=1X1=", 1, 25, b"2G1"),
    ("pad_operation", b"ACGT", [30] * 4, "2M2P2M", 0, 0, b"4"),
    ("skip_operation", b"ACGT", [30] * 4, "2M2N2M", 2, 60, b"2A0C0"),
    ("case_insensitive_matching", b"acgt", [30] * 4, "4M", 0, 0, b"4"),
    ("insertion_at_end", b"ACGTTT", [30, 30, 30, 30, 20, 20], "4M2I", 2, 0, b"4"),
    ("deletion_at_end", b"AC", [30, 30], "2M2D", 2, 0, b"2^GT0"),
    ("mixed_matches_and_masks", b"ACNTTC", [30, 30, 0, 30, 25, 30], "6M", 2, 25, b"2G1A1"),
    ("regenerate_alignment_tags_raw_happy_path", b"ATGT", [30, 30, 25, 30], "4M", 1, 30, b"1C2"),
    ("regenerate_alignment_tags_raw_with_masked_bases", b"ANGT", [30, 0, 30, 30], "4M", 1, 0, b"1C2"),
    ("regenerate_alignment_tags_zero_ref_span_returns_true", b"ACGT", [30] * 4, "4I", 0, 0, b"0"),
    ("regenerate_alignment_tags_raw_zero_ref_span_returns_true", b"ACGT", [30] * 4, "4I", 0, 0, b"0"),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_alignment_tags(case):
    _, seq, quals, cigar, nm, uq, md = case
    assert regen(seq, quals, cigar) == (nm, uq, md)


def test_alignment_tags_unmapped_read():
    r = bytearray(make_record(name=b"q", flags=0x4, ref_id=-1, pos=-1, cigar=[], seq=b"ACGT",
                              tags=[(b"NM", "i", 7), (b"MD", "Z", b"6A7C8T9G"), (b"UQ", "i", 237)]))
    O.regenerate(r, 0, SQ, {b"chr1": CHR1})
    assert not {b"NM", b"MD", b"UQ"} & set(tags(r))


def test_alignment_tags_regenerate_tags_fgbio_equivalent():
    got = regen(b"AAACAAAATA", [20] * 10, "10M", genome={b"chr1": b"A" * 20},
                tags=[(b"NM", "i", 7), (b"MD", "Z", b"6A7C8T9G"), (b"UQ", "i", 237)])
    assert got == (2, 40, b"3A4A1")


def test_alignment_tags_raw_validates_bounds():
    r = make_record(name=b"q", ref_id=0, pos=0, cigar="8M", seq=b"ACGTACGT")
    cut = r[:O.aux_offset(r) - 8]   # the qualities removed
    with pytest.raises(O.FilterError):
        O.process_record(bytearray(cut), 0, O.Config(), SQ, {b"chr1": CHR1})


def test_alignment_tags_raw_rejects_short_record():
    with pytest.raises(O.FilterError):
        O.process_record(bytearray(10), 0, O.Config(), SQ, {b"chr1": CHR1})


# ---- tag_reversal.rs -----------------------------------------------------------------------------------------------
def b_array(tag: bytes, sub: str, vals) -> bytes:
    fmt = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}[sub]
    return tag + b"B" + sub.encode() + struct.pack("<I%d%s" % (len(vals), fmt), len(vals), *vals)


def reversed_record(aux: bytes, flags: int = 0x10) -> bytearray:
    r = bytearray(make_record(name=b"q", flags=flags, ref_id=-1, pos=-1, cigar=[], seq=b"ACGT")) + aux
    O.reverse_per_base_tags(r)
    return r


@pytest.mark.parametrize("sub,vals", [("c", [1, 2, 3]), ("C", [1, 2, 3]), ("s", [1, 2, 3]), ("S", [1, 2, 3]),
                                      ("i", [1, 2, 3]), ("I", [1, 2, 3]), ("f", [1.0, 2.0, 3.0])])
def test_reverse_buf_value_all_array_types(sub, vals):
    r = reversed_record(b_array(b"cd", sub, vals))
    assert tags(r)[b"cd"] == ("B" + sub, vals[::-1])


def test_reverse_buf_value_non_array():
    r = reversed_record(b"cdi" + struct.pack("<i", 42))
    assert tags(r)[b"cd"] == ("i", 42)


def test_reverse_per_base_tags_raw_string_tag_aq():
    assert tags(reversed_record(b"aqZIIHG\0"))[b"aq"] == ("Z", b"GHII")


@pytest.mark.parametrize("tag", [b"ac", b"bc"])
def test_reverse_per_base_tags_raw_revcomp_string_tags(tag):
    assert tags(reversed_record(tag + b"ZACGA\0"))[tag] == ("Z", b"TCGT")


def test_reverse_per_base_tags_raw_short_record():
    with pytest.raises(O.FilterError):
        O.process_record(bytearray(16), 0, O.Config(reverse_per_base_tags=True), SQ, None)


def test_reverse_per_base_tags_raw_positive_strand():
    aux = b_array(b"cd", "S", [1, 2, 3, 4])
    assert tags(reversed_record(aux, flags=0))[b"cd"] == ("BS", [1, 2, 3, 4])


def test_reverse_per_base_tags_raw_negative_strand():
    assert tags(reversed_record(b_array(b"cd", "S", [1, 2, 3, 4])))[b"cd"] == ("BS", [4, 3, 2, 1])


# ---- commands/filter.rs ------------------------------------------------------------------------------------------
def decide(recs, passes):
    """template_passes through filter_records' template branch: the kept records of one template whose records pass
    as `passes` says (a failing record is given a low cD)."""
    out = []
    for r, ok in zip(recs, passes):
        out.append(bytes(make_record(name=b"t", flags=R.Rec(r).flags, ref_id=-1, pos=-1, cigar=[], seq=b"ACGT",
                                     tags=[(b"cD", "i", 10 if ok else 0), (b"cd", "Bs", [5] * 4)])))
    cfg = O.Config(min_reads=(1,), max_base_error_rate=(1.0,))
    return O.filter_records(out, b"", cfg, None)[2]["passed"]


def test_template_passes_all_pass():
    r1 = make_record(name=b"t", flags=0x41 | 0x4, ref_id=-1, pos=-1, cigar=[], seq=b"ACGT")
    r2 = make_record(name=b"t", flags=0x81 | 0x4, ref_id=-1, pos=-1, cigar=[], seq=b"GGGG")
    assert decide([r1, r2], [True, True]) == 2


def test_template_passes_one_fails():
    r1 = make_record(name=b"t", flags=0x41 | 0x4, ref_id=-1, pos=-1, cigar=[], seq=b"ACGT")
    r2 = make_record(name=b"t", flags=0x81 | 0x4, ref_id=-1, pos=-1, cigar=[], seq=b"GGGG")
    assert decide([r1, r2], [True, False]) == 0


def test_is_duplex_consensus_simplex():
    assert not R.is_duplex_consensus(R.Rec(make_record(seq=b"ACGT")).aux())


def test_is_duplex_consensus_with_tag():
    assert R.is_duplex_consensus(R.Rec(make_record(seq=b"ACGT", cigar="4M", tags=[(b"aD", "i", 10)])).aux())


def _no_call_record(seq, duplex=False):
    t = ([(b"aD", "i", 10), (b"bD", "i", 8), (b"aE", "f", 0.01), (b"bE", "f", 0.01), (b"aM", "i", 10),
          (b"bM", "i", 8)] if duplex else [(b"cD", "i", 10), (b"cE", "f", 0.01)])
    return make_record(seq=seq, cigar=[], ref_id=-1, pos=-1, quals=[30] * len(seq), tags=t)


def _check(r, max_nc, duplex=False):   # check_filters_raw / check_duplex_filters_raw
    th = R.FilterThresholds(5, 0.1, 0.1)
    aux = R.Rec(r).aux()
    st = R.filter_duplex_read(aux, th, th, th) if duplex else R.filter_read(aux, th)
    return st == R.FILTER_PASS and R.check_no_call_and_quality(r, None, max_nc)


def test_check_filters_raw_no_call_fraction_mode():
    r = _no_call_record(b"AANNTTGGCC")
    assert _check(r, 0.2) and not _check(r, 0.19)


def test_check_filters_raw_no_call_count_mode_pass():
    r = _no_call_record(b"AANNNTTGGC")
    assert _check(r, 5.0) and _check(r, 3.0)


def test_check_filters_raw_no_call_count_mode_fail():
    assert not _check(_no_call_record(b"AANNNTTGGC"), 2.0)


def test_check_duplex_filters_raw_no_call_count_mode():
    r = _no_call_record(b"AANNNTTGGC", duplex=True)
    assert _check(r, 5.0, True) and not _check(r, 2.0, True)


def _cons(name, flags, ref_id, pos0, seq, cd, ce, extra=()):
    return bytes(make_record(name=name, flags=flags, ref_id=ref_id, pos=pos0, cigar=([] if flags & 4 else None),
                             seq=seq, quals=[35] * len(seq),
                             tags=list(extra) + [(b"cd", "Bs", cd), (b"ce", "Bs", ce)]))


def test_process_record_raw_no_reference():
    r = bytearray(_cons(b"unmapped_read", 0x4, -1, -1, b"ACGTACGT", [10] * 8, [0] * 8))
    assert O.process_record(r, 0, O.Config(min_reads=(1,), max_no_call_fraction=0.2), [], None) == (0, True)


def test_process_record_raw_no_reference_mapped_fails():
    r = bytearray(_cons(b"mapped_read", 0, 0, 99, b"ACGTACGT", [10] * 8, [0] * 8))
    with pytest.raises(O.FilterError, match="--ref is required"):
        O.process_record(r, 0, O.Config(min_reads=(1,), max_no_call_fraction=0.2), SQ, None)


def _simplex(name, pos1, bases, quals, depth, err, cd, ce, flags=0):   # create_simplex_consensus_record
    return bytes(make_record(name=name, flags=flags, ref_id=0, pos=pos1 - 1, seq=bases, quals=quals,
                             tags=[(b"cD", "i", depth), (b"cM", "i", depth), (b"cE", "f", err), (b"cd", "Bs", cd),
                                   (b"ce", "Bs", ce)]))


A1000 = {b"chr1": b"A" * 1000}


@pytest.mark.parametrize("reverse", [False, True])
def test_filter_execute_regenerates_and_reverses_tags(reverse):
    """test_filter_execute_regenerates_tags / test_filter_execute_reverse_per_base_tags: the one read passes, and its
    tags are regenerated against the all-A reference."""
    r = _simplex(b"read1", 100, b"AAAA", [30] * 4, 10, 0.01, [10] * 4, [0] * 4)
    cfg = O.Config(min_reads=(1,), max_read_error_rate=(1.0,), max_base_error_rate=(1.0,), min_base_quality=10,
                   max_no_call_fraction=1.0, reverse_per_base_tags=reverse)
    kept, _, st = O.filter_records([r], HDR % 1000, cfg, A1000)
    assert st["passed"] == 1
    out = kept[4:]
    assert (tags(out)[b"NM"][1], tags(out)[b"UQ"][1], tags(out)[b"MD"][1]) == (0, 0, b"4")


def test_filter_execute_with_supplementary_records():
    primary = _simplex(b"read_with_supp", 100, b"AAAA", [30] * 4, 10, 0.01, [10] * 4, [0] * 4)
    supp = _simplex(b"read_with_supp", 500, b"CCCC", [30] * 4, 10, 0.01, [10] * 4, [0] * 4, flags=0x800)
    supp_fail = _simplex(b"read_with_supp", 600, b"GGGG", [30] * 4, 2, 0.5, [2] * 4, [0] * 4, flags=0x800)
    cfg = O.Config(min_reads=(5,), max_read_error_rate=(0.1,), max_base_error_rate=(0.3,), min_base_quality=10,
                   max_no_call_fraction=0.5)
    kept, rej, st = O.filter_records([primary, supp, supp_fail], HDR % 1000, cfg, A1000)
    assert (st["passed"], st["failed"]) == (2, 1)
    assert rej[4:].startswith(supp_fail[:14])   # the failing supplementary is the reject


# ---- tests/integration/test_filter_command.rs ----------------------------------------------------------------------
ACGT10K = {b"chr1": b"ACGTACGT" * 1250}
DEFAULTS = dict(max_read_error_rate=(0.025,), max_base_error_rate=(0.1,), max_no_call_fraction=0.2)


def _run(recs, genome, **kw):
    cfg = O.Config(**{**DEFAULTS, **kw})
    return O.filter_records(recs, HDR % 10000, cfg, genome)


def test_filter_command_basic():
    r1 = _cons(b"cons1", 0, 0, 99, b"ACGTACGT", [10] * 8, [0] * 8)
    r2 = _cons(b"cons2", 0, 0, 199, b"ACGTACGT", [5] * 8, [0] * 8)
    assert _run([r1, r2], ACGT10K, min_reads=(1,), max_no_call_fraction=1.0)[2]["passed"] == 2


def test_filter_command_rejects_low_depth():
    good = _cons(b"good", 0, 0, 99, b"ACGTACGT", [10] * 8, [0] * 8)
    low = _cons(b"low_depth", 0, 0, 199, b"ACGTACGT", [1] * 8, [0] * 8)
    kept, rej, st = _run([good, low], ACGT10K, min_reads=(3,))
    assert (st["passed"], st["failed"]) == (1, 1)
    assert R.Rec(kept[4:]).name == b"good" and R.Rec(rej[4:]).name == b"low_depth"


def test_filter_command_with_stats():
    r = bytes(make_record(name=b"cons1", ref_id=0, pos=99, seq=b"ACGTACGT", quals=[35] * 8,
                          tags=[(b"cD", "i", 10), (b"cM", "i", 8), (b"cE", "f", 0.005)]))
    _, _, st = _run([r], ACGT10K, min_reads=(1,))
    from fgumi_b200.filter import filter_stats_text
    text = filter_stats_text(st)
    assert text.strip() and "total_reads" in text and st["total"] == 1


def test_filter_command_no_ref_unmapped_reads():
    r1 = _cons(b"cons1", 0x4, -1, -1, b"ACGTACGT", [10] * 8, [0] * 8)
    r2 = _cons(b"cons2", 0x4, -1, -1, b"ACGTACGT", [5] * 8, [0] * 8)
    assert _run([r1, r2], None, min_reads=(1,), max_no_call_fraction=1.0)[2]["passed"] == 2


def test_filter_command_no_ref_with_rejects():
    good = _cons(b"good", 0x4, -1, -1, b"ACGTACGT", [10] * 8, [0] * 8)
    low = _cons(b"low_depth", 0x4, -1, -1, b"ACGTACGT", [1] * 8, [0] * 8)
    kept, rej, st = _run([good, low], None, min_reads=(3,))
    assert (st["passed"], st["failed"]) == (1, 1) and R.Rec(rej[4:]).name == b"low_depth"


def test_filter_command_no_ref_mapped_reads_fails():
    r = _cons(b"cons1", 0, 0, 99, b"ACGTACGT", [10] * 8, [0] * 8)
    with pytest.raises(O.FilterError, match="--ref is required"):
        _run([r], None, min_reads=(1,))
