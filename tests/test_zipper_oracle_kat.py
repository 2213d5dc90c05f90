"""tests/zipper_oracle.py pinned to ports of the reference's own tests: src/lib/commands/zipper.rs (#[test]s from line
1399), the TagInfo tests (zipper.rs:1730, 2204; fgumi-umi lib.rs), the tag editors of crates/fgumi-raw-bam/src/tags.rs
and the BAM cases of tests/integration/test_zipper_command.rs.  Each port builds the reference test's records (its
SamBuilder defaults: 100-base reads, 100M, MAPQ 60) and checks the oracle's output against the test's expected values.

Reference tests with no port, and why:
- test_peek_stdin_bgzf_* (4): stdin format detection; stdin is not offered.
- test_raw_restore_unconverted_bases_* and test_raw_restore_removes_nm_md_when_bases_changed (10): the EM-seq
  restoration; --restore-unconverted-bases is not offered.
- test_exclude_missing_reads_parsing, test_skip_tc_tags_parsing, test_restore_unconverted_bases_parsing: CLI parsing.
- test_file_not_found_error: the CLI's file checks (bamio.find_dict_path's lookup is tested in test_zipper_records.py).
- test_multithreaded_processing: the reference's writer threads; its per-record expectations are test_basic_merge's,
  and the library's thread counts are compared in test_zipper_records.py.
- The SAM-input cases of test_zipper_command.rs: SAM text on the mapped side is not offered.
"""
import struct

import pytest

from tests import zipper_oracle as O
from tests.bam_builder import make_record, parse_records

SEQ = b"A" * 100


def mapped(name, flags, pos, cigar="100M", ref=0, mapq=60, tags=(), seq=None):
    s = SEQ if seq is None else seq
    return make_record(name=name, flags=flags, ref_id=ref, pos=pos, mapq=mapq, cigar=cigar, seq=s, tags=tags)


def unmapped(name, flags, tags=()):
    return make_record(name=name, flags=flags | 0x4, ref_id=-1, pos=-1, mapq=0, cigar=[], seq=SEQ, tags=tags)


def upair(name, tags=(), qc2=False):
    return [unmapped(name, 0x49, tags), unmapped(name, 0x89 | (0x200 if qc2 else 0), tags)]


def mpair(name, s1, s2, rev1=False, rev2=True, tags=()):
    """add_pair_with_attrs(name, start1, start2, ...): 1-based starts, R2 on the reverse strand by default."""
    return [mapped(name, 0x41 | (0x10 if rev1 else 0) | (0x20 if rev2 else 0), s1 - 1, tags=tags),
            mapped(name, 0x81 | (0x10 if rev2 else 0) | (0x20 if rev1 else 0), s2 - 1, tags=tags)]


def run(u, m, **kw):
    out, _, stats = O.zipper(u, m, **kw)
    return parse_records(O.stream(out)), stats


PG = (b"PG", "Z", b"bwa")


def test_basic_merge():
    u = upair(b"q1", [(b"RX", "Z", b"ACGT"), (b"xy", "i", 1234)]) + upair(b"q2", [(b"RX", "Z", b"GGTA"), (b"xy", "i", 4567)])
    m = mpair(b"q1", 100, 200, tags=[PG, (b"AS", "i", 77)]) + mpair(b"q2", 500, 700, tags=[PG, (b"AS", "i", 16)])
    recs, _ = run(u, m)
    assert len(recs) == 4
    for r in recs:
        for t in (b"RX", b"xy", b"AS", b"PG", b"MC", b"MQ"):
            assert t in r["tags"]
    assert recs[0]["tags"][b"RX"] == b"ACGT" and recs[2]["tags"][b"xy"] == 4567


def test_unpaired_reads():
    u = [unmapped(b"q1", 0, [(b"RX", "Z", b"ACGT"), (b"xy", "i", 1234)]),
         unmapped(b"q2", 0, [(b"RX", "Z", b"GGTA"), (b"xy", "i", 4567)])]
    m = [mapped(b"q1", 0, 99, tags=[PG, (b"AS", "i", 77)]), mapped(b"q2", 0x10, 499, tags=[PG, (b"AS", "i", 16)])]
    recs, _ = run(u, m)
    assert len(recs) == 2
    for r in recs:
        assert {b"RX", b"xy", b"AS"} <= set(r["tags"])


def _rev_attrs():
    return [(b"n1", "Bs", [1, 2, 3, 4, 5]), (b"n2", "Bs", [2, 3, 4, 5, 6]), (b"s1", "Z", b"abcde"),
            (b"s2", "Z", b"vwxyz"), (b"s3", "Z", b"AGAGG")]


def _check_rev(r):
    t = r["tags"]
    assert b"AS" not in t
    if r["flags"] & 0x10:
        assert t[b"n1"] == [5, 4, 3, 2, 1] and t[b"n2"] == [6, 5, 4, 3, 2] and t[b"s1"] == b"edcba"
        assert t[b"s3"] == b"CCTCT"
    else:
        assert t[b"n1"] == [1, 2, 3, 4, 5] and t[b"s1"] == b"abcde" and t[b"s3"] == b"AGAGG"
    assert t[b"s2"] == b"vwxyz"


def test_tag_removal_reverse_revcomp():
    recs, _ = run(upair(b"q1", _rev_attrs()), mpair(b"q1", 100, 200, tags=[PG, (b"AS", "i", 77)]),
                  remove=["AS"], reverse=["n1", "n2", "s1"], revcomp=["s3"])
    assert len(recs) == 2
    for r in recs:
        _check_rev(r)


def test_consensus_tag_set():
    u = [unmapped(b"q1", 0, [(b"aD", "Z", b"AAAGG"), (b"bD", "Z", b"AAAGC"), (b"ad", "Bs", [3, 3, 4, 4, 2])])]
    m = [mapped(b"q1", 0, 99, tags=[PG, (b"AS", "i", 77)]), mapped(b"q1", 0x800 | 0x10, 199, tags=[PG, (b"AS", "i", 77)])]
    recs, _ = run(u, m, reverse=["Consensus"], revcomp=["Consensus"])
    assert len(recs) == 2
    for r in recs:
        t = r["tags"]
        if r["flags"] & 0x10:
            assert (t[b"aD"], t[b"bD"], t[b"ad"]) == (b"CCTTT", b"GCTTT", [2, 4, 4, 3, 3])
        else:
            assert (t[b"aD"], t[b"bD"], t[b"ad"]) == (b"AAAGG", b"AAAGC", [3, 3, 4, 4, 2])


def test_unmapped_only_reads():
    u = [unmapped(b"q%d" % i, 0, [(b"RX", "Z", b"ACGT")]) for i in (1, 2, 3)]
    m = [mapped(b"q1", 0, 99, tags=[PG]), mapped(b"q3", 0x10, 199, tags=[PG])]
    recs, stats = run(u, m)
    assert [r["name"] for r in recs] == [b"q1", b"q2", b"q3"]
    assert recs[1]["flags"] & 0x4
    assert stats == [2, 1, 0, 3]


def test_tag_info_expansion():
    _, rev, rc = O.tag_info([], ["Consensus"], ["Consensus"])
    assert {"ad", "ae", "bd", "be", "cd"} <= rev and {"aD", "bD", "cD"} <= rc
    assert "ce" not in rev


@pytest.mark.parametrize("rev,rc,expect", [([], [], False), (["n1"], [], True), ([], ["s1"], True),
                                           (["n1"], ["s1"], True)])
def test_tag_info_has_revs_or_revcomps(rev, rc, expect):
    _, a, b = O.tag_info([], rev, rc)
    assert bool(a or b) == expect


def test_mate_info_fixing():
    recs, _ = run(upair(b"q1", [(b"RX", "Z", b"ACGT")]), mpair(b"q1", 100, 200, tags=[PG, (b"AS", "i", 77)]))
    for r in recs:
        assert b"MQ" in r["tags"] and b"MC" in r["tags"]


def test_qc_flag_transfer():
    recs, _ = run(upair(b"q1", [(b"RX", "Z", b"ACGT")], qc2=True), mpair(b"q1", 100, 200, tags=[PG]))
    assert not recs[0]["flags"] & 0x200 and recs[1]["flags"] & 0x200


def test_qc_flag_removal():
    recs, _ = run([unmapped(b"q1", 0, [(b"RX", "Z", b"ACGT")])], [mapped(b"q1", 0x200, 99)])
    assert len(recs) == 1 and not recs[0]["flags"] & 0x200


def test_tag_operations_on_secondary_and_supplementary():
    m = [mapped(b"q1", 0, 99, tags=[PG, (b"AS", "i", 77)]), mapped(b"q1", 0x100 | 0x10, 199, tags=[PG, (b"AS", "i", 77)]),
         mapped(b"q1", 0x800 | 0x10, 299, tags=[PG, (b"AS", "i", 77)])]
    recs, _ = run([unmapped(b"q1", 0, _rev_attrs())], m, remove=["AS"], reverse=["n1", "n2", "s1"], revcomp=["s3"])
    assert len(recs) == 3
    assert sum(1 for r in recs if r["flags"] & 0x900) == 2 and sum(1 for r in recs if r["flags"] & 0x10) == 2
    for r in recs:
        _check_rev(r)


def test_empty_unmapped():
    with pytest.raises(ValueError):
        run([], [mapped(b"q1", 0, 99, tags=[PG])])


def test_both_inputs_empty():
    assert run([], [])[0] == []


def test_merge_mixed_strands():
    recs, _ = run(upair(b"q1", [(b"RX", "Z", b"ACGT"), (b"xy", "i", 1234)]), mpair(b"q1", 100, 200, tags=[PG]))
    assert len(recs) == 2 and all({b"RX", b"xy"} <= set(r["tags"]) for r in recs)


def test_multiple_secondary_alignments():
    m = [mapped(b"q1", 0, 99, tags=[PG])] + [mapped(b"q1", 0x100, 199 + i * 100) for i in range(3)]
    recs, _ = run([unmapped(b"q1", 0, [(b"RX", "Z", b"ACGT")])], m)
    assert len(recs) == 4 and all(r["tags"][b"RX"] == b"ACGT" for r in recs)


def test_r2_only_mapping():
    recs, _ = run(upair(b"q1", [(b"RX", "Z", b"ACGT")]), [mapped(b"q1", 0x81, 199)])
    assert len(recs) == 1 and not recs[0]["flags"] & 0x40 and recs[0]["tags"][b"RX"] == b"ACGT"


def test_exclude_missing_reads():
    u = upair(b"q1", [(b"RX", "Z", b"ACGT")]) + upair(b"q2", [(b"RX", "Z", b"ACGT")]) + upair(b"q3", [(b"RX", "Z", b"ACGT")])
    m = mpair(b"q1", 100, 200, tags=[PG]) + mpair(b"q3", 300, 400, tags=[PG])
    assert len(run(u, m)[0]) == 6
    recs, stats = run(u, m, exclude_missing=True)
    assert len(recs) == 4 and all(r["name"] != b"q2" for r in recs) and stats[2] == 1


def tc(r):
    v = r["tags"].get(b"tc")
    return None if v is None else tuple(v)


def test_add_pa_tag_to_supplementary_r1():
    m = [mapped(b"q1", 0x41, 99, "8M", seq=b"A" * 8), mapped(b"q1", 0x841, 4999, "8M", seq=b"A" * 8)]
    recs, _ = run([unmapped(b"q1", 0x41)], m)
    assert tc(recs[1]) == (0, 100, 0, 0, 100, 0) and tc(recs[0]) is None


def test_add_pa_tag_to_secondary_reverse_strand():
    m = [mapped(b"q1", 0x51, 199, "8M", seq=b"A" * 8), mapped(b"q1", 0x141, 2999, "8M", seq=b"A" * 8)]
    recs, _ = run([unmapped(b"q1", 0x41)], m)
    assert tc(recs[1])[:3] == (0, 207, 1)


def test_add_pa_tag_paired_end_r2_supplementary():
    m = [mapped(b"q1", 0x41, 99, "8M", seq=b"A" * 8), mapped(b"q1", 0x91, 299, "8M", seq=b"A" * 8),
         mapped(b"q1", 0x881, 4999, "4M", seq=b"A" * 4)]
    recs, _ = run([unmapped(b"q1", 0x41), unmapped(b"q1", 0x81)], m)
    assert tc(recs[2]) == (0, 100, 0, 0, 307, 1)


def test_no_pa_tag_when_no_primary():
    recs, _ = run([unmapped(b"q1", 0x41)], [mapped(b"q1", 0x841, 4999, "4M", seq=b"A" * 4)])
    assert tc(recs[0]) is None


def test_pa_tag_added_during_merge():
    m = mpair(b"q1", 100, 200) + [mapped(b"q1", 0x841, 4999, "12M", seq=b"A" * 12)]
    recs, _ = run(upair(b"q1", [(b"RX", "Z", b"ACGT")]), m)
    sup = [r for r in recs if r["flags"] & 0x800][0]
    assert tc(sup) == (0, 100, 0, 0, 299, 1)


def test_add_pa_tag_early_exit_no_secondary_supplementary():
    m = [mapped(b"q1", 0x41, 99, "4M", seq=b"A" * 4), mapped(b"q1", 0x91, 199, "4M", seq=b"A" * 4)]
    recs, _ = run([unmapped(b"q1", 0x41), unmapped(b"q1", 0x81)], m)
    assert all(tc(r) is None for r in recs)


def test_add_pa_tag_only_to_secondary_supplementary():
    m = [mapped(b"q1", 0x41, 99, "4M", seq=b"A" * 4), mapped(b"q1", 0x141, 4999, "4M", seq=b"A" * 4)]
    recs, _ = run([unmapped(b"q1", 0x41)], m)
    assert tc(recs[0]) is None and tc(recs[1]) is not None


@pytest.mark.parametrize("skip", [True, False])
def test_skip_tc_tags(skip):
    m = [mapped(b"q1", 0x41, 99, "4M", seq=b"A" * 4), mapped(b"q1", 0x841, 4999, "4M", seq=b"A" * 4)]
    recs, _ = run([unmapped(b"q1", 0x41)], m, skip_tc=skip)
    assert (tc(recs[1]) is None) == skip


def test_as_xs_normalization():
    m = [mapped(b"q1", 0, 99, tags=[(b"AS", "i", 77), (b"XS", "i", 50)])]
    out, _, _ = O.zipper([unmapped(b"q1", 0, [(b"RX", "Z", b"ACGT")])], m)
    r = out[0]
    assert b"ASc\x4d" in r and b"XSc\x32" in r   # Int8(77), Int8(50)


def test_as_xs_normalization_large_values():
    m = [mapped(b"q1", 0, 99, tags=[(b"AS", "i", 300), (b"XS", "i", 70000)])]
    r = O.zipper([unmapped(b"q1", 0, [(b"RX", "Z", b"ACGT")])], m)[0][0]
    assert b"ASs" + struct.pack("<h", 300) in r and b"XSi" + struct.pack("<i", 70000) in r


def test_negative_strand_r1_tag_copying():
    recs, _ = run(upair(b"q1", [(b"s1", "Z", b"abcde"), (b"s3", "Z", b"AGAGG")]), mpair(b"q1", 100, 200, rev1=True, rev2=False),
                  reverse=["s1"], revcomp=["s3"])
    assert recs[0]["tags"][b"s1"] == b"edcba" and recs[0]["tags"][b"s3"] == b"CCTCT"
    assert recs[1]["tags"][b"s1"] == b"abcde"


def test_negative_strand_both_reads():
    recs, _ = run(upair(b"q1", [(b"s1", "Z", b"abcde")]), mpair(b"q1", 100, 200, rev1=True, rev2=True), reverse=["s1"])
    assert all(r["tags"][b"s1"] == b"edcba" for r in recs)


def test_fix_mate_info_values():
    # both mapped: R1 + at 100, R2 - at 200 (100M): TLEN 200, mate fields, MQ / MC, ms from the mate's AS
    m = [mapped(b"q1", 0x41, 99, tags=[(b"AS", "i", 77)], mapq=30), mapped(b"q1", 0x91, 199, tags=[(b"AS", "i", 55)], mapq=40)]
    recs, _ = run(upair(b"q1"), m)
    r1, r2 = recs
    assert (r1["mate_ref_id"], r1["mate_pos"], r2["mate_pos"]) == (0, 199, 99)
    assert (r1["tlen"], r2["tlen"]) == (200, -200)
    assert r1["flags"] & 0x20 and not r2["flags"] & 0x20
    assert (r1["tags"][b"MQ"], r2["tags"][b"MQ"]) == (40, 30)
    assert (r1["tags"][b"MC"], r2["tags"][b"MC"]) == (b"100M", b"100M")
    assert (r1["tags"][b"ms"], r2["tags"][b"ms"]) == (55, 77)


def test_fix_mate_info_supplementary():
    m = [mapped(b"q1", 0x41, 99, mapq=30), mapped(b"q1", 0x91, 199, mapq=40, tags=[(b"AS", "i", 55)]),
         mapped(b"q1", 0x841, 999, "50M", seq=b"A" * 50)]
    recs, _ = run(upair(b"q1"), m)
    s = recs[2]
    assert (s["mate_ref_id"], s["mate_pos"], s["tlen"]) == (0, 199, 200)
    assert s["flags"] & 0x20 and not s["flags"] & 0x8
    assert (s["tags"][b"MQ"], s["tags"][b"MC"], s["tags"][b"ms"]) == (40, b"100M", 55)


def test_fix_mate_info_one_unmapped():
    m = [mapped(b"q1", 0x41, 99, mapq=30), make_record(name=b"q1", flags=0x85, ref_id=-1, pos=-1, mapq=0, cigar=[], seq=SEQ)]
    recs, _ = run(upair(b"q1"), m)
    r1, r2 = recs
    assert (r2["ref_id"], r2["pos"]) == (0, 99)
    assert r1["flags"] & 0x8 and b"MQ" not in r1["tags"] and b"MC" not in r1["tags"] and r1["tlen"] == 0
    assert r2["tags"][b"MQ"] == 30 and r2["tags"][b"MC"] == b"100M" and r2["tlen"] == 0


def test_fix_mate_info_r2_supplementary():
    m = [mapped(b"q1", 0x41, 99, mapq=30, tags=[(b"AS", "i", 11)]), mapped(b"q1", 0x91, 199, mapq=40),
         mapped(b"q1", 0x881, 999, "50M", seq=b"A" * 50)]
    recs, _ = run(upair(b"q1"), m)
    s = recs[2]
    assert (s["mate_pos"], s["tlen"]) == (99, -200)
    assert not s["flags"] & 0x20
    assert (s["tags"][b"MQ"], s["tags"][b"MC"], s["tags"][b"ms"]) == (30, b"100M", 11)


def test_fix_mate_info_both_unmapped():
    m = [make_record(name=b"q1", flags=0x4D, ref_id=0, pos=5, cigar=[], seq=SEQ, tags=[(b"MQ", "i", 3), (b"MC", "Z", b"1M")]),
         make_record(name=b"q1", flags=0x9D, ref_id=0, pos=5, cigar=[], seq=SEQ)]
    recs, _ = run(upair(b"q1"), m)
    for r in recs:
        assert (r["ref_id"], r["pos"], r["mate_ref_id"], r["mate_pos"], r["tlen"]) == (-1, -1, -1, -1, 0)
        assert r["flags"] & 0x8 and b"MQ" not in r["tags"] and b"MC" not in r["tags"]
    assert recs[0]["flags"] & 0x20 and not recs[1]["flags"] & 0x20


def test_varied_tag_types_roundtrip():
    tags = [(b"zi", "i", -5), (b"zc", "c", -3), (b"zC", "C", 200), (b"zs", "s", -300), (b"zS", "S", 60000),
            (b"zI", "I", 4000000000), (b"zf", "f", 1.5), (b"zA", "A", b"Q"), (b"zZ", "Z", b"str"), (b"zH", "H", b"1AE3"),
            (b"zB", "Bi", [1, -2, 3]), (b"zF", "Bf", [0.5])]
    u = unmapped(b"q1", 0, tags)
    out = O.zipper([u], [mapped(b"q1", 0, 99)])[0][0]
    assert [e[2] for e in O.entries(bytearray(out))] == [e[2] for e in O.entries(bytearray(u))]   # every type verbatim


# ---- tags.rs editors -------------------------------------------------------------------------------------------

def rec_with(tags):
    return bytearray(make_record(name=b"r", seq=b"AC", tags=tags))


def aux(r):
    return bytes(r[O.aux_off(r):])


def test_update_int_tag_in_place_for_i():
    r = rec_with([(b"MQ", "i", 5), (b"xx", "Z", b"a")])
    O.update_int(r, b"MQ", 60)
    assert aux(r) == b"MQi" + struct.pack("<i", 60) + b"xxZa\0"


def test_update_int_tag_moves_other_types():
    r = rec_with([(b"MQ", "C", 5), (b"xx", "Z", b"a")])
    O.update_int(r, b"MQ", 200)
    assert aux(r) == b"xxZa\0MQC\xc8"


def test_update_int_tag_appends_when_absent():
    r = rec_with([])
    O.update_int(r, b"MQ", 70000)
    assert aux(r) == b"MQi" + struct.pack("<i", 70000)


@pytest.mark.parametrize("v,enc", [(-1, b"c\xff"), (127, b"c\x7f"), (128, b"C\x80"), (255, b"C\xff"),
                                   (256, b"S\x00\x01"), (-129, b"s\x7f\xff"), (65536, b"i\x00\x00\x01\x00")])
def test_append_int_tag_smallest_type(v, enc):
    r = rec_with([])
    O.append_int(r, b"XX", v)
    assert aux(r) == b"XX" + enc


def test_update_string_tag_same_length_in_place():
    r = rec_with([(b"MC", "Z", b"10M"), (b"xx", "Z", b"a")])
    O.update_string(r, b"MC", b"5S5")
    assert aux(r) == b"MCZ5S5\0xxZa\0"


def test_update_string_tag_other_length_spliced():
    r = rec_with([(b"MC", "Z", b"10M"), (b"xx", "Z", b"a")])
    O.update_string(r, b"MC", b"5S95M")
    assert aux(r) == b"MCZ5S95M\0xxZa\0"


def test_update_string_tag_appends_when_absent():
    r = rec_with([(b"xx", "Z", b"a")])
    O.update_string(r, b"MC", b"1M")
    assert aux(r) == b"xxZa\0MCZ1M\0"


@pytest.mark.parametrize("typ,v,enc", [("C", 200, b"s\xc8\x00"), ("i", 5, b"c\x05"), ("I", 70000, b"i\x70\x11\x01\x00"),
                                       ("S", 60000, b"i\x60\xea\x00\x00"), ("s", -5, b"c\xfb")])
def test_normalize_int_tag_to_smallest_signed(typ, v, enc):
    r = rec_with([(b"AS", typ, v), (b"xx", "Z", b"a")])
    O.normalize(r, b"AS")
    assert aux(r) == b"xxZa\0AS" + enc


def test_normalize_leaves_values_past_i32_and_non_integers():
    for tags in ([(b"AS", "I", 3000000000)], [(b"AS", "Z", b"7")], [(b"AS", "f", 1.0)]):
        r = rec_with(tags + [(b"xx", "Z", b"a")])
        before = bytes(r)
        O.normalize(r, b"AS")
        assert bytes(r) == before


def test_reverse_array_and_string_in_place():
    r = rec_with([(b"ad", "Bs", [1, 2, 3]), (b"s1", "Z", b"abc"), (b"s3", "Z", b"AcgN")])
    O.reverse_in_place(r, b"ad", ord("B"), False)
    O.reverse_in_place(r, b"s1", ord("Z"), False)
    O.reverse_in_place(r, b"s3", ord("Z"), True)
    assert aux(r) == b"adBs" + struct.pack("<I3h", 3, 3, 2, 1) + b"s1Zcba\0s3ZNCGT\0"


def test_remove_tag_first_only_and_absent():
    r = rec_with([(b"xx", "Z", b"a"), (b"yy", "i", 1)])
    O.remove_tag(r, b"zz")
    O.remove_tag(r, b"xx")
    assert aux(r) == b"yyi" + struct.pack("<i", 1)


# ---- tests/integration/test_zipper_command.rs, BAM input ------------------------------------------------------

def test_integration_basic_pairs_keep_order_and_tags():
    u, m = [], []
    for i in range(5):
        u += upair(b"read%d" % i, [(b"RX", "Z", b"AACC")])
        m += mpair(b"read%d" % i, 100 + 10 * i, 300 + 10 * i, tags=[(b"AS", "i", 90)])
    recs, stats = run(u, m, remove=["AS"])
    assert [r["name"] for r in recs] == [b"read%d" % (i // 2) for i in range(10)]
    assert all(b"AS" not in r["tags"] and r["tags"][b"RX"] == b"AACC" for r in recs)
    assert stats == [5, 0, 0, 10]


def test_integration_mismatched_names_fail():
    with pytest.raises(ValueError):
        run(upair(b"a"), mpair(b"b", 100, 200))
