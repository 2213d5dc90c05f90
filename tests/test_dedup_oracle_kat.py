"""tests/dedup_oracle.py pinned by ports of the reference's own `dedup` tests (dedup.rs:1218-2770) and of the three
scenarios of tests/integration/test_dedup_command.rs.  Pure Python: no library, no device."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import group_oracle as G     # noqa: E402
from oracle import umi_oracle as U       # noqa: E402
from tests import dedup_oracle as D      # noqa: E402
from tests.bam_builder import make_record, parse_records   # noqa: E402

PF = 0x1 | 0x40


def tpl(name, quals, r2_quals=None):
    """create_test_template / create_paired_test_template (dedup.rs:1218-1268)."""
    recs = [make_record(name, PF if r2_quals is None else PF | 0x20, 0, 99, 60, "4M", seq=b"ACGT", quals=quals)]
    if r2_quals is not None:
        recs.append(make_record(name, 0x1 | 0x80 | 0x10, 0, 199, 60, "4M", seq=b"ACGT", quals=r2_quals))
    return D.build_templates(recs)[0]


# ---- score_template (dedup.rs:1228-1306, 2396-2450) ----------------------------------------------------------------
@pytest.mark.parametrize("q1,q2,want", [
    ([20] * 4, None, 60), ([10] * 4, None, 40), ([10] * 4, [10] * 4, 80), ([40] * 4, [40] * 4, 120),
    ([5] * 4, [15] * 4, 80), ([10, 20, 5, 30], [8, 12, 25, 3], 10 + 15 + 5 + 15 + 8 + 12 + 15 + 3)])
def test_score_template(q1, q2, want):
    assert D.score_template(tpl(b"q1", q1, q2)) == want


def test_score_ignores_secondary_and_supplementary():
    recs = [make_record(b"a", PF, 0, 99, 60, "4M", seq=b"ACGT", quals=[30] * 4),
            make_record(b"a", PF | 0x800, 0, 500, 60, "4M", seq=b"ACGT", quals=[30] * 4)]
    assert D.score_template(D.build_templates(recs)[0]) == 60


def test_score_clamped_at_record_end():
    r = make_record(b"a", PF, 0, 99, 60, "4M", seq=b"ACGT", quals=[30] * 4)
    assert D.read_score(r[:-2]) == 30 and D.read_score(r[:32]) == 0


# ---- mark_duplicates_in_family (dedup.rs:1342-1598) -----------------------------------------------------------------
@pytest.mark.parametrize("scores,keep", [
    ([], 0), ([40], 0), ([60, 20], 0), ([20, 60], 1), ([60, 40, 20], 0), ([20, 60, 40], 1), ([20, 40, 60], 2),
    ([20, 60, 40, 32], 1), ([40, 40], 0), ([40, 40, 40], 0), ([20, 40, 40], 1), ([40] * 4, 0), ([20, 32, 40, 40], 2)])
def test_mark_duplicates_representative(scores, keep):
    assert D.representative(scores) == keep
    if scores:   # the rule the library applies: the first template with the highest score
        assert keep == scores.index(max(scores))


def test_mark_duplicates_counts_reads_and_templates():
    recs = []
    for i, q in enumerate(([15] * 4, [5] * 4, [10] * 4)):
        recs.append(make_record(b"q%d" % i, 0, 0, 99, 60, "4M", seq=b"ACGT", quals=q, tags=[(b"RX", "Z", b"AC")]))
    out, d = D.dedup_stream(recs, b"", D.Config(strategy=U.IDENTITY, edits=0))
    st = dict(zip(D.STATS, d.stats))
    assert st["unique_templates"] == 1 and st["duplicate_templates"] == 2 and st["duplicate_reads"] == 2
    assert [r["flags"] & 0x400 for r in parse_records(out)] == [0, 0x400, 0x400]


# ---- filter_template (dedup.rs:1601-1750, 2078-2150, 2262-2330, 2605-2770) -------------------------------------------
def frag(name=b"a", umi=b"ACGTACGT", mapq=60, flags=PF, tags=(), seq=b"ACGT"):
    t = ([(b"RX", "Z", umi)] if umi is not None else []) + list(tags)
    return make_record(name, flags, 0, 99, mapq, "4M", seq=seq, tags=t)


def filt(recs, **kw):
    cfg = D.Config(**dict(dict(min_map_q=20), **kw))
    m = [0] * 6
    ok = D.filter_template(D.build_templates(recs)[0], cfg, m)
    return ok, m


def test_filter_accepts_valid():
    assert filt([frag(flags=PF | 0x8)]) == (True, [1, 1, 0, 0, 0, 0])


def test_filter_low_mapq():
    assert filt([frag(mapq=10, flags=PF | 0x8)]) == (False, [1, 0, 0, 1, 0, 0])


def test_filter_n_in_umi():
    assert filt([frag(umi=b"ACNTACGT", flags=PF | 0x8)])[1][4] == 1


def test_filter_short_umi():
    assert filt([frag(umi=b"ACG", flags=PF | 0x8)], min_umi_length=5)[1][5] == 1


def test_filter_missing_umi():
    assert filt([frag(umi=None, flags=PF | 0x8)]) == (False, [1, 0, 0, 1, 0, 0])


def test_filter_qc_fail():
    assert filt([frag(flags=PF | 0x8 | 0x200)])[1][2] == 1
    assert filt([frag(flags=PF | 0x8 | 0x200)], include_non_pf=True)[0]


def test_filter_unmapped_always_rejected():
    r = make_record(b"a", PF | 0x4 | 0x8, -1, -1, 0, "", seq=b"ACGT", tags=[(b"RX", "Z", b"ACGT")])
    assert filt([r], min_map_q=0) == (False, [1, 0, 0, 1, 0, 0])


def test_filter_paired_r2_cases():
    def pr(umi2=b"AC-GT", mapq2=60):
        return [make_record(b"a", PF | 0x20, 0, 99, 60, "4M", 0, 199, seq=b"ACGT", tags=[(b"RX", "Z", b"AC-GT"),
                                                                                       (b"MQ", "i", mapq2)]),
                make_record(b"a", 0x1 | 0x80 | 0x10, 0, 199, mapq2, "4M", 0, 99, seq=b"ACGT",
                            tags=[(b"RX", "Z", umi2), (b"MQ", "i", 60)])]
    assert filt(pr()) == (True, [1, 1, 0, 0, 0, 0])           # counted once per template
    assert filt(pr(mapq2=10)) == (False, [1, 0, 0, 1, 0, 0])
    assert filt(pr(umi2=b"AN-GT"))[1][4] == 1
    m = [0] * 6
    assert not D.filter_template(D.Template(b"x", None, None, []), D.Config(), m) and m == [1, 0, 0, 1, 0, 0]


def test_filter_truncated_aux_rejected():
    r = frag(flags=PF | 0x8)
    assert filt([r[:-4]])[1][3] == 1   # the UMI's NUL is cut off: no UMI


@pytest.mark.parametrize("typ,val,ok", [("c", 10, False), ("c", -1, False), ("C", 30, True), ("s", 10, False),
                                        ("S", 300, True), ("i", 300, True), ("i", 10, False), ("I", 20, True)])
def test_filter_mate_mq_signed_any_integer_type(typ, val, ok):
    r = frag(flags=0x1 | 0x40, tags=[(b"MQ", typ, val)])
    assert filt([r])[0] is ok


def test_filter_mq_minus_one_fails_at_zero_and_float_mq_is_ignored():
    assert not filt([frag(flags=0x1 | 0x40, tags=[(b"MQ", "c", -1)])], min_map_q=0)[0]
    assert filt([frag(flags=0x1 | 0x40, tags=[(b"MQ", "f", 1.0)])])[0]


@pytest.mark.parametrize("umi", [None, b"ACNT", b"AC"])
def test_filter_no_umi_mode_skips_umi_checks(umi):
    assert filt([frag(umi=umi, flags=PF | 0x8)], no_umi=True, min_umi_length=4)[0]


# ---- umi_for_read, orientation, is_r1_earlier, truncate_umis (dedup.rs:1754-2030) ------------------------------------
def test_umi_for_read():
    assert U.umi_for_read(b"ACGT", True, U.IDENTITY, U.MAPPED, 0) == b"ACGT"
    assert U.umi_for_read(b"acgt", True, U.ADJACENCY, U.MAPPED, 1) == b"ACGT"
    assert U.umi_for_read(b"AAAA-CCCC", True, U.PAIRED, U.MAPPED, 1) == b"aa:AAAA-bb:CCCC"
    assert U.umi_for_read(b"AAAA-CCCC", False, U.PAIRED, U.MAPPED, 1) == b"bb:AAAA-aa:CCCC"
    with pytest.raises(U.UmiError):
        U.umi_for_read(b"AAAACCCC", True, U.PAIRED, U.MAPPED, 1)


def test_pair_orientation():
    f = make_record(b"a", PF, 0, 99, 60, "4M", seq=b"ACGT")
    r = make_record(b"a", PF | 0x10, 0, 99, 60, "4M", seq=b"ACGT")
    assert G.orientation(f, f) == (True, True) and G.orientation(r, f) == (False, True)
    assert G.orientation(r, r) == (False, False) and G.orientation(None, r) == (True, False)


def test_is_r1_earlier():
    a = make_record(b"a", PF, 0, 99, 60, "4M", seq=b"ACGT")
    b = make_record(b"a", 0x81, 0, 199, 60, "4M", seq=b"ACGT")
    c = make_record(b"a", 0x81, 1, 9, 60, "4M", seq=b"ACGT")
    assert G.is_r1_earlier(a, b) and not G.is_r1_earlier(b, a) and G.is_r1_earlier(a, a) and G.is_r1_earlier(a, c)


def test_truncate_umis():
    assert U.truncate_umis([b"ACGTAC", b"ACGTTT"], None) == [b"ACGTAC", b"ACGTTT"]
    assert U.truncate_umis([b"ACGTAC", b"ACGTTT"], 4) == [b"ACGT", b"ACGT"]
    with pytest.raises(U.UmiError):
        U.truncate_umis([b"ACG", b"ACGTTT"], 4)


# ---- metric arithmetic (dedup.rs:1308-1340, 2151-2260) --------------------------------------------------------------
def test_metrics_arithmetic():
    s = [0] * len(D.STATS)
    assert D.dedup_metrics(s)["duplicate_rate"] == 0.0
    s[0], s[1], s[2] = 100, 25, 75
    assert D.dedup_metrics(s)["duplicate_rate"] == 0.75
    s[0], s[1], s[2] = 4, 0, 4
    assert D.dedup_metrics(s)["duplicate_rate"] == 1.0
    assert list(D.dedup_metrics(s)) == ["total_templates", "unique_templates", "duplicate_templates", "duplicate_rate",
                                        "total_reads", "unique_reads", "duplicate_reads", "secondary_reads",
                                        "supplementary_reads", "missing_tc_tag"]


# ---- Template::from_records and position grouping with secondary / supplementary records ---------------------------
def test_template_record_order_and_two_primaries():
    p1 = make_record(b"a", PF, 0, 99, 60, "4M", seq=b"ACGT")
    p2 = make_record(b"a", 0x81, 0, 199, 60, "4M", seq=b"ACGT")
    s1 = [make_record(b"a", PF | 0x800, 0, 300 + i, 60, "4M", seq=b"ACGT") for i in range(2)]
    s2 = [make_record(b"a", 0x81 | 0x100, 0, 400 + i, 60, "4M", seq=b"ACGT") for i in range(2)]
    both = make_record(b"a", PF | 0x900, 0, 500, 60, "4M", seq=b"ACGT")   # secondary wins
    t = D.build_templates([s2[0], s1[0], p2, both, s1[1], p1, s2[1]])[0]
    assert t.records == [p1, p2, s1[1], s1[0], both, s2[1], s2[0]]
    with pytest.raises(D.DedupError):
        D.build_templates([p1, p1])


def test_position_grouping_keeps_secondaries():
    def pr(name, pos):
        return [
            make_record(name, PF | 0x20, 0, pos, 60, "4M", 0, pos + 100, seq=b"ACGT", tags=[(b"MC", "Z", b"4M")]),
            make_record(name, 0x81 | 0x10, 0, pos + 100, 60, "4M", 0, pos, seq=b"ACGT", tags=[(b"MC", "Z", b"4M")])]
    sup = lambda name: make_record(name, PF | 0x800, 0, 5000, 60, "4M", seq=b"ACGT")   # noqa: E731
    recs = [sup(b"z")] + [sup(b"y")] + pr(b"a", 100) + [sup(b"a")] + [sup(b"b")] + pr(b"b", 100) + pr(b"c", 900)
    keep, begin = D.group_by_position(recs)
    # z and y share the default key; a's supplementary continues a; b's leading supplementary opens a default-key
    # group that b's primaries (a new key, a continued QNAME) join
    assert keep == [1] * len(recs) and begin == [0, 2, 5, 8, 10]


# ---- tests/integration/test_dedup_command.rs ------------------------------------------------------------------------
def dup_group(base, umi, count, start):
    out = []
    for i in range(count):
        name = b"%s_%d" % (base, i)
        t = [(b"RX", "Z", umi), (b"MC", "Z", b"8M")]
        out.append(make_record(name, 0x1 | 0x40, 0, start - 1, 60, "8M", 0, start + 99, 108, b"ACGTACGT", [30] * 8, t))
        out.append(make_record(name, 0x1 | 0x80 | 0x10, 0, start + 99, 60, "8M", 0, start - 1, -108, b"ACGTACGT",
                               [30] * 8, t))
    return out


def test_command_basic_and_remove():
    recs = dup_group(b"dup1", b"ACGTACGT", 3, 100) + dup_group(b"dup2", b"TGCATGCA", 2, 500)
    out, d = D.dedup_stream(recs, b"", D.Config())
    assert len(parse_records(out)) == 10
    assert sum(1 for r in parse_records(out) if r["flags"] & 0x400) == 6
    out, d = D.dedup_stream(recs, b"", D.Config(remove_duplicates=True))
    assert 2 <= len(parse_records(out)) < 10 and len(parse_records(out)) == 4


def test_command_no_umi_pileup():
    recs = []
    for i in range(5000):
        name = b"read_%05d" % i
        recs.append(make_record(name, 0x1 | 0x2 | 0x40 | 0x20, 0, 99, 60, "8M", 0, 199, 108, b"ACGTACGT", [30] * 8,
                                [(b"MC", "Z", b"8M")]))
        recs.append(make_record(name, 0x1 | 0x2 | 0x80 | 0x10, 0, 199, 60, "8M", 0, 99, -108, b"ACGTACGT", [30] * 8,
                                [(b"MC", "Z", b"8M")]))
    out, d = D.dedup_stream(recs, b"", D.Config(no_umi=True))
    parsed = parse_records(out)
    assert len(parsed) == 10000
    assert len({r["name"] for r in parsed if not r["flags"] & 0x400}) == 1
    assert sum(1 for r in parsed if not r["flags"] & 0x400) == 2
    assert {r["tags"][b"MI"] for r in parsed} == {b"0"}
