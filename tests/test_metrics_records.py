"""The metrics collector's host exports against tests/metrics_oracle.py (no GPU): the template pass, names and
buckets, the interval parser, the float text, and the planning-only collector."""
import ctypes as C
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgumi_b200 import lib as L           # noqa: E402
from fgumi_b200 import metrics as M       # noqa: E402
from tests import metrics_oracle as O     # noqa: E402
from tests import metrics_streams as S    # noqa: E402


def test_struct_sizes():
    lib = L.load()
    assert lib.fgb_struct_size(15) == C.sizeof(L.FgbMetricsOptions)
    assert lib.fgb_struct_size(16) == C.sizeof(L.FgbMetricsTemplate) == 64


@pytest.mark.parametrize("name,expected", [
    ("", 142_593_372), ("A", 309_601_938), ("AB", 1_297_118_606), ("ABC", 417_488_640), ("read1", -958_943_510),
    ("read2", 1_466_959_157), ("read10", -87_319_652), ("SRR099966.100", -1_840_920_289),
    ("M00517:73:000000000-A5AEH:1:1101:15541:1541", 1_482_717_766),
    ("NB500947:HT3JMBGX2:1:11101:19204:10048", -1_636_484_024)])
def test_murmur3_htsjdk_vectors(name, expected):   # shared_metrics.rs:717-732
    assert M.name_fraction(name.encode())[0] == expected
    assert O.name_hash(name.encode()) == expected


@pytest.mark.parametrize("name", [b"r\xc3\xa9ad", b"\xff\xfe", b"a\xe2\x82", b"\xf0\x9f\x98\x80x", b"\xed\xa0\x80",
                                  b"\xc0\xaf", b"q\xf4\x90\x80\x80", "名前".encode()])
def test_non_ascii_names(name):
    h, f, b = M.name_fraction(name)
    assert h == O.name_hash(name)
    assert f == O.hash_fraction_of(h)
    assert b == O.bucket_of(f)


def test_bucket_boundaries():
    imax = 2 ** 31 - 1
    hashes = [-2 ** 31, -imax, imax, 0, 1, -1]
    for fr in O.FRACTIONS:
        c = int(fr * imax)
        hashes += [c - 1, c, c + 1, -c, -(c + 1)]
    for h in hashes:
        h = max(-2 ** 31, min(imax, h))
        assert M.bucket(h) == O.bucket_of(O.hash_fraction_of(h)), h
    assert M.bucket(-2 ** 31) == 0          # wrapping_abs keeps i32::MIN: just below -1
    assert O.hash_fraction_of(-2 ** 31) < -1


def test_interval_parser_both_formats():
    bed = b"# comment\nchr1\t100\t200\tname\n\nchr2\t5\t6\n"
    assert M.parse_intervals(bed) == O.parse_intervals(bed) == [("chr1", 100, 200), ("chr2", 5, 6)]
    il = b"@HD\tVN:1.6\n@SQ\tSN:chr1\tLN:1000\nchr1\t101\t200\t+\tt1\n"
    assert M.parse_intervals(il) == O.parse_intervals(il) == [("chr1", 100, 200)]
    for bad in (b"chr1\t100\n", b"chr1\tx\t5\n", b"chr1\t1\t99999999999\n"):
        with pytest.raises(ValueError):
            M.parse_intervals(bad)
        with pytest.raises(ValueError):
            O.parse_intervals(bad)


@pytest.mark.parametrize("v", [0.0, 1.0, 0.5, 0.05, 0.1, 0.15, 1 / 3, 2 / 3, 1e-4, 1.5e-4, 1e-5, 9.99e-5, 1e-6,
                               1.25e-6, 1e-7, 123.0, 1e15, 9999999999999998.0, 1e16, 1.5e16, 1e17, 1e-300, 5e-324,
                               1.7976931348623157e308, 0.000123456789, 12345.678])
def test_float_text(v):
    assert M.format_float(v) == O.fmt_float(v)


def test_float_text_known():
    assert [M.format_float(v) for v in (1.0, 0.00001, 1e-6, 0.0, 1e16, 1e15)] == \
        ["1.0", "0.00001", "1e-6", "0.0", "1e16", "1000000000000000.0"]


def _expected_templates(records, intervals=None):
    ivs = O.parse_intervals(intervals) if intervals else []
    return list(O.templates(S.HEADER, records, ivs))


def test_host_templates_against_oracle():
    recs = []
    recs += S.pair(b"a1", b"1/A", b"AAA-CCC")
    recs += S.pair(b"a2", b"1/B", b"CCC-AAA", pos1=300, pos2=100)          # mates swapped: the same key
    recs += S.pair(b"a3", b"05/A", b"AAA-CCC", cigar="3S17M")
    recs += S.pair(b"a4", b"x", b"AAA", ref1=0, pos1=500, ref2=1, pos2=500)  # inter-contig
    recs += S.pair(b"na\xc3\xafve", b"7", b"G-T")
    recs += [S.pair(b"single", b"1", b"A")[0]]                              # one record: skipped
    b, off = S.to_arrays(recs)
    got = M.host_templates(S.HEADER, b, off)
    exp = _expected_templates(recs)
    kept = [t for t in got if t["status"] == L.FGB_OK + 2]
    assert len(kept) == len(exp) == 5
    for g, e in zip(kept, exp):
        key = (g["ref1"], g["start1"] + 1, bool(g["strand1"]), g["ref2"], g["start2"] + 1, bool(g["strand2"]))
        assert key == e[0]
        assert g["bucket"] == O.bucket_of(e[3])
    assert got[-1]["status"] == 0
    assert [t["mi_canonical"] for t in kept] == [1, 1, 0, 0, 1]
    assert [t["mi_kind"] for t in kept] == [1, 2, 1, 0, 0]
    assert kept[4]["name_ascii"] == 0


def test_host_templates_intervals():
    recs = S.pair(b"in", b"1/A", b"A-C", pos1=100, pos2=300) + S.pair(b"out", b"2/A", b"A-C", pos1=5000, pos2=5200) + \
        S.pair(b"x", b"3/A", b"A-C", ref1=1, pos1=100, ref2=0, pos2=300)
    b, off = S.to_arrays(recs)
    for iv in (b"chr1\t310\t400\n", b"chr1\t319\t400\n", b"@SQ\tSN:chr1\tLN:1\nchr1\t320\t400\t+\tx\n",
               b"chr2\t0\t100\nchrX\t0\t1000000\n"):
        got = [t["status"] for t in M.host_templates(S.HEADER, b, off, iv)]
        exp_names = {e[4] for e in _expected_templates(recs, iv)}
        assert got == [2 if 2 * k in exp_names else 1 for k in range(3)], iv


def test_host_templates_errors():
    recs = S.pair(b"a", b"1/A", b"A-C") + S.pair(b"b", None, b"A-C") + S.pair(b"c", b"3", None) + \
        S.pair(b"d", b"\xff", b"A-C") + S.pair(b"e", b"1", b"\xc3")
    b, off = S.to_arrays(recs)
    assert [t["status"] for t in M.host_templates(S.HEADER, b, off)] == [2, 3, 5, 4, 6]
    dup = S.pair(b"a", b"1", b"A-C") + [S.pair(b"a", b"1", b"A-C")[0]]
    b, off = S.to_arrays(dup)
    with pytest.raises(M.MetricsError) as e:
        M.host_templates(S.HEADER, b, off)
    assert e.value.bad_record == 2


def test_planning_only_collector_refuses():
    m = M.MetricsCollector(S.HEADER, duplex=True, device=L.FGB_DEVICE_NONE)
    b, off = S.to_arrays(S.pair(b"a", b"1/A", b"A-C"))
    with pytest.raises(M.MetricsError) as e:
        m.add_records(b, off)
    assert e.value.status == L.FGB_ERR_NO_DEVICE
    with pytest.raises(M.MetricsError) as e:
        m.finish()
    assert e.value.status == L.FGB_ERR_NO_DEVICE


def test_create_refuses_bad_options():
    with pytest.raises(L.FgbError):
        M.MetricsCollector(S.HEADER, duplex=True, device=L.FGB_DEVICE_NONE, min_ab_reads=1, min_ba_reads=2)
    with pytest.raises(L.FgbError):
        M.MetricsCollector(S.HEADER, duplex=True, device=L.FGB_DEVICE_NONE, intervals=b"chr1\t1\n")
