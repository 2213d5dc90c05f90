"""tests/metrics_oracle.py pinned to ports of the reference's own tests: src/lib/commands/shared_metrics.rs,
simplex_metrics.rs and duplex_metrics.rs (their #[cfg(test)] modules)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import metrics_oracle as O     # noqa: E402
from tests import metrics_streams as S    # noqa: E402


def _rows(text):
    lines = text.splitlines()
    head = lines[0].split("\t")
    return [dict(zip(head, ln.split("\t"))) for ln in lines[1:]]


@pytest.mark.parametrize("name", ["", "A", "read1", "SRR099966.100", "a much longer read name here"])
def test_hash_fraction_in_unit_range(name):   # shared_metrics.rs:736-746
    assert 0.0 <= O.hash_fraction(name.encode()) <= 1.0


def test_inter_reference_pairs_are_retained():   # shared_metrics.rs:752-772
    recs = S.pair(b"same_1", b"1", b"ACGT-TGCA", 0, 100, 0, 300) + S.pair(b"same_2", b"2", b"ACGT-TGCA", 0, 100, 0, 300) + \
        S.pair(b"inter_1", b"3", b"ACGT-TGCA", 0, 500, 1, 500)
    t = list(O.templates(S.HEADER, recs, []))
    assert [x[1] for x in t] == ["1", "2", "3"]


def test_simplex_family_size_counts():   # simplex_metrics.rs:488-551
    recs = S.pair(b"grp1_mi1_0", b"1/A", b"AAA", pos1=100, pos2=200) + \
        S.pair(b"grp1_mi1_1", b"1/A", b"AAA", pos1=100, pos2=200) + \
        S.pair(b"grp1_mi2_0", b"2/A", b"CCC", pos1=100, pos2=200) + \
        S.pair(b"grp2_mi3_0", b"3/A", b"GGG", pos1=300, pos2=400)
    rows = {int(r["family_size"]): r for r in _rows(O.collect(S.HEADER, recs, duplex=False)["family_sizes"])}
    assert (rows[1]["cs_count"], rows[1]["ss_count"]) == ("1", "2")
    assert (rows[2]["cs_count"], rows[2]["ss_count"]) == ("0", "1")
    assert (rows[3]["cs_count"], rows[3]["ss_count"]) == ("1", "0")


def test_simplex_downsampling_generates_fractions():   # simplex_metrics.rs:554-589
    recs = [r for i in range(50) for r in S.pair(b"read_%d" % i, b"%d/A" % i, b"AAA", pos1=100, pos2=200)]
    rows = _rows(O.collect(S.HEADER, recs, duplex=False)["yield_metrics"])
    assert len(rows) == 20
    for a, b in zip(rows, rows[1:]):
        assert float(b["fraction"]) > float(a["fraction"]) and int(b["ss_families"]) >= int(a["ss_families"])


def test_duplex_counts_umis_once_per_read_pair():   # duplex_metrics.rs:732-785
    recs = S.pair(b"q1", b"1/A", b"AAA-CCC") + S.pair(b"q2", b"1/A", b"AAA-CCC") + S.pair(b"q3", b"1/B", b"CCC-AAA")
    rows = {r["umi"]: r for r in _rows(O.collect(S.HEADER, recs)["umi_counts"])}
    assert rows["AAA"]["raw_observations"] == "3" and rows["CCC"]["raw_observations"] == "3"
    assert rows["AAA"]["unique_observations"] == "1"


def test_duplex_error_corrects_umis():   # duplex_metrics.rs:787-854
    recs = S.pair(b"q1", b"1/A", b"AAA-CCC") + S.pair(b"q2", b"1/A", b"AAA-CCC") + S.pair(b"q3", b"1/A", b"AAT-CCC")
    rows = {r["umi"]: r for r in _rows(O.collect(S.HEADER, recs)["umi_counts"])}
    assert rows["AAA"]["raw_observations"] == "3" and rows["AAA"]["raw_observations_with_errors"] == "1"
    assert "AAT" not in rows


def test_duplex_family_sizes_and_min_reads():   # duplex_metrics.rs:1031-1288
    recs = []
    for i in range(3):
        recs += S.pair(b"a%d" % i, b"1/A", b"AAA-CCC")
    recs += S.pair(b"b0", b"1/B", b"CCC-AAA")
    for i in range(2):
        recs += S.pair(b"c%d" % i, b"2/A", b"GGG-TTT")
    out = O.collect(S.HEADER, recs)
    pairs = {(int(r["ab_size"]), int(r["ba_size"])): int(r["count"]) for r in _rows(out["duplex_family_sizes"])}
    assert pairs == {(3, 1): 1, (2, 0): 1}
    full = _rows(out["yield_metrics"])[-1]
    assert (full["ds_families"], full["ds_duplexes"], full["ss_families"]) == ("2", "1", "3")
    full = _rows(O.collect(S.HEADER, recs, min_ab_reads=3, min_ba_reads=2)["yield_metrics"])[-1]
    assert full["ds_duplexes"] == "0"


def test_only_inserts_overlapping_intervals():   # duplex_metrics.rs:1290-1422, 1832-1976
    recs = S.pair(b"in", b"1/A", b"AAA-CCC", pos1=100, pos2=300) + S.pair(b"out", b"2/A", b"AAA-CCC", pos1=5000,
                                                                           pos2=5200)
    for iv in (b"chr1\t150\t250\n", b"@HD\tVN:1.6\nchr1\t151\t250\t+\tx\n"):
        full = _rows(O.collect(S.HEADER, recs, intervals=iv)["yield_metrics"])[-1]
        assert full["read_pairs"] == "1"


def test_expected_duplex_umi_fraction():   # duplex_metrics.rs:1485-1604
    recs = S.pair(b"q1", b"1/A", b"AAA-CCC") + S.pair(b"q2", b"1/B", b"CCC-AAA") + \
        S.pair(b"q3", b"2/A", b"AAA-GGG", pos1=700, pos2=900)
    out = O.collect(S.HEADER, recs, duplex_umi_counts=True)
    single = {r["umi"]: float(r["fraction_unique_observations"]) for r in _rows(out["umi_counts"])}
    for r in _rows(out["duplex_umi_counts"]):
        a, b = r["umi"].split("-")
        assert float(r["fraction_unique_observations_expected"]) == single[a] * single[b]


def test_reject_consensus_input():   # duplex_metrics.rs:1606-1672, simplex_metrics.rs:603-629
    recs = S.pair(b"read1", b"1", b"A", r1_tags=[(b"cD", "i", 5)])
    with pytest.raises(O.MetricsOracleError):
        O.collect(S.HEADER, recs)


def test_min_ab_must_not_be_below_min_ba():   # duplex_metrics.rs:1711-1727
    with pytest.raises(ValueError):
        O.collect(S.HEADER, [], min_ab_reads=1, min_ba_reads=2)


def test_empty_umi_components():   # duplex_metrics.rs:1978-2040
    recs = S.pair(b"q1", b"1/A", b"AAA-") + S.pair(b"q2", b"1/A", b"AAA-CCC")
    rows = {r["umi"]: r for r in _rows(O.collect(S.HEADER, recs)["umi_counts"])}
    assert rows["AAA"]["raw_observations"] == "1"
