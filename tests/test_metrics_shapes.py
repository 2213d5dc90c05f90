"""The metrics shape helpers (tests/metrics_shapes.py) against tests/metrics_oracle.py, and the collector's host
template pass on every record layout (no GPU): bucket-targeted names, the count-only reference, the interval index,
fgb_host_metrics_templates and the ideal-duplex fraction's binomial sum."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgumi_b200 import metrics as M       # noqa: E402
from tests import metrics_oracle as O     # noqa: E402
from tests import metrics_shapes as X     # noqa: E402
from tests import metrics_streams as S    # noqa: E402


def test_names_by_bucket():
    pool = X.NamePool(b"nm")
    for b in range(X.N_FRACTIONS):
        names = pool.take(b, 25)
        assert len(set(names)) == 25
        for nm in names:
            assert O.bucket_of(O.hash_fraction(nm)) == b, nm
        for nm in names[:3]:
            assert M.name_fraction(nm)[2] == b
    # the vectorised hash itself, on names of odd and even lengths
    for n in (1, 2, 7, 12, 31):
        rows = np.random.default_rng(n).integers(32, 127, (40, n)).astype(np.uint8)
        got = X.murmur3_ascii(rows)
        assert [int(h) for h in got] == [O.name_hash(r.tobytes()) for r in rows]
        assert list(X.buckets_of(got)) == [O.bucket_of(O.hash_fraction_of(int(h))) for h in got]
    edge = np.array([-2 ** 31, -(2 ** 31 - 1), 2 ** 31 - 1, 0, 107374182, 107374183, -107374183], np.int64)
    assert list(X.buckets_of(edge)) == [O.bucket_of(O.hash_fraction_of(int(h))) for h in edge]


def _count_tables(recs, duplex, header=S.HEADER):
    return X.CountReference.from_templates(O.templates(header, recs, [])).tables(duplex)


def _three(tables):
    return {k: v for k, v in tables.items() if k in ("family_sizes", "duplex_family_sizes", "yield_metrics")}


def _close(got, exp):
    """Every byte, but the ideal fraction within 1e-12 relative."""
    assert sorted(got) == sorted(exp)
    for name in exp:
        gl, el = got[name].splitlines(), exp[name].splitlines()
        assert len(gl) == len(el), name
        for g, e in zip(gl, el):
            if g != e:
                g, e = g.split("\t"), e.split("\t")
                assert name == "yield_metrics" and g[:-1] == e[:-1], (name, g, e)
                assert abs(float(g[-1]) - float(e[-1])) <= 1e-12 * abs(float(e[-1])), (g, e)


@pytest.mark.parametrize("duplex", [True, False])
@pytest.mark.parametrize("stream", ["random", "random_odd", "big", "boundary"])
def test_count_reference_matches_oracle(stream, duplex):
    recs = {"random": lambda: S.random_stream(1, 300, odd_mi_rate=0.2, suffix_rate=0.85),
            "random_odd": lambda: S.random_stream(12, 200, max_size=12, odd_mi_rate=0.5, suffix_rate=0.5),
            "big": lambda: S.random_stream(3, 40, big_family=70),
            "boundary": lambda: X.boundary_stream(range(0, 20, 3))}[stream]()
    _close(_count_tables(recs, duplex), _three(O.collect(S.HEADER, recs, duplex=duplex)))


def test_count_reference_thresholds():
    recs = S.random_stream(2, 200, max_size=9)
    for opts in (dict(min_ab_reads=3, min_ba_reads=2), dict(min_ab_reads=5, min_ba_reads=5)):
        ref = X.CountReference.from_templates(O.templates(S.HEADER, recs, [])).tables(True, **opts)
        _close(ref, _three(O.collect(S.HEADER, recs, duplex=True, **opts)))
    ref = X.CountReference.from_templates(O.templates(S.HEADER, recs, [])).tables(False, min_reads=3)
    _close(ref, _three(O.collect(S.HEADER, recs, duplex=False, min_reads=3)))


def test_boundary_stream_reaches_every_bound():
    ref = X.CountReference.from_templates(O.templates(S.HEADER, X.boundary_stream(), []))
    for f in range(X.N_FRACTIONS):
        cs, ss, ds, ab, ba, _ = ref.fraction(f)
        for n in (1, 7, 8, 31, 32, 33):
            assert n in set(ss.tolist())
        assert {0, 31, 32, 33} <= set(ds.tolist())
        assert {31, 32, 33} <= set(cs.tolist())
        pairs = set(zip(ab.tolist(), ba.tolist()))
        assert {(7, 0), (7, 7), (8, 0), (8, 7), (8, 8), (31, 31), (32, 1)} <= pairs


def test_overflow_count_worst_case():
    """Families of 8 one-strand templates in bucket 0, four to a group: 20 pair entries per family and 20 CS entries
    per group, 3.125 per template -- the densest the bounds allow, and well inside 6 n + 64."""
    recs = X.worst_case_overflow(64)
    ref = X.CountReference.from_templates(O.templates(S.HEADER, recs, []))
    assert ref.overflow() == 20 * 64 * 4 + 20 * 64
    assert ref.overflow() <= 6 * ref.n + 64


@pytest.mark.parametrize("ivs", [
    [],
    [("chr1", 100, 200)],
    [("chr1", 0, 1000), ("chr1", 10, 20)],                        # nested: the running maximum decides
    [("chr1", 10, 20), ("chr1", 0, 1000), ("chr1", 500, 501)],    # unsorted
    [("chr1", 50, 99), ("chr1", 50, 99), ("chr1", 120, 130)],     # duplicates
    [("chr2", 100, 200), ("chrZ", 0, 10 ** 9)],                   # an absent contig
    [("chr1", -5, 3), ("chr1", 2 ** 31 - 2, 2 ** 31 - 1)],
])
def test_interval_index_matches_oracle(ivs):
    idx = X.IntervalIndex(ivs)
    spans = [(n, s, e) for n in ("chr1", "chr2", "chr3", None) for s in (-1, 0, 1, 19, 20, 21, 99, 100, 101, 199, 200,
                                                                         201, 999, 1000, 1001)
             for e in (s, s + 1, s + 50, s + 1000)]
    for n, s, e in spans:
        assert idx(n, s, e) == O.overlaps(ivs, n, s, e), (n, s, e)
    # touching at both ends: start == e meets, s == end - 1 meets, s == end does not
    for n, s, e in ivs:
        assert X.IntervalIndex(ivs)(n, e, e + 10) == O.overlaps(ivs, n, e, e + 10)
        assert X.IntervalIndex(ivs)(n, s - 10, s + 1) == O.overlaps(ivs, n, s - 10, s + 1)


def test_exome_intervals_index_matches_oracle():
    recs, spans = X.exome_stream(4, 300)
    ivs = X.exome_intervals(5, spans, n=3000)
    idx = X.IntervalIndex(ivs)
    got = [idx(*sp) for sp in spans]
    assert got == [O.overlaps(ivs, *sp) for sp in spans]
    assert 0 < sum(got) < len(got)
    for picard in (False, True):
        text = X.interval_text(ivs, picard)
        assert [tuple(v) for v in O.parse_intervals(text)] == [tuple(v) for v in ivs]
    exp = O.collect(X.HEADER3, recs, intervals=X.interval_text(ivs))
    assert O.collect(X.HEADER3, recs, overlap=idx) == exp


def test_host_templates_every_layout():
    """fgb_host_metrics_templates against O.templates on every layout and name the builder makes."""
    recs = X.layout_stream(X.NamePool(b"L"))
    b, off = S.to_arrays(recs)
    got = X.host_template_array(S.HEADER, b, off)
    exp = list(O.templates(S.HEADER, recs, []))
    runs = [0] + [i for i in range(1, len(recs)) if recs[i][32:32 + recs[i][8]] != recs[i - 1][32:32 + recs[i - 1][8]]]
    assert len(got) == len(runs)
    kept = [(i, t) for i, t in enumerate(got) if t["status"] == 2]
    assert [runs[i] for i, _ in kept] == [e[4] for e in exp]
    for (i, g), e in zip(kept, exp):
        key = (int(g["ref1"]), int(g["start1"]) + 1, bool(g["strand1"]), int(g["ref2"]), int(g["start2"]) + 1,
               bool(g["strand2"]))
        assert key == e[0], (recs[runs[i]][32:40], key, e[0])
        body = bytes(b[int(off[g["r1"]]):int(off[g["r1"] + 1])])
        assert body[g["mi_off"]:g["mi_off"] + g["mi_len"]].decode() == e[1]
        assert body[g["rx_off"]:g["rx_off"] + g["rx_len"]].decode() == e[2]
        assert g["bucket"] == O.bucket_of(e[3])
    skipped = {bytes(recs[runs[i]][32:32 + recs[runs[i]][8] - 1]) for i, t in enumerate(got) if t["status"] == 0}
    assert len(skipped) == 5          # lone, unmapped mate, unmapped R1, tid -1, no CIGAR
    sizes = {len(r) for r in recs}
    assert {65535, 65536, 65541} <= sizes
    assert any(len(r[32:32 + r[8] - 1]) == 254 for r in recs)


@pytest.mark.parametrize("thresholds", [(1, 1), (3, 2), (10, 10), (50, 50), (200, 200), (2500, 2500)])
def test_ideal_fraction_ratio_sum(thresholds):
    """binom_interval_half, restated, against scipy's CDF for families of 2 to 5 000 templates: within the 1e-12
    relative tolerance the collector's yield table is compared with.  The difference of two lgamma-term CDFs it
    replaced was 1.03e-12 off at (200, 200) and 401 templates."""
    a, b = thresholds
    for n in list(range(max(2, a + b - 1), a + b + 40)) + [735, 1000, 2047, 4999, 5000]:
        got, exp = X.ideal_fraction_ratio([n], a, b), O.ideal_fraction([n], a, b)
        assert abs(got - exp) <= 1e-12 * abs(exp) or got == exp == 0.0, (n, got, exp)
    sizes = [20, 64, 400, 401, 1000, 5000]
    got, exp = X.ideal_fraction_ratio(sizes, a, b), O.ideal_fraction(sizes, a, b)
    assert abs(got - exp) <= 1e-12 * abs(exp) or got == exp == 0.0
