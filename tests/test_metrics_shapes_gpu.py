"""The device metrics collector at the shapes users collect, against tests/metrics_oracle.py (and, at bench size, the
count-only reference of tests/metrics_shapes.py): every shared-histogram boundary in every fraction, the worst-case
overflow list, wide and colliding MI keys, group output of ~50 k templates across thread counts, staging and call
cuts, one huge family and one huge group, exome-size interval lists and every template layout.  Every case compares
each table's text (test_metrics_records_gpu._compare's rule) and stats() with counts taken from the oracle's templates.

The oracle of the large streams is computed once per module, in worker processes, while the device cases run."""
import multiprocessing as mp
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgumi_b200 import metrics as M                   # noqa: E402
from tests import metrics_oracle as O                 # noqa: E402
from tests import metrics_shapes as X                 # noqa: E402
from tests import metrics_streams as S                # noqa: E402
from tests.test_metrics_records_gpu import _compare   # noqa: E402

pytestmark = pytest.mark.gpu
STAT_KEYS = ("kept", "outside", "groups", "ds_families", "overflow")


def _run(header, records, duplex=True, cuts=None, calls=1, **opts):
    """The collector over `records`, cut into calls at the given record indices (QNAME-run starts) or evenly."""
    m = M.MetricsCollector(header, duplex=duplex, device=0, **opts)
    b, off = S.to_arrays(records)
    if cuts is None:
        starts = _run_starts(records)
        cuts = [starts[int(k)] for k in np.linspace(0, len(starts), calls + 1)[1:-1].astype(int)]
    bounds = [0] + sorted(set(cuts)) + [len(records)]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        if hi > lo:
            m.add_records(b[int(off[lo]):int(off[hi])], off[lo:hi + 1] - off[lo])
    return m.finish(), m


def _run_starts(records):
    return [i for i in range(len(records)) if i == 0 or records[i][32:32 + records[i][8]] !=
            records[i - 1][32:32 + records[i - 1][8]]]


def _stats(m):
    return {k: m.stats()[k] for k in STAT_KEYS}


# ---- the large streams and their oracle results, computed once ----------------------------------------------------
def group_output(n_sites, seed, strategy, **kw):
    from fgumi_b200 import bamio, group, synth
    hdr, b, off = synth.mapped_templates(n_sites, seed=seed, **kw)
    keep, begin = group.group_by_position(b, off, hdr)
    kb, koff = group.compact(b, off, keep)
    gr = group.ReadGrouper(0, strategy=strategy, edits=1, n_threads=16)
    gr.add_groups(kb, koff, begin)
    bodies, rec_off = bamio.split_stream(gr.flush())
    return hdr, [bytes(bodies[int(rec_off[i]):int(rec_off[i + 1])]) for i in range(len(rec_off) - 1)]


SCALE_KW = dict(molecules=2, mean_family=2.0, secondary_rate=0.05, unmapped_mate_rate=0.05, cross_contig_rate=0.05,
                reverse_rate=0.3, amplicon_molecules=300)


def huge_stream():
    """One DS family of 20 000 templates in one group, then one group of 60 000 templates over 1 500 families."""
    sb = X.StreamBuilder(b"h")
    rng = np.random.default_rng(3)
    sb.group([X.fam(b"1", 10_000, 10_000, bucket=rng.integers(0, 20, 20_000).tolist())])
    sb.group([X.fam(b"%d" % (k + 2), 20, 19, 1, bucket=rng.integers(0, 20, 40).tolist()) for k in range(1_500)])
    return sb.records


@pytest.fixture(scope="module")
def large():
    """(streams {name: (header, records)}, oracle jobs {(name, duplex): async tables}, a stats cache): the oracle
    runs in spawned workers (it dominates the file's time) and each result is awaited where a case first needs it."""
    streams = {
        "duplex_group": group_output(15_000, 7, "paired", paired_umis=True, **SCALE_KW),
        "simplex_group": group_output(15_000, 8, "adjacency", **SCALE_KW),
        "random": (S.HEADER, S.random_stream(21, 4_000, odd_mi_rate=0.2, suffix_rate=0.85)),
        "huge": (S.HEADER, huge_stream()),
    }
    pool = mp.get_context("spawn").Pool(min(8, os.cpu_count() or 1))
    jobs = {}
    for name, (hdr, recs) in streams.items():
        for duplex in (True, False):
            if name == "duplex_group" and not duplex or name == "simplex_group" and duplex:
                continue
            opts = dict(duplex_umi_counts=True) if duplex else {}
            jobs[name, duplex] = pool.apply_async(X.oracle_job, ((hdr, recs, duplex, opts),))
    pool.close()
    yield streams, jobs, {}
    pool.terminate()
    pool.join()


def _expect(large, name, duplex):
    return large[1][name, duplex].get(timeout=1800)


def _expect_stats(large, name):
    """X.expected_stats of a large stream, once."""
    cache = large[2]
    if name not in cache:
        cache[name] = X.expected_stats(*large[0][name])
    return cache[name]


# ---- 1. every histogram boundary in every fraction ----------------------------------------------------------------
@pytest.mark.parametrize("duplex", [True, False])
def test_every_boundary_in_every_fraction(duplex):
    recs = X.boundary_stream()
    opts = dict(duplex_umi_counts=True) if duplex else {}
    got, m = _run(S.HEADER, recs, duplex, n_threads=4, **opts)
    _compare(got, O.collect(S.HEADER, recs, duplex=duplex, **opts))
    exp = X.expected_stats(S.HEADER, recs)
    assert _stats(m) == exp
    # sizes >= kSmall and pairs with ab >= kPair take the overflow list (host/metrics_device.h); the tables alone cannot
    # tell which path a size took
    assert exp["overflow"] > 0


# ---- 2. the worst-case overflow list ------------------------------------------------------------------------------
@pytest.mark.parametrize("duplex", [True, False])
def test_worst_case_overflow(duplex):
    recs = X.worst_case_overflow(1_600)     # 51 200 templates, 3.125 overflow entries each
    got, m = _run(S.HEADER, recs, duplex)
    ref = X.CountReference.from_templates(O.templates(S.HEADER, recs, []))
    _compare({k: v for k, v in got.items() if k in ("family_sizes", "duplex_family_sizes", "yield_metrics")},
             ref.tables(duplex))
    n = m.stats()["kept"]
    assert n == ref.n == 51_200
    assert m.stats()["overflow"] == ref.overflow() == 20 * 6_400 + 20 * 1_600
    assert m.stats()["overflow"] <= 6 * n + 64


# ---- 3. wide and colliding MI keys --------------------------------------------------------------------------------
def wide_mi_stream():
    sb = X.StreamBuilder(b"m")
    f = X.fam
    b19 = [k % 20 for k in range(40)]
    sb.group([f(b"x0", 3, 1, bucket=b19[:4]), f(b"0", 3, 2, bucket=b19[4:9])])   # dictionary id 0 beside 0: bit 63
    sb.group([f(b"1", 3, 1, bucket=0), f(b"4294967297", 3, 2, bucket=b19[:5])])   # equal low 32 bits
    sb.group([f(b"999999999999999999", 2, 2, bucket=1), f(b"1000000000000000000", 3, bucket=2),
              f(b"18446744073709551617", 2, 1, bucket=3)])
    sb.group([f(b"5", n_0=2, bucket=4), f(b"05", n_0=2, bucket=5), f(b"5", 2, 1, bucket=6)])
    sb.group([f(b"", 2, 2, 1, bucket=b19[:5])])                                      # empty bases: /A, /B and ""
    sb.group([f(b"5/A", 2, 1, bucket=7), f(b"5/a", n_0=2, bucket=8), f(b"5", 1, bucket=9)])
    for _ in range(3):                                                              # one base in adjacent groups
        sb.group([f(b"77", 2, 1, bucket=b19[:3])])
    sb.group([f(b"78", 1, 1, bucket=0), f(b"77", 1, bucket=0)])
    for k in range(30):                                                             # distant reuse, and across calls
        sb.group([f(b"%d" % (100 + k), 1, 1, bucket=k % 20)])
    sb.group([f(b"1", 2, 2, bucket=10), f(b"5", 1, 1, bucket=11), f(b"x0", 1, 1, bucket=12)])
    sb.group([f(b"1", 2, bucket=13)])
    return sb.records


@pytest.mark.parametrize("calls", [1, 3])
@pytest.mark.parametrize("duplex", [True, False])
def test_wide_and_colliding_mi_keys(duplex, calls):
    recs = wide_mi_stream()
    opts = dict(duplex_umi_counts=True) if duplex else {}
    got, m = _run(S.HEADER, recs, duplex, calls=calls, **opts)
    _compare(got, O.collect(S.HEADER, recs, duplex=duplex, **opts))
    assert _stats(m) == X.expected_stats(S.HEADER, recs)


# ---- 4. group output and random streams of 40-60 k templates against the full oracle --------------------------------
@pytest.mark.parametrize("name,duplex", [("duplex_group", True), ("simplex_group", False), ("random", True),
                                         ("random", False)])
def test_scale_against_oracle(large, name, duplex):
    hdr, recs = large[0][name]
    opts = dict(duplex_umi_counts=True) if duplex else {}
    texts = []
    for threads in (1, 16):
        got, m = _run(hdr, recs, duplex, n_threads=threads, **opts)
        texts.append(got)
    assert texts[0] == texts[1]
    assert m.stats()["kept"] > 40_000
    _compare(texts[0], _expect(large, name, duplex))
    assert _stats(m) == _expect_stats(large, name)


def _cuts_inside(hdr, records, calls):
    """calls - 1 cut points at template starts, alternately inside a coordinate group and inside a DS family."""
    tpls = list(O.templates(hdr, records, []))
    inside_group = [i for i in range(1, len(tpls)) if tpls[i][0] == tpls[i - 1][0] and
                    O._base(tpls[i][1])[0] != O._base(tpls[i - 1][1])[0]]
    inside_fam = [i for i in range(1, len(tpls)) if tpls[i][0] == tpls[i - 1][0] and
                  O._base(tpls[i][1])[0] == O._base(tpls[i - 1][1])[0]]
    cuts = []
    for k in range(calls - 1):
        pick = inside_fam if k % 2 else inside_group
        cuts.append(tpls[pick[(k + 1) * len(pick) // calls]][4])
    return cuts


@pytest.mark.parametrize("calls", [1, 7, 101])
@pytest.mark.parametrize("name,duplex", [("duplex_group", True), ("simplex_group", False)])
def test_scale_staged_and_cut(large, name, duplex, calls, monkeypatch):
    hdr, recs = large[0][name]
    opts = dict(duplex_umi_counts=True) if duplex else {}
    monkeypatch.setenv("FGB_METRICS_STAGE_BYTES", "4096")
    got, m = _run(hdr, recs, duplex, cuts=_cuts_inside(hdr, recs, calls), device_bytes=4 << 20, n_threads=4, **opts)
    assert m.stats()["runs"] >= max(calls, 4)
    _compare(got, _expect(large, name, duplex))


# ---- 5. the bench workload (at 70 000 of its 200 000 sites) against the count-only reference ---------------------------------------------------------------
def test_bench_size_counts():
    from fgumi_b200 import bamio, group, synth
    hdr, b, off = synth.mapped_templates(70_000, molecules=2, mean_family=2.0, paired_umis=True, umi_error_rate=0.01,
                                         seed=1)
    keep, begin = group.group_by_position(b, off, hdr)
    kb, koff = group.compact(b, off, keep)
    gr = group.ReadGrouper(0, strategy="paired", edits=1, n_threads=16)
    gr.add_groups(kb, koff, begin)
    bodies, rec_off = bamio.split_stream(gr.flush())
    ref = X.CountReference.from_host_templates(hdr, bodies, rec_off)
    assert ref.n > 250_000 and ref.n_groups > 65_536   # more groups than 16 bits of group id hold, in one pass
    for duplex in (True, False):
        m = M.MetricsCollector(hdr, duplex=duplex, device=0, n_threads=16)
        m.add_records(bodies, rec_off)
        got = m.finish()
        _compare({k: v for k, v in got.items() if k in ("family_sizes", "duplex_family_sizes", "yield_metrics")},
                 ref.tables(duplex))
        assert _stats(m) == {"kept": ref.n, "outside": 0, "groups": ref.n_groups, "ds_families": ref.n_families,
                             "overflow": ref.overflow()}


# ---- 6. one huge family and one huge group ------------------------------------------------------------------------
@pytest.mark.parametrize("duplex", [True, False])
def test_huge_family_and_group(large, duplex, monkeypatch):
    hdr, recs = large[0]["huge"]
    monkeypatch.setenv("FGB_METRICS_STAGE_BYTES", "65536")
    got, m = _run(hdr, recs, duplex, calls=5, device_bytes=8 << 20, n_threads=8,
                  **(dict(duplex_umi_counts=True) if duplex else {}))
    assert m.stats()["runs"] >= 5 and m.stats()["groups"] == 2
    _compare(got, _expect(large, "huge", duplex))
    assert _stats(m) == _expect_stats(large, "huge")


# ---- 7. exome-size interval lists ---------------------------------------------------------------------------------
@pytest.mark.parametrize("picard", [False, True])
@pytest.mark.parametrize("duplex", [True, False])
def test_exome_intervals(duplex, picard):
    recs, spans = X.exome_stream(6, 2_000)
    ivs = X.exome_intervals(7, spans)
    assert len(ivs) == 200_000
    text = X.interval_text(ivs, picard)
    idx = X.IntervalIndex(ivs)
    opts = dict(duplex_umi_counts=True) if duplex else {}
    got, m = _run(X.HEADER3, recs, duplex, calls=3, intervals=text, **opts)
    _compare(got, O.collect(X.HEADER3, recs, duplex=duplex, overlap=idx, **opts))
    exp = X.expected_stats(X.HEADER3, recs, overlap=idx)
    assert _stats(m) == exp
    assert exp["kept"] > 0 and exp["outside"] > 0


# ---- 8. template layouts on the device ----------------------------------------------------------------------------
@pytest.mark.parametrize("duplex", [True, False])
def test_template_layouts(duplex):
    """Each layout's template is followed by a plain twin with the same MI base and the ReadInfoKey the oracle computes
    for it: a right key makes a CS group of 2, a wrong key (or MI read off another record) splits it."""
    recs = X.layout_stream(X.NamePool(b"L"))
    opts = dict(duplex_umi_counts=True) if duplex else {}
    got, m = _run(S.HEADER, recs, duplex, **opts)
    _compare(got, O.collect(S.HEADER, recs, duplex=duplex, **opts))
    exp = X.expected_stats(S.HEADER, recs)
    assert _stats(m) == exp
    assert exp["groups"] * 2 == exp["kept"]
    assert "2\t%d\t" % exp["groups"] in got["family_sizes"]


# ---- the ideal-duplex fraction at high thresholds -----------------------------------------------------------------
@pytest.mark.parametrize("thresholds", [(10, 10), (50, 50), (200, 200)])
def test_ideal_fraction_at_thresholds(thresholds):
    sb = X.StreamBuilder(b"i")
    for k, n in enumerate((20, 64, 400, 401, 1000, 5000)):
        sb.group([X.fam(b"%d" % (k + 1), (n + 1) // 2, n // 2, bucket=k % 3)])
    opts = dict(min_ab_reads=thresholds[0], min_ba_reads=thresholds[1])
    got, _ = _run(S.HEADER, sb.records, True, **opts)
    ref = X.CountReference.from_templates(O.templates(S.HEADER, sb.records, [])).tables(True, **opts)
    _compare({k: got[k] for k in ref}, ref)
