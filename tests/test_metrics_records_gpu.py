"""The device metrics collector (fgb_metrics_*) against tests/metrics_oracle.py: every table's text, both modes, with
and without --duplex-umi-counts and intervals, across staged runs and calls, and the errors with the records they
name."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgumi_b200 import lib as L           # noqa: E402
from fgumi_b200 import metrics as M       # noqa: E402
from tests import metrics_oracle as O     # noqa: E402
from tests import metrics_streams as S    # noqa: E402

pytestmark = pytest.mark.gpu


def _compare(got, exp):
    assert sorted(got) == sorted(exp)
    for name in exp:
        if name != "yield_metrics" or not exp[name].startswith("fraction\tread_pairs\tcs_families\tss_families\tds"):
            assert got[name] == exp[name], name
            continue
        gl, el = got[name].splitlines(), exp[name].splitlines()
        assert len(gl) == len(el)
        for g, e in zip(gl, el):   # every byte but the ideal fraction (scipy vs statrs), within 1e-12 relative
            g, e = g.split("\t"), e.split("\t")
            assert g[:-1] == e[:-1]
            if g[-1] != e[-1]:
                assert abs(float(g[-1]) - float(e[-1])) <= 1e-12 * abs(float(e[-1])), (g, e)


def _run(records, duplex=True, calls=1, intervals=None, **opts):
    m = M.MetricsCollector(S.HEADER, duplex=duplex, intervals=intervals, device=0, **opts)
    b, off = S.to_arrays(records)
    cuts = np.linspace(0, len(records), calls + 1).astype(int)
    name = lambda i: records[i][32:32 + records[i][8]]
    for k in range(calls):
        lo, hi = int(cuts[k]), int(cuts[k + 1])
        while 0 < lo < len(records) and name(lo) == name(lo - 1):
            lo += 1
        while 0 < hi < len(records) and name(hi) == name(hi - 1):
            hi += 1
        if k + 1 == calls:
            hi = len(records)
        if hi > lo:
            m.add_records(b[int(off[lo]):int(off[hi])], off[lo:hi + 1] - off[lo])
        cuts[k + 1] = hi
    return m.finish(), m


def _oracle(records, duplex=True, intervals=None, **opts):
    return O.collect(S.HEADER, records, duplex=duplex, intervals=intervals, **opts)


@pytest.mark.parametrize("duplex", [True, False])
@pytest.mark.parametrize("umi_counts", [False, True])
def test_random_streams(duplex, umi_counts):
    recs = S.random_stream(1, 300, odd_mi_rate=0.2, suffix_rate=0.85)
    opts = dict(duplex_umi_counts=umi_counts) if duplex else {}
    got, _ = _run(recs, duplex, **opts)
    _compare(got, _oracle(recs, duplex, **opts))


@pytest.mark.parametrize("duplex", [True, False])
def test_intervals_and_thresholds(duplex):
    recs = S.random_stream(2, 200)
    for iv in (b"chr1\t0\t30000\nchr2\t60000\t90000\n", b"@SQ\tSN:chr1\tLN:1\nchr2\t1\t50000\t+\tx\n", b"chrZ\t0\t1\n"):
        opts = dict(min_ab_reads=3, min_ba_reads=2, duplex_umi_counts=True) if duplex else dict(min_reads=3)
        got, _ = _run(recs, duplex, intervals=iv, **opts)
        _compare(got, _oracle(recs, duplex, intervals=iv, **opts))


@pytest.mark.parametrize("duplex", [True, False])
def test_overflow_families(duplex):
    recs = S.random_stream(3, 40, big_family=70)
    got, m = _run(recs, duplex, duplex_umi_counts=duplex) if duplex else _run(recs, duplex)
    assert m.stats()["overflow"] > 0
    _compare(got, _oracle(recs, duplex, **(dict(duplex_umi_counts=True) if duplex else {})))


@pytest.mark.parametrize("calls", [1, 3, 17])
def test_staged_runs_and_calls(calls, monkeypatch):
    recs = S.random_stream(4, 120, big_family=40)   # the big group spans several 4 KiB runs
    monkeypatch.setenv("FGB_METRICS_STAGE_BYTES", "4096")
    got, m = _run(recs, True, calls=calls, device_bytes=64 << 10, duplex_umi_counts=True)
    assert m.stats()["runs"] >= max(calls, 2)
    _compare(got, _oracle(recs, True, duplex_umi_counts=True))


def test_group_output_of_synthetic_workload():
    from fgumi_b200 import bamio, group, synth
    hdr, b, off = synth.mapped_templates(300, molecules=3, mean_family=3.0, paired_umis=True, umi_error_rate=0.02,
                                         seed=5)
    keep, begin = group.group_by_position(b, off, hdr)
    kb, koff = group.compact(b, off, keep)
    gr = group.ReadGrouper(0, strategy="paired", edits=1)
    gr.add_groups(kb, koff, begin)
    bodies, rec_off = bamio.split_stream(gr.flush())
    recs = [bytes(bodies[int(rec_off[i]):int(rec_off[i + 1])]) for i in range(len(rec_off) - 1)]
    for duplex in (True, False):
        m = M.MetricsCollector(hdr, duplex=duplex, device=0, n_threads=4, duplex_umi_counts=duplex)
        m.add_records(bodies, rec_off)
        got = m.finish()
        _compare(got, O.collect(hdr, recs, duplex=duplex, duplex_umi_counts=duplex))


def test_empty_input():
    got, _ = _run([], True)
    _compare(got, _oracle([], True))


def _error(records, duplex=True, calls=1, **opts):
    with pytest.raises(M.MetricsError) as e:
        _run(records, duplex, calls=calls, **opts)
    with pytest.raises(O.MetricsOracleError) as o:
        _oracle(records, duplex, **{k: v for k, v in opts.items() if k != "n_threads"})
    assert e.value.bad_record == o.value.record
    return e.value


def test_missing_tags_outside_intervals_fail():
    good = S.random_stream(6, 5)
    bad = S.pair(b"zz1", None, b"AAA-CCC", pos1=90000, pos2=90200)
    err = _error(good + bad + S.random_stream(7, 3), intervals=b"chr1\t0\t10\n")
    assert "MI" in str(err)
    bad = S.pair(b"zz2", b"4/A", None, pos1=90000, pos2=90200)
    assert "RX" in str(_error(good + bad, calls=2))


def test_consensus_input_fails():
    recs = S.random_stream(8, 3)
    cons = S.pair(b"c1", b"1/A", b"A-C", r1_tags=[(b"cD", "i", 3), (b"MI", "Z", b"1/A"), (b"RX", "Z", b"A-C")])
    err = _error(cons + recs)
    assert "consensus" in str(err)


def test_mixed_dna_umi_fails():
    recs = S.random_stream(9, 4, suffix_rate=1.0)
    bad = S.pair(b"u1", b"900/A", b"AC-GT", pos1=77000, pos2=77200) + \
        S.pair(b"u2", b"900/A", b"A+-GT", pos1=77000, pos2=77200)
    _error(recs + bad + S.random_stream(10, 2), n_threads=3)
    _error(recs + bad, duplex=False)


def test_min_ab_below_min_ba_refused():
    with pytest.raises(L.FgbError):
        M.MetricsCollector(S.HEADER, duplex=True, device=0, min_ab_reads=1, min_ba_reads=2)
    with pytest.raises(ValueError):
        O.collect(S.HEADER, [], duplex=True, min_ab_reads=1, min_ba_reads=2)


def test_metrics_files(tmp_path):
    from fgumi_b200 import bamio
    import struct
    recs = S.random_stream(11, 50)
    path = str(tmp_path / "in.bam")
    text = S.HEADER
    refs = [ln.split(b"\t") for ln in text.split(b"\n") if ln.startswith(b"@SQ")]
    raw = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for r in refs:
        nm = r[1][3:] + b"\0"
        raw += struct.pack("<i", len(nm)) + nm + struct.pack("<i", int(r[2][3:]))
    raw += b"".join(struct.pack("<I", len(x)) + x for x in recs)
    with open(path, "wb") as f:
        bamio._write_bgzf(f, raw, 1, 1)
    bamio.duplex_metrics_file(path, str(tmp_path / "d"), duplex_umi_counts=True, batch_records=37)
    exp = _oracle(recs, True, duplex_umi_counts=True)
    for name, suffix in (("family_sizes", ".family_sizes.txt"), ("duplex_family_sizes", ".duplex_family_sizes.txt"),
                         ("umi_counts", ".umi_counts.txt"), ("duplex_umi_counts", ".duplex_umi_counts.txt")):
        assert open(str(tmp_path / "d") + suffix).read() == exp[name]
    bamio.simplex_metrics_file(path, str(tmp_path / "s"), batch_records=37)
    exp = _oracle(recs, False)
    assert open(str(tmp_path / "s") + ".simplex_yield_metrics.txt").read() == exp["yield_metrics"]
