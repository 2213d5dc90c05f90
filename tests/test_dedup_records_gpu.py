"""`fgumi dedup` on the device against tests/dedup_oracle.py: the deduper's flush (template scores on the device beside
fgb_umi_assign) byte-identical to the oracle with identical counters and histograms over the strategy grid, mark and
remove, 1 and 6 threads, several flushes; fgb_record_quality_scores against numpy at every alignment of the quality
slice, 0xFF qualities, 65 535-base reads, qualities cut short by the record's end, an empty call and one of several
staging chunks and grid waves; bamio.dedup_file on a BAM built from tests/bam_builder.py records."""
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import umi_oracle as U       # noqa: E402
from tests import dedup_oracle as D      # noqa: E402
from tests.bam_builder import make_record   # noqa: E402
from tests.dedup_streams import edit, pack, records_of   # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = {U.IDENTITY: "identity", U.EDIT: "edit", U.ADJACENCY: "adjacency", U.PAIRED: "paired"}


@pytest.fixture(scope="module")
def mods():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, dedup, engine, synth
    return dedup, synth, bamio, engine


@pytest.fixture(scope="module")
def eng(mods):
    e = mods[3].Engine(0)
    yield e
    e.close()


def stream(synth, seed, paired, n_sites=30):
    hdr, b, off = synth.mapped_templates(n_sites, molecules=5, mean_family=3.0, umi_length=4 if paired else 8,
                                         paired_umis=paired, seed=seed, umi_error_rate=0.05, n_umi_rate=0.03,
                                         low_mapq_rate=0.05, qc_fail_rate=0.05, unmapped_mate_rate=0.4,
                                         secondary_rate=0.3, cross_contig_rate=0.2)
    return hdr, edit(records_of(b, off), seed)


GRID = [(s, k) for s in (U.IDENTITY, U.EDIT, U.ADJACENCY, U.PAIRED) for k in range(3) if not (s == U.IDENTITY and k)]


@pytest.mark.parametrize("strategy,k", GRID)
@pytest.mark.parametrize("remove", [False, True])
def test_deduper_flush_matches_oracle(mods, strategy, k, remove):
    dedup, synth, _, _ = mods
    paired = strategy == U.PAIRED
    variants = [dict(), dict(min_map_q=30, include_non_pf=True)]
    if not paired:
        variants += [dict(no_umi=True), dict(min_umi_length=6)]
    later = 0   # families whose kept template is not the first in (MI, QNAME) order: the scores decided
    for vi, opts in enumerate(variants):
        threads = 1 if vi % 2 == 0 else 6
        hdr, recs = stream(synth, 7 * strategy + k + 100 * vi + 1000 * remove, paired)
        cfg = D.Config(strategy=strategy, edits=k, first_mi=3, remove_duplicates=remove, **opts)
        _, begin = D.group_by_position(recs, hdr)
        od = D.Deduper(cfg)
        gd = dedup.Deduper(0, NAMES[strategy], k, n_threads=threads, first_mi=3, remove_duplicates=remove, **opts)
        b, off = pack(recs)
        cuts = [0, len(begin) // 3, 2 * len(begin) // 3, len(begin) - 1]
        for lo, hi in zip(cuts, cuts[1:]):   # three flushes, the MI base carried
            od.add_groups(recs, begin[lo:hi + 1])
            gd.add_groups(b, off, np.asarray(begin[lo:hi + 1], np.uint64))
            assert gd.flush() == od.flush()
        st = gd.stats()
        assert [st[n] for n in D.STATS] == od.stats
        assert gd.histogram() == od.family_sizes
        assert gd.metrics() == D.dedup_metrics(od.stats)
        later += od.later_representatives
        tm = gd.last_timing()
        assert len(tm) == 7 and tm["score_phase_ms"] > 0 and tm["score_kernel_ms"] > 0
        gd.close()
    assert later > 0


def np_scores(recs):
    return np.array([D.read_score(r) for r in recs], np.uint32)


def test_quality_scores_every_alignment(mods, eng):
    """l_seq 0-64 with names that put the quality slice at every offset modulo 16, qualities 0-255 (0xFF included)."""
    dedup = mods[0]
    rng = np.random.default_rng(1)
    recs = []
    for l_seq in range(65):
        for name_len in range(1, 17):
            q = rng.integers(0, 256, size=l_seq, dtype=np.uint8)
            q[rng.random(l_seq) < 0.2] = 0xFF
            recs.append(make_record(b"n" * name_len, 0, 0, 9, 60, None, seq=b"A" * l_seq, quals=q.tobytes()))
    # a leading pad record of each length 32..47 shifts every following record's start, so the device sees all 16
    # alignments of the slice start within the chunk as well
    for pad in range(16):
        recs.insert(0, make_record(b"p" * (pad + 1), 4, -1, -1, 0, "", seq=b""))
        b, off = pack(recs)
        assert (dedup.record_quality_scores(eng, b, off) == np_scores(recs)).all()


def test_quality_scores_long_reads_and_cut_records(mods, eng):
    dedup = mods[0]
    rng = np.random.default_rng(2)
    recs = []
    for l_seq in (65535, 65534, 40000, 301):
        q = rng.integers(0, 256, size=l_seq, dtype=np.uint8)
        recs.append(make_record(b"long%d" % l_seq, 0, 0, 9, 60, "%dM" % l_seq, seq=b"C" * l_seq, quals=q.tobytes(),
                                tags=[(b"RX", "Z", b"ACGT")]))
    full = make_record(b"cut", 0, 0, 9, 60, "100M", seq=b"G" * 100, quals=bytes([40] * 100))
    for cut in (1, 7, 16, 50, 99, 100):   # qualities cut short by the record's end
        recs.append(full[:len(full) - cut])
    recs.append(full[:32 + full[8] + 4])  # the record ends before its sequence: score 0
    b, off = pack(recs)
    got = dedup.record_quality_scores(eng, b, off)
    assert (got == np_scores(recs)).all() and got[-1] == 0 and got[0] > 65535


def test_quality_scores_empty_and_large(mods, eng):
    dedup = mods[0]
    assert len(dedup.record_quality_scores(eng, np.zeros(0, np.uint8), np.zeros(1, np.uint64))) == 0
    # 37.7 MB of 269-byte records: three 16 MiB staging chunks and many passes of the grid over each
    rng = np.random.default_rng(3)
    base = [make_record(b"r%06d" % i, 0x1 | 0x40, 0, i, 60, "150M", seq=b"A" * 150,
                        quals=rng.integers(0, 256, size=150, dtype=np.uint8).tobytes()) for i in range(2000)]
    recs = base * 70
    b, off = pack(recs)
    assert int(off[-1]) > 2 * (16 << 20)
    want = np.tile(np_scores(base), 70)
    assert (dedup.record_quality_scores(eng, b, off) == want).all()


def test_quality_scores_short_record(mods, eng):
    dedup = mods[0]
    from fgumi_b200 import lib as L
    recs = [make_record(b"a", 0, 0, 9, 60, "4M", seq=b"ACGT"), b"\0" * 31]
    b, off = pack(recs)
    with pytest.raises(L.FgbError, match="record 1") as e:
        dedup.record_quality_scores(eng, b, off)
    assert e.value.status == L.FGB_ERR_LAYOUT


def _dup_pairs(prefix, umi, count, start, tc=True):
    out = []
    for i in range(count):
        name = b"%s_%d" % (prefix, i)
        t = [(b"RX", "Z", umi), (b"MC", "Z", b"8M")]
        q = [(5 + 3 * i) % 15] * 8   # below the cap of 15: the last template of each family scores highest
        out.append(make_record(name, 0x1 | 0x40, 0, start - 1, 60, "8M", 0, start + 99, 108, b"ACGTACGT", q, t))
        out.append(make_record(name, 0x1 | 0x80 | 0x10, 0, start + 99, 60, "8M", 0, start - 1, -108, b"ACGTACGT", q,
                               t))
        if i == 1:
            out.append(make_record(name, 0x1 | 0x40 | 0x800, 0, start + 500, 60, "8M", 0, start + 99, 0, b"ACGTACGT",
                                   q, t + ([(b"tc", "i", 1)] if tc else [])))
    return out


def _write_bam(bamio, path, hdr, recs):
    from fgumi_b200.caller import bgzf_compress
    with open(path, "wb") as f:
        f.write(bgzf_compress(bamio.mapped_bam_header(hdr) + b"".join(struct.pack("<I", len(r)) + r for r in recs)))


HDR = b"@HD\tVN:1.6\tSO:unsorted\tGO:query\tSS:template-coordinate\n@SQ\tSN:chr1\tLN:100000\n@PG\tID:bwa\tPN:bwa\n"


@pytest.mark.parametrize("remove", [False, True])
def test_dedup_file_round_trip(mods, tmp_path, remove):
    dedup, _, bamio, _ = mods
    recs = _dup_pairs(b"dup1", b"ACGTACGT", 3, 100) + _dup_pairs(b"dup2", b"TGCATGCA", 2, 500)
    inp, outp = str(tmp_path / "in.bam"), str(tmp_path / "out.bam")
    _write_bam(bamio, inp, HDR, recs)
    d = dedup.Deduper(0, "adjacency", 1, remove_duplicates=remove, n_threads=2)
    bamio.dedup_file(inp, outp, d)
    text, ob, ooff, _ = bamio.read_bam(outp)
    expect, od = D.dedup_stream(recs, HDR, D.Config(remove_duplicates=remove))
    got = b"".join(struct.pack("<I", int(ooff[i + 1] - ooff[i])) + ob[int(ooff[i]):int(ooff[i + 1])].tobytes()
                   for i in range(len(ooff) - 1))
    assert got == expect
    assert text == bamio.group_header(HDR, "fgumi_b200 dedup") and "PP:bwa" in text.decode().splitlines()[-1]
    assert d.metrics() == D.dedup_metrics(od.stats) and d.metrics()["duplicate_templates"] == 3
    from tests.bam_builder import parse_records
    kept = {r["name"] for r in parse_records(got) if not r["flags"] & 0x400}
    assert kept == {b"dup1_2", b"dup2_1"}   # the best-scoring template, not the first by name
    d.close()


def test_dedup_file_rejects_coordinate_order(mods, tmp_path):
    dedup, _, bamio, _ = mods
    inp = str(tmp_path / "in.bam")
    _write_bam(bamio, inp, b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:100000\n",
               _dup_pairs(b"a", b"ACGTACGT", 2, 100))
    d = dedup.Deduper(0)
    with pytest.raises(ValueError, match="template-coordinate"):
        bamio.dedup_file(inp, str(tmp_path / "out.bam"), d)
    d.close()


def test_dedup_file_missing_tc_raises_after_writing(mods, tmp_path):
    dedup, _, bamio, _ = mods
    recs = _dup_pairs(b"a", b"ACGTACGT", 3, 100, tc=False)
    inp, outp = str(tmp_path / "in.bam"), str(tmp_path / "out.bam")
    _write_bam(bamio, inp, HDR, recs)
    d = dedup.Deduper(0)
    with pytest.raises(ValueError, match="1 secondary/supplementary"):
        bamio.dedup_file(inp, outp, d)
    _, ob, ooff, _ = bamio.read_bam(outp)
    assert len(ooff) - 1 == len(recs)
    # the same deduper on an input whose records all carry tc: only this input's records count
    good = str(tmp_path / "good.bam")
    _write_bam(bamio, good, HDR, _dup_pairs(b"b", b"ACGTACGT", 3, 900))
    bamio.dedup_file(good, outp, d)
    assert d.stats()["missing_tc_tag"] == 1
    d.close()
