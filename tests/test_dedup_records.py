"""`fgumi dedup` from raw records on the host: the library's position grouping with secondary and supplementary records
(fgb_host_dedup_group_by_position) and planning-only deduper (fgb_deduper_pending, fgb_deduper_flush_with_ids)
against tests/dedup_oracle.py on seeded streams.  CPU only: the assignment and the template scores of the flush come
from the oracle."""
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

NAMES = {U.IDENTITY: "identity", U.EDIT: "edit", U.ADJACENCY: "adjacency", U.PAIRED: "paired"}


@pytest.fixture(scope="module")
def dd():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import dedup
    return dedup


def stream(seed, paired=False, **kw):
    from fgumi_b200 import synth
    args = dict(molecules=4, mean_family=2.5, umi_length=4 if paired else 8, paired_umis=paired, seed=seed,
                umi_error_rate=0.05, n_umi_rate=0.03, low_mapq_rate=0.05, qc_fail_rate=0.05, unmapped_mate_rate=0.4,
                secondary_rate=0.3, cross_contig_rate=0.2)
    args.update(kw)
    hdr, b, off = synth.mapped_templates(6, **args)
    return hdr, edit(records_of(b, off), seed)


def pair(name, pos, umi, **kw):
    t = [(b"RX", "Z", umi), (b"MC", "Z", b"10M")]
    return [make_record(name, 0x1 | 0x40 | 0x20, 0, pos, 60, "10M", 0, pos + 100, seq=b"A" * 10, tags=t),
            make_record(name, 0x1 | 0x80 | 0x10, 0, pos + 100, 60, "10M", 0, pos, seq=b"A" * 10, tags=t)]


@pytest.mark.parametrize("seed", range(6))
def test_group_by_position_matches_oracle(dd, seed):
    hdr, recs = stream(seed, seed % 2 == 1)
    b, off = pack(recs)
    keep, begin = dd.group_by_position(b, off, hdr)
    okeep, obegin = D.group_by_position(recs, hdr)
    assert keep.tolist() == okeep and begin.tolist() == obegin
    assert len(begin) > 3


def test_group_by_position_secondary_placements(dd):
    """Secondary and supplementary records before their primaries, after them, alone at the start, between groups."""
    def sup(name, pos, flag=0x1 | 0x40 | 0x800):
        return make_record(name, flag, 0, pos, 60, "10M", seq=b"A" * 10, tags=[])
    recs = ([sup(b"s0", 7), sup(b"s1", 9)] + [sup(b"a", 900)] + pair(b"a", 100, b"AC") + [sup(b"a", 901, 0x181)] +
            pair(b"b", 100, b"AC") + [sup(b"x", 5)] + pair(b"c", 400, b"GT") + [sup(b"c", 1, 0x1 | 0x80 | 0x900)])
    b, off = pack(recs)
    keep, begin = dd.group_by_position(b, off, b"")
    okeep, obegin = D.group_by_position(recs, b"")
    assert keep.tolist() == okeep == [1] * len(recs) and begin.tolist() == obegin
    # s0, s1 and a's leading supplementary share the default key, a's primaries continue its QNAME, and a's trailing
    # secondary has the default key again | pair b | x | pair c with its secondary
    assert obegin == [0, 6, 8, 9, 12]


def test_group_by_position_missing_mc(dd):
    bad = make_record(b"zz", 0x1 | 0x40, 0, 99, 60, "10M", 0, 199, seq=b"A" * 10, tags=[(b"RX", "Z", b"AAAA")])
    ok_sec = make_record(b"zz", 0x1 | 0x40 | 0x100, 0, 99, 60, "10M", 0, 199, seq=b"A" * 10, tags=[])
    b, off = pack(pair(b"a", 100, b"AAAA") + [ok_sec])
    dd.group_by_position(b, off, b"")   # a secondary record is not MC-checked
    b, off = pack(pair(b"a", 100, b"AAAA") + [bad])
    with pytest.raises(ValueError, match="record 2 \\(zz\\)"):
        dd.group_by_position(b, off, b"")


GRID = [(s, k) for s in (U.IDENTITY, U.EDIT, U.ADJACENCY, U.PAIRED) for k in range(3) if not (s == U.IDENTITY and k)]


@pytest.mark.parametrize("strategy,k", GRID)
@pytest.mark.parametrize("remove", [False, True])
def test_planning_deduper_matches_oracle(dd, strategy, k, remove):
    paired = strategy == U.PAIRED
    variants = [dict(), dict(min_map_q=30, include_non_pf=True)]
    if not paired:
        variants += [dict(no_umi=True), dict(min_umi_length=6)]
    later = 0   # families whose kept template is not the first in (MI, QNAME) order: the scores decided
    for vi, opts in enumerate(variants):
        threads = 1 if vi % 2 == 0 else 6
        seed = 100 * strategy + 10 * k + vi + 1000 * remove
        hdr, recs = stream(seed, paired)
        cfg = D.Config(strategy=strategy, edits=k, first_mi=7, remove_duplicates=remove, **opts)
        _, begin = D.group_by_position(recs, hdr)
        od = D.Deduper(cfg)
        pd = dd.Deduper(None, NAMES[strategy], k, n_threads=threads, first_mi=7, remove_duplicates=remove, **opts)
        b, off = pack(recs)
        half = len(begin) // 2
        for lo, hi in ((0, half), (half, len(begin) - 1)):   # two flushes, the MI base carried
            od.add_groups(recs, begin[lo:hi + 1])
            pd.add_groups(b, off, np.asarray(begin[lo:hi + 1], np.uint64))
            assert pd.pending() == od.pending()
            kinds, ids, counts = od.assign()
            scores = od.scores()
            assert pd.flush_with_ids(kinds, ids, counts, scores) == od.flush((kinds, ids, counts), scores)
        st = pd.stats()
        assert [st[n] for n in D.STATS] == od.stats
        assert pd.histogram() == od.family_sizes
        assert pd.metrics() == D.dedup_metrics(od.stats)
        later += od.later_representatives
        assert st["duplicate_templates"] > 0 and st["secondary_reads"] > 0 and st["missing_tc_tag"] > 0
        pd.close()
    assert later > 0


def test_cell_barcodes_split_groups(dd):
    recs = pair(b"a", 100, b"ACGTACGT") + pair(b"b", 100, b"ACGTACGT")
    recs = [r + b"CBZC1\0" for r in recs[:2]] + [r + b"CBZC2\0" for r in recs[2:]]
    b, off = pack(recs)
    _, begin = dd.group_by_position(b, off, b"")
    assert begin.tolist() == D.group_by_position(recs, b"")[1] == [0, 2, 4]
    _, begin = dd.group_by_position(b, off, b"", None)
    assert begin.tolist() == [0, 4]


def _fails(dd, recs, groups, match, **kw):
    from fgumi_b200 import lib as L
    b, off = pack(recs)
    d = dd.Deduper(None, **kw)
    ok = pair(b"ok", 5000, b"AAAA-CCCC" if kw.get("strategy") == "paired" else b"ACGTACGT")
    ob, ooff = pack(ok)
    d.add_groups(ob, ooff, np.array([0, 2], np.uint64))
    before = (d.pending(), d.stats())
    with pytest.raises(L.FgbError, match=match):
        d.add_groups(b, off, np.asarray(groups, np.uint64))
    assert (d.pending(), d.stats()) == before   # nothing of the failing call stays
    d.close()


def test_two_primary_r1_fails_the_call(dd):
    recs = pair(b"a", 100, b"ACGTACGT")
    _fails(dd, recs + [recs[0]], [0, 3], "Multiple", strategy="identity", edits=0)


def test_paired_umi_without_dash_fails_the_call(dd):
    recs = pair(b"a", 100, b"AAAA-CCCC") + pair(b"b", 100, b"AAAACCCC")
    _fails(dd, recs, [0, 4], "2 segments", strategy="paired", edits=1)


def test_umi_not_utf8_fails_the_call(dd):
    recs = pair(b"a", 100, b"ACGT\xffCGT")
    _fails(dd, recs, [0, 2], "UTF-8", strategy="adjacency", edits=1)


def test_bad_options(dd):
    from fgumi_b200 import lib as L
    d = dd.Deduper(None, "adjacency", 1)
    with pytest.raises(L.FgbError):
        d.flush()   # planning only
    d.close()
    for kw in (dict(strategy="paired", min_umi_length=4), dict(strategy="paired", no_umi=True)):
        with pytest.raises(L.FgbError):
            dd.Deduper(None, **kw)
    opt = L.FgbDedupOptions()
    opt.umi.rules = L.FGB_UMI_RULES_UNMAPPED
    import ctypes as C
    h = C.c_void_p()
    assert L.load().fgb_deduper_create(L.FGB_DEVICE_NONE, C.byref(opt), C.byref(h)) == L.FGB_ERR_INVALID_ARG
    # identity with edits: the reference forces 0 edits (dedup.rs:940-947) where fgb_umi_assign would refuse them
    opt = L.FgbDedupOptions()
    opt.umi.strategy, opt.umi.edits, opt.umi.rules = 0, 1, L.FGB_UMI_RULES_MAPPED
    assert L.load().fgb_deduper_create(L.FGB_DEVICE_NONE, C.byref(opt), C.byref(h)) == L.FGB_OK
    L.load().fgb_deduper_destroy(h)
    gopt = L.FgbGroupOptions()   # the same options, which the grouper passes through unchanged, are refused there
    gopt.umi.strategy, gopt.umi.edits, gopt.umi.rules = 0, 1, L.FGB_UMI_RULES_MAPPED
    assert L.load().fgb_grouper_create(L.FGB_DEVICE_NONE, C.byref(gopt), C.byref(h)) == L.FGB_ERR_INVALID_ARG


def test_struct_size_of_dedup_options(dd):
    from fgumi_b200 import lib as L
    import ctypes as C
    assert L.load().fgb_struct_size(13) == C.sizeof(L.FgbDedupOptions) == 40
