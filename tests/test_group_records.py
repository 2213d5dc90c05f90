"""`fgumi group` from raw records on the host: oracle/group_oracle.py pinned by ports of the reference's own tests,
then the library's position grouping (fgb_host_group_by_position) and planning-only grouper (fgb_grouper_pending,
fgb_grouper_flush_with_ids) against the oracle on seeded mapped streams.  CPU only: the assignment of the flush comes
from the oracle's assigners."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import group_oracle as G     # noqa: E402
from oracle import umi_oracle as U       # noqa: E402
from tests.bam_builder import make_record, parse_records   # noqa: E402

NAMES = {U.IDENTITY: "identity", U.EDIT: "edit", U.ADJACENCY: "adjacency", U.PAIRED: "paired"}


@pytest.fixture(scope="module")
def grp():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import group
    return group


def pair(name, pos, umi, mate_pos=None, rev1=False, mapq=60, flags_extra=0, ref=0, mate_ref=0, tags=(), cigar="10M",
         mc=b"10M"):
    """An FR pair as SamBuilder::add_pair builds it: R1 at pos, R2 at mate_pos (1-based positions)."""
    mate_pos = pos + 100 if mate_pos is None else mate_pos
    f1 = 0x1 | 0x40 | (0x10 if rev1 else 0x20) | flags_extra
    f2 = 0x1 | 0x80 | (0x20 if rev1 else 0x10)
    t = [(b"RX", "Z", umi)] if umi is not None else []
    t += [(b"MC", "Z", mc)] + list(tags)
    r1 = make_record(name, f1, ref, pos - 1, mapq, cigar, mate_ref, mate_pos - 1, seq=b"A" * 10, tags=t)
    r2 = make_record(name, f2, mate_ref, mate_pos - 1, mapq, cigar, ref, pos - 1, seq=b"A" * 10, tags=t)
    return [r1, r2]


def run(records, **kw):
    cfg = G.Config(**kw)
    out, g = G.group_stream(records, b"", cfg)
    return parse_records(out), g


def mis(recs):
    return [(r["name"], r["tags"].get(b"MI")) for r in recs]


# ---- ports of group.rs's tests (group.rs:2046-) ----------------------------------------------------------------
def test_basic_grouping_identity():
    recs = pair(b"a", 100, b"AAAAAAAA") + pair(b"b", 100, b"AAAAAAAA") + pair(b"c", 100, b"CCCCCCCC")
    out, g = run(recs, strategy=U.IDENTITY, edits=0)
    assert len(out) == 6
    m = dict(mis(out))
    assert m[b"a"] == m[b"b"] != m[b"c"]
    assert g.family_sizes == {2: 1, 1: 1}


def test_adjacency_merges_one_edit():
    recs = pair(b"a", 100, b"AAAAAAAA") + pair(b"b", 100, b"AAAAAAAA") + pair(b"c", 100, b"AAAAAAAT")
    out, _ = run(recs, strategy=U.ADJACENCY, edits=1)
    assert len({m for _, m in mis(out)}) == 1


def test_n_in_umi_discarded():
    recs = pair(b"a", 100, b"AAAANAAA") + pair(b"b", 100, b"AAAAAAAA")
    out, g = run(recs, strategy=U.IDENTITY, edits=0)
    assert [r["name"] for r in out] == [b"b", b"b"]
    assert g.stats[4] == 2 and g.stats[0] == 4 and g.stats[1] == 2   # per read


def test_lowercase_n_is_not_n():
    out, g = run(pair(b"a", 100, b"AAAAnAAA"), strategy=U.IDENTITY, edits=0)
    assert len(out) == 2 and g.stats[4] == 0


def test_min_mapq():
    recs = pair(b"a", 100, b"AAAAAAAA", mapq=10) + pair(b"b", 100, b"AAAAAAAA", mapq=30)
    out, g = run(recs, strategy=U.IDENTITY, edits=0, min_map_q=20)
    assert {r["name"] for r in out} == {b"b"} and g.stats[3] == 2


def test_mate_mq_tag_cast_as_u8():
    # MQ:i:256 reads as 0 (`as u8`), below min_map_q 1
    out, g = run(pair(b"a", 100, b"AAAAAAAA", tags=[(b"MQ", "i", 256)]), strategy=U.IDENTITY, edits=0)
    assert out == [] and g.stats[3] == 2
    out, _ = run(pair(b"a", 100, b"AAAAAAAA", tags=[(b"MQ", "i", 257)]), strategy=U.IDENTITY, edits=0)
    assert len(out) == 2


def test_non_pf():
    recs = pair(b"a", 100, b"AAAAAAAA", flags_extra=0x200)
    out, g = run(recs, strategy=U.IDENTITY, edits=0)
    assert out == [] and g.stats[2] == 2
    out, g = run(recs, strategy=U.IDENTITY, edits=0, include_non_pf=True)
    assert len(out) == 2


def test_single_end_reads():
    recs = [make_record(b"s%d" % i, 0, 0, 99, 60, "10M", seq=b"A" * 10, tags=[(b"RX", "Z", u)])
            for i, u in enumerate([b"ACGT", b"ACGT", b"TTTT"])]
    out, g = run(recs, strategy=U.IDENTITY, edits=0)
    assert len(out) == 3 and g.family_sizes == {2: 1, 1: 1}


def test_missing_raw_tag_discarded():
    out, g = run(pair(b"a", 100, None), strategy=U.IDENTITY, edits=0)
    assert out == [] and g.stats[3] == 2


def test_too_short_umi():
    recs = pair(b"a", 100, b"ACGT") + pair(b"b", 100, b"ACGTACGT")
    out, g = run(recs, strategy=U.IDENTITY, edits=0, min_umi_length=6)
    assert {r["name"] for r in out} == {b"b"} and g.stats[5] == 2


def test_truncated_umis_group_together():
    recs = pair(b"a", 100, b"ACGTACGTAA") + pair(b"b", 100, b"ACGTACGTCC")
    out, _ = run(recs, strategy=U.IDENTITY, edits=0, min_umi_length=8)
    assert len({m for _, m in mis(out)}) == 1


def test_cross_contig_pair():
    recs = pair(b"a", 100, b"AAAAAAAA", mate_ref=1, mate_pos=500) + pair(b"b", 100, b"AAAAAAAA", mate_ref=1, mate_pos=500)
    keep, begin = G.group_by_position(recs)
    assert begin == [0, 4]
    out, _ = run(recs, strategy=U.IDENTITY, edits=0)
    assert len({m for _, m in mis(out)}) == 1


def test_pair_orientation_split():
    # same UMI, opposite orientations: separate calls, so separate molecules for non-paired strategies
    recs = pair(b"a", 100, b"AAAAAAAA", 200) + pair(b"b", 200, b"AAAAAAAA", 100, rev1=True)
    recs = recs[:2] + [recs[3], recs[2]]
    keep, begin = G.group_by_position(recs)
    assert begin == [0, 4]
    out, _ = run(recs, strategy=U.IDENTITY, edits=0)
    assert len({m for _, m in mis(out)}) == 2


def test_paired_strategy_no_split():
    recs = pair(b"a", 100, b"AAAA-CCCC", 200) + pair(b"b", 200, b"CCCC-AAAA", 100, rev1=True)
    recs = recs[:2] + [recs[3], recs[2]]
    out, _ = run(recs, strategy=U.PAIRED, edits=1)
    m = {n: v for n, v in mis(out)}
    assert m[b"a"][:-2] == m[b"b"][:-2] and {m[b"a"][-1:], m[b"b"][-1:]} == {b"A", b"B"}


def test_paired_umi_without_dash_drops_group():
    recs = pair(b"a", 100, b"AAAACCCC") + pair(b"b", 100, b"AAAA-CCCC") + pair(b"c", 5000, b"GGGG-TTTT")
    out, g = run(recs, strategy=U.PAIRED, edits=1)
    assert {r["name"] for r in out} == {b"c"} and g.stats[7] == 1 and g.stats[1] == 6


def test_no_umi_groups_by_position():
    recs = pair(b"a", 100, None) + pair(b"b", 100, None) + pair(b"c", 3000, None)
    out, g = run(recs, strategy=U.ADJACENCY, edits=1, no_umi=True)
    m = dict(mis(out))
    assert m[b"a"] == m[b"b"] == b"0" and m[b"c"] == b"1"


def test_no_umi_refused_with_paired():
    with pytest.raises(G.GroupError):
        G.Grouper(G.Config(strategy=U.PAIRED, no_umi=True))
    with pytest.raises(G.GroupError):
        G.Grouper(G.Config(strategy=U.PAIRED, min_umi_length=4))


def test_position_group_sizes_and_metrics():
    recs = (pair(b"a", 100, b"AAAAAAAA") + pair(b"b", 100, b"CCCCCCCC") + pair(b"c", 100, b"CCCCCCCC")
            + pair(b"d", 3000, b"GGGGGGGG"))
    out, g = run(recs, strategy=U.IDENTITY, edits=0)
    assert g.group_sizes == {2: 1, 1: 1} and g.family_sizes == {1: 2, 2: 1}
    m = G.grouping_metrics(g.stats, g.family_sizes)
    assert m["total_families"] == 3 and m["median_reads_per_molecule"] == 1 and m["max_reads_per_molecule"] == 2
    assert m["avg_reads_per_molecule"] == pytest.approx(8 / 3)


def test_mi_counter_is_consecutive_across_groups():
    recs = pair(b"a", 100, b"AAAAAAAA") + pair(b"b", 3000, b"CCCCCCCC") + pair(b"c", 3000, b"GGGGGGGG")
    out, g = run(recs, strategy=U.IDENTITY, edits=0, first_mi=10)
    assert sorted({int(v) for _, v in mis(out)}) == [10, 11, 12] and g.stats[8] == 13


# ---- RecordPositionGrouper / build_templates_from_records (grouper.rs) and GroupKey (base.rs) ------------------
def test_group_key_lower_first():
    r = pair(b"a", 500, b"A", mate_pos=100)[0]   # the mate is reverse at 100 with 10M: its 5' end is 109
    k = G.position_key(r, {}, None)
    assert k[:3] == (0, 109, 1) and k[3:6] == (0, 500, 0)


def test_group_key_single_without_mc():
    r = make_record(b"a", 0x1 | 0x40, 0, 99, 60, "5S10M", 0, 299, seq=b"A" * 15, tags=[])
    assert G.position_key(r, {}, None)[:6] == (0, 95, 0, G.I32_MAX, G.I32_MAX, 255)


def test_group_key_library_and_cell():
    hdr = b"@RG\tID:x\tLB:L1\n@RG\tID:y\tLB:L1\n@RG\tID:z\tLB:L2\n@RG\tID:w\n"
    libs = G.library_index(hdr)
    assert libs == {b"x": 1, b"y": 1, b"z": 2, b"w": 0}
    r = make_record(b"a", 0, 0, 9, 60, "10M", seq=b"A" * 10, tags=[(b"RG", "Z", b"z"), (b"CB", "Z", b"C1")])
    assert G.position_key(r, libs, b"CB")[6:] == (2, b"C1")


def test_missing_mc_is_an_error():
    r1 = make_record(b"a", 0x1 | 0x40, 0, 99, 60, "10M", 0, 199, seq=b"A" * 10, tags=[(b"RX", "Z", b"AAAA")])
    with pytest.raises(G.GroupError) as e:
        G.group_by_position([r1])
    assert e.value.record == 0


def test_secondary_supplementary_skipped_and_unmapped_mate_continues():
    r1 = make_record(b"a", 0x1 | 0x8 | 0x40, 0, 99, 60, "10M", 0, 99, seq=b"A" * 10, tags=[(b"RX", "Z", b"AC")])
    sup = make_record(b"a", 0x1 | 0x40 | 0x800, 0, 500, 60, "10M", 0, 99, seq=b"A" * 10, tags=[])
    r2 = make_record(b"a", 0x1 | 0x4 | 0x80, 0, 99, 0, "", 0, 99, seq=b"A" * 10, tags=[(b"RX", "Z", b"AC")])
    other = make_record(b"b", 0, 0, 599, 60, "10M", seq=b"A" * 10, tags=[(b"RX", "Z", b"AC")])
    keep, begin = G.group_by_position([r1, sup, r2, other])
    assert keep == [1, 0, 1, 1] and begin == [0, 2, 3]


def test_templates_from_consecutive_names():
    recs = pair(b"a", 100, b"A") + pair(b"b", 100, b"A")
    t = G.build_templates(recs)
    assert [x[0] for x in t] == [b"a", b"b"] and all(x[1] is not None and x[2] is not None for x in t)
    with pytest.raises(G.GroupError):
        G.build_templates([recs[0], recs[0]])


# ---- update_string_tag (tags.rs) ----------------------------------------------------------------------------
def test_update_string_tag_forms():
    base = make_record(b"a", 4, -1, -1, 0, "", seq=b"AC", tags=[(b"XX", "i", 5), (b"MI", "Z", b"12")])
    same = G.update_string_tag(base, b"MI", b"34")
    assert same.endswith(b"MIZ34\0") and len(same) == len(base)
    longer = G.update_string_tag(base, b"MI", b"345")
    assert longer.endswith(b"MIZ345\0")
    plain = make_record(b"a", 4, -1, -1, 0, "", seq=b"AC", tags=[(b"XX", "i", 5)])
    assert G.update_string_tag(plain, b"MI", b"7") == plain + b"MIZ7\0"
    # an integer MI of the same value length keeps its type byte (find_tag_bounds is type-agnostic)
    imi = make_record(b"a", 4, -1, -1, 0, "", seq=b"AC", tags=[(b"MI", "i", 5)])
    assert G.update_string_tag(imi, b"MI", b"123")[-7:-4] == b"MIi"


# ---- the library against the oracle ------------------------------------------------------------------------------
def _stream(seed, paired, **kw):
    from fgumi_b200 import synth
    return synth.mapped_templates(6, molecules=4, mean_family=2.5, umi_length=4 if paired else 8,
                                  paired_umis=paired, seed=seed, **kw)


def _records(bodies, off):
    return [bodies[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


ERRS = dict(umi_error_rate=0.05, n_umi_rate=0.05, low_mapq_rate=0.05, qc_fail_rate=0.05, unmapped_mate_rate=0.4,
            secondary_rate=0.1, cross_contig_rate=0.2)


@pytest.mark.parametrize("seed", range(4))
def test_group_by_position_matches_oracle(grp, seed):
    hdr, b, off = _stream(seed, seed % 2 == 1, **ERRS)
    keep, begin = grp.group_by_position(b, off, hdr)
    okeep, obegin = G.group_by_position(_records(b, off), hdr)
    assert keep.tolist() == okeep and begin.tolist() == obegin


def test_group_by_position_missing_mc(grp):
    r = make_record(b"zz", 0x1 | 0x40, 0, 99, 60, "10M", 0, 199, seq=b"A" * 10, tags=[(b"RX", "Z", b"AAAA")])
    ok = pair(b"a", 100, b"AAAA")
    recs = ok + [r]
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in recs])
    with pytest.raises(ValueError, match="record 2 \\(zz\\)"):
        grp.group_by_position(np.frombuffer(b"".join(recs), np.uint8), off, b"")


GRID = [(s, rules, k) for s in (U.IDENTITY, U.EDIT, U.ADJACENCY, U.PAIRED) for rules in (U.MAPPED, U.UNMAPPED)
        for k in range(4) if not (s == U.IDENTITY and k)]


@pytest.mark.parametrize("strategy,rules,k", GRID)
def test_planning_grouper_matches_oracle(grp, strategy, rules, k):
    paired = strategy == U.PAIRED
    variants = [dict(), dict(min_map_q=30, include_non_pf=True)]
    if not paired:
        variants += [dict(no_umi=True), dict(min_umi_length=6)]
    for vi, opts in enumerate(variants):
        threads = 1 if vi % 2 == 0 else 6
        seed = 100 * strategy + 10 * rules + k + vi
        kw = dict(ERRS, no_dash_rate=0.15 if paired else 0.0)
        hdr, b, off = _stream(seed, paired, **kw)
        recs = _records(b, off)
        cfg = G.Config(strategy=strategy, edits=k, rules=rules, first_mi=7, **opts)
        keep, begin = G.group_by_position(recs, hdr)
        kept = [r for r, x in zip(recs, keep) if x]
        og = G.Grouper(cfg)
        pg = grp.ReadGrouper(None, NAMES[strategy], k, allow_unmapped=rules == U.UNMAPPED, n_threads=threads,
                             first_mi=7, **opts)
        kb = np.frombuffer(b"".join(kept), np.uint8)
        koff = np.zeros(len(kept) + 1, np.uint64)
        koff[1:] = np.cumsum([len(x) for x in kept])
        half = len(begin) // 2
        for lo, hi in ((0, half), (half, len(begin) - 1)):   # two flushes, the MI base carried
            og.add_groups(kept, begin[lo:hi + 1])
            pg.add_groups(kb, koff, np.asarray(begin[lo:hi + 1], np.uint64))
            assert pg.pending() == og.pending()
            kinds, ids, counts = og.assign()
            assert pg.flush_with_ids(kinds, ids, counts) == og.flush((kinds, ids, counts))
        st = pg.stats()
        assert [st[n] for n in G.STATS] == og.stats
        assert pg.histogram("family") == og.family_sizes and pg.histogram("position") == og.group_sizes
        assert pg.metrics() == G.grouping_metrics(og.stats, og.family_sizes)
        if paired:
            assert st["groups_dropped"] > 0
        pg.close()


def test_planning_grouper_refuses_flush_and_bad_options(grp):
    from fgumi_b200 import lib as L
    g = grp.ReadGrouper(None, "adjacency", 1)
    with pytest.raises(L.FgbError):
        g.flush()
    g.close()
    with pytest.raises(L.FgbError):
        grp.ReadGrouper(None, "paired", 1, min_umi_length=4)
    with pytest.raises(L.FgbError):
        grp.ReadGrouper(None, "paired", 1, no_umi=True)


def test_two_primary_r1_fails_the_call_and_queues_nothing(grp):
    recs = pair(b"a", 100, b"AAAAAAAA") + pair(b"b", 3000, b"CCCCCCCC")
    bad = recs[:2] + [recs[2], recs[2]]
    off = np.zeros(len(bad) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in bad])
    g = grp.ReadGrouper(None, "identity", 0)
    from fgumi_b200 import lib as L
    with pytest.raises(L.FgbError, match="Multiple"):
        g.add_groups(np.frombuffer(b"".join(bad), np.uint8), off, np.array([0, 2, 4], np.uint64))
    assert g.pending() == [] and g.stats()["total_records"] == 0
    g.close()


def test_existing_mi_tag_overwrite_splice_and_append(grp):
    """Input records that already carry the assign tag: Z of the same length (overwritten in place), longer, shorter
    and empty (spliced), an integer MI whose value width matches (overwritten, type byte kept) or not (spliced), and
    none (appended) -- the library's bytes against the oracle's."""
    variants = [[(b"MI", "Z", b"9")], [(b"MI", "Z", b"99999")], [(b"MI", "Z", b"")], [(b"MI", "i", 7)],
                [(b"MI", "C", 7)], [(b"MI", "Z", b"12"), (b"XY", "i", 3)], []]
    recs = []
    for i, v in enumerate(variants):
        recs += pair(b"t%02d" % i, 100, b"ACGTACG" + b"ACGT"[i % 4:i % 4 + 1], tags=v)
    recs += pair(b"u", 3000, b"ACGTACGT", tags=[(b"MI", "Z", b"55")])
    keep, begin = G.group_by_position(recs)
    og = G.Grouper(G.Config(strategy=U.IDENTITY, edits=0, first_mi=98))
    og.add_groups(recs, begin)
    pg = grp.ReadGrouper(None, "identity", 0, first_mi=98)
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in recs])
    pg.add_groups(np.frombuffer(b"".join(recs), np.uint8), off, np.asarray(begin, np.uint64))
    kinds, ids, counts = og.assign()
    want = og.flush((kinds, ids, counts))
    assert pg.flush_with_ids(kinds, ids, counts) == want
    types = {r["name"]: r["tags"].get(b"MI") for r in parse_records(want)}
    assert isinstance(types[b"t03"], int) and types[b"t03"] != 7      # MI:i overwritten in place, type kept
    assert all(isinstance(v, bytes) for n, v in types.items() if n != b"t03")
    pg.close()


def test_struct_sizes_of_group_options(grp):
    from fgumi_b200 import lib as L
    import ctypes as C
    lib = L.load()
    assert lib.fgb_struct_size(10) == C.sizeof(L.FgbUmiOptions) == 24
    assert lib.fgb_struct_size(11) == C.sizeof(L.FgbGroupOptions) == 40

