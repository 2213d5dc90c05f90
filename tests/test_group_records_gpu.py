"""The record-level grouper on the device (fgb_grouper_flush through fgb_umi_assign) against oracle/group_oracle.py:
byte-identical streams, histograms and counters over the strategy grid, batches split across calls and flushes, an
amplicon-like position group large enough for the enumeration form, bamio.group_file on a generated BAM, and
bamio.group_and_call (mapped BAM -> group -> simplex / duplex in memory) against the oracle's group followed by the
record oracle's callers."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import group_oracle as G     # noqa: E402
from oracle import umi_oracle as U       # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = {U.IDENTITY: "identity", U.EDIT: "edit", U.ADJACENCY: "adjacency", U.PAIRED: "paired"}
ERRS = dict(umi_error_rate=0.05, n_umi_rate=0.05, low_mapq_rate=0.05, qc_fail_rate=0.05, unmapped_mate_rate=0.4,
            secondary_rate=0.1, cross_contig_rate=0.2)


@pytest.fixture(scope="module")
def mods():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, group, synth
    return group, synth, bamio


def _kept(group, synth, seed, paired, n_sites=40, **kw):
    hdr, b, off = synth.mapped_templates(n_sites, molecules=5, mean_family=3.0, umi_length=4 if paired else 8,
                                         paired_umis=paired, seed=seed, **kw)
    keep, begin = group.group_by_position(b, off, hdr)
    kb, koff = group.compact(b, off, keep)
    recs = [kb[int(koff[i]):int(koff[i + 1])].tobytes() for i in range(len(koff) - 1)]
    return kb, koff, begin, recs


GRID = [(s, rules, k) for s in (U.IDENTITY, U.EDIT, U.ADJACENCY, U.PAIRED) for rules in (U.MAPPED, U.UNMAPPED)
        for k in range(4) if not (s == U.IDENTITY and k)]


@pytest.mark.parametrize("strategy,rules,k", GRID)
def test_grouper_matches_oracle(mods, strategy, rules, k):
    group, synth, _ = mods
    paired = strategy == U.PAIRED
    variants = [dict(), dict(min_map_q=30, include_non_pf=True)] + ([] if paired else [dict(no_umi=True),
                                                                                       dict(min_umi_length=6)])
    for vi, opts in enumerate(variants):
        kw = dict(ERRS, no_dash_rate=0.15 if paired else 0.0)
        kb, koff, begin, recs = _kept(group, synth, 1000 * strategy + 100 * rules + 10 * k + vi, paired, **kw)
        og = G.Grouper(G.Config(strategy=strategy, edits=k, rules=rules, first_mi=3, **opts))
        g = group.ReadGrouper(0, NAMES[strategy], k, allow_unmapped=rules == U.UNMAPPED, first_mi=3,
                              n_threads=1 if vi % 2 == 0 else 6, **opts)
        half = len(begin) // 2
        for lo, hi in ((0, half), (half, len(begin) - 1)):
            og.add_groups(recs, begin[lo:hi + 1])
            g.add_groups(kb, koff, begin[lo:hi + 1])
            assert g.flush() == og.flush()
        st = g.stats()
        assert [st[n] for n in G.STATS] == og.stats
        assert g.histogram("family") == og.family_sizes and g.histogram("position") == og.group_sizes
        g.close()


def test_split_across_calls_and_flushes_changes_no_byte(mods):
    group, synth, _ = mods
    kb, koff, begin, _ = _kept(group, synth, 7, False, n_sites=60, **ERRS)
    whole = group.ReadGrouper(0, "adjacency", 1, n_threads=4)
    whole.add_groups(kb, koff, begin)
    ref = whole.flush()
    parts = group.ReadGrouper(0, "adjacency", 1, n_threads=3)
    out = b""
    cuts = [0, 5, 6, 17, 30, len(begin) - 1]
    for i in range(len(cuts) - 1):
        parts.add_groups(kb, koff, begin[cuts[i]:cuts[i + 1] + 1])
        if i % 2:
            out += parts.flush()
    out += parts.flush()
    assert out == ref
    assert parts.histogram("family") == whole.histogram("family") and parts.stats() == whole.stats()
    whole.close()
    parts.close()


@pytest.mark.parametrize("strategy", ["adjacency", "edit"])
def test_amplicon_group_enumeration_form(mods, strategy):
    group, synth, _ = mods
    kb, koff, begin, recs = _kept(group, synth, 11, False, n_sites=2, amplicon_molecules=1500, umi_error_rate=0.03)
    og = G.Grouper(G.Config(strategy=U.STRATEGIES[strategy], edits=1, rules=U.UNMAPPED))
    og.add_groups(recs, begin)
    assert max(len(set(c)) for gr in og.pending() for c in gr) >= 1000   # distinct UMIs above the enumeration threshold
    g = group.ReadGrouper(0, strategy, 1, allow_unmapped=True, n_threads=4)
    g.add_groups(kb, koff, begin)
    assert g.flush() == og.flush()
    g.close()


def test_group_file_matches_oracle(mods, tmp_path):
    group, synth, bamio = mods
    hdr, b, off = synth.mapped_templates(30, molecules=4, seed=5, **ERRS)
    inp, outp = str(tmp_path / "in.bam"), str(tmp_path / "out.bam")
    payload = bamio.mapped_bam_header(hdr)
    for i in range(len(off) - 1):
        payload += np.uint32(off[i + 1] - off[i]).tobytes() + b[int(off[i]):int(off[i + 1])].tobytes()
    from fgumi_b200.caller import bgzf_compress
    with open(inp, "wb") as f:
        f.write(bgzf_compress(payload))
    g = group.ReadGrouper(0, "adjacency", 1, n_threads=2)
    bamio.group_file(inp, outp, g)
    text, ob, ooff, _ = bamio.read_bam(outp)
    recs = [b[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]
    expect, _ = G.group_stream(recs, hdr, G.Config(strategy=U.ADJACENCY, edits=1))
    got = b"".join(np.uint32(ooff[i + 1] - ooff[i]).tobytes() + ob[int(ooff[i]):int(ooff[i + 1])].tobytes()
                   for i in range(len(ooff) - 1))
    assert got == expect
    assert text == bamio.group_header(hdr) and "PP:bwa" in text.decode().splitlines()[-1]
    g.close()
    with pytest.raises(ValueError):
        bamio.check_group_sort_order(b"@HD\tVN:1.6\tSO:coordinate\n", False)


# ---- mapped BAM -> group -> simplex / duplex, against the oracle's group followed by the record oracle's callers ----
def _write_bam(bamio, path, hdr, b, off):
    from fgumi_b200.caller import bgzf_compress
    payload = bamio.mapped_bam_header(hdr) + b"".join(
        np.uint32(off[i + 1] - off[i]).tobytes() + b[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1))
    with open(path, "wb") as f:
        f.write(bgzf_compress(payload))


def _oracle_group_call(hdr, b, off, cfg, oracle, duplex):
    """group_oracle's stream, grouped by MI (the base MI for duplex; records without MI skipped), each group through
    the record oracle's caller."""
    recs = [b[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]
    stream, _ = G.group_stream(recs, hdr, cfg)
    tagged, p = [], 0
    while p < len(stream):
        n = int.from_bytes(stream[p:p + 4], "little")
        r = stream[p + 4:p + 4 + n]
        p += 4 + n
        mi = G.find_string_tag(r, b"MI")
        if mi is not None:
            tagged.append((mi[:-2] if duplex and mi[-2:] in (b"/A", b"/B") else mi, r))
    want, count, i = bytearray(), 0, 0
    while i < len(tagged):
        j = i + 1
        while j < len(tagged) and tagged[j][0] == tagged[i][0]:
            j += 1
        d, n = oracle.consensus_reads([r for _, r in tagged[i:j]])
        want += d
        count += n
        i = j
    return bytes(want), count


@pytest.mark.parametrize("strategy", ["identity", "adjacency"])
def test_group_then_simplex_matches_oracle(mods, strategy, tmp_path):
    group, synth, bamio = mods
    import fgumi_b200 as fg
    from oracle import record_oracle as R
    from tests import oracle_lib as O
    from tests.test_record_oracle_kat import vote_fn
    hdr, b, off = synth.mapped_templates(40, molecules=4, mean_family=4.0, seed=31, **ERRS)
    path = str(tmp_path / "in.bam")
    _write_bam(bamio, path, hdr, b, off)
    k = 0 if strategy == "identity" else 1
    g = group.ReadGrouper(0, strategy, k, n_threads=4)
    opt = fg.VanillaUmiConsensusOptions(min_reads=1, min_consensus_base_quality=2, min_input_base_quality=10)
    caller = fg.VanillaUmiConsensusCaller("fgumi", "A", opt, device=0, n_threads=4)
    got = bamio.group_and_call(path, g, caller)
    oracle = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(min_reads=1, min_consensus_base_quality=2,
                                                                  min_input_base_quality=10), vote_fn, O.builder_call)
    want, count = _oracle_group_call(hdr, b, off, G.Config(strategy=U.STRATEGIES[strategy], edits=k), oracle, False)
    assert count > 50 and got.count == count
    assert got.data == want
    g.close()
    caller.close()


def test_group_then_duplex_matches_oracle(mods, tmp_path):
    group, synth, bamio = mods
    import fgumi_b200 as fg
    from oracle import record_oracle as R
    from tests import oracle_lib as O
    from tests.test_caller_parity import duplex_job_fn
    from tests.test_record_oracle_kat import vote_fn
    hdr, b, off = synth.mapped_templates(40, molecules=4, mean_family=6.0, umi_length=4, paired_umis=True,
                                         reverse_rate=0.5, seed=37, **dict(ERRS, no_dash_rate=0.05))
    path = str(tmp_path / "in.bam")
    _write_bam(bamio, path, hdr, b, off)
    g = group.ReadGrouper(0, "paired", 1, n_threads=4)
    caller = fg.DuplexConsensusCaller("fgumi", "A", min_reads=(1, 1, 0), device=0, n_threads=4)
    got = bamio.group_and_call(path, g, caller)
    oracle = R.DuplexCallerOracle("fgumi", "A", min_reads=(1, 1, 0), per_base=True, vote_fn=vote_fn,
                                  builder_fn=O.builder_call, duplex_job_fn=duplex_job_fn)
    want, count = _oracle_group_call(hdr, b, off, G.Config(strategy=U.PAIRED, edits=1), oracle, True)
    assert count > 20 and got.count == count
    assert got.data == want
    assert g.stats()["groups_dropped"] > 0
    g.close()
    caller.close()

