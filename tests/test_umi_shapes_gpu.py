"""fgb_umi_assign / fgb_umi_edges on the H100 at the shapes real batches reach (tests/umi_shapes.py): both kernel forms
on the same calls (FGB_UMI_ENUM_MIN_KEYS forces either form onto any 2-bit call at k <= 2), several enumeration calls
in one batch next to all-pairs, edge-free, single-key and empty calls, the byte comparator over several CTAs and
tiles of one call, 31- and 32-base keys, mixed-length calls whose BitEncs collide, and the grouper flushing two
amplicon sites at once.  Expected results come from the oracle (oracle/umi_oracle.py, oracle/group_oracle.py), with
the capture lists of large calls from U.edges_enum or from the numpy reference, and are computed once per case."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import group_oracle as G     # noqa: E402
from oracle import umi_oracle as U       # noqa: E402
from tests import umi_shapes as S        # noqa: E402
from tests.test_umi_assign import batch  # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = {U.IDENTITY: "identity", U.EDIT: "edit", U.ADJACENCY: "adjacency", U.PAIRED: "paired"}
RULES = {U.MAPPED: "mapped", U.UNMAPPED: "unmapped"}
TWO_BIT = [(U.ADJACENCY, U.MAPPED), (U.ADJACENCY, U.UNMAPPED), (U.EDIT, U.UNMAPPED), (U.PAIRED, U.UNMAPPED)]
ENUM, ALL_PAIRS = "1", str(1 << 62)     # FGB_UMI_ENUM_MIN_KEYS: every 2-bit call at k <= 2 in one form or the other


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as g
    g.build()
    import fgumi_b200
    return fgumi_b200


class _Run:
    """One UmiAssigner; every call returns plain lists."""

    def __init__(self, fg, strategy, rules, k):
        self.a = fg.UmiAssigner(0, NAMES[strategy], k, RULES[rules], n_threads=4)

    def assign(self, groups):
        r = self.a.assign(groups)
        return r.kinds.tolist(), r.ids.tolist(), r.mi_counts.tolist()

    def edges(self, calls):
        return [self.a.edges(c) for c in calls]

    def close(self):
        self.a.close()


def _forms(fg, monkeypatch, strategy, rules, k, fn, settings=(ENUM, ALL_PAIRS)):
    """fn(run) under each setting of FGB_UMI_ENUM_MIN_KEYS (None: the product's thresholds)."""
    out = []
    run = _Run(fg, strategy, rules, k)
    try:
        for v in settings:
            if v is None:
                monkeypatch.delenv("FGB_UMI_ENUM_MIN_KEYS", raising=False)
            else:
                monkeypatch.setenv("FGB_UMI_ENUM_MIN_KEYS", v)
            out.append(fn(run))
    finally:
        run.close()
        monkeypatch.delenv("FGB_UMI_ENUM_MIN_KEYS", raising=False)
    return out


def _oracle_edges(strategy, rules, k, calls):
    out = []
    for c in calls:
        keys, _ = U.prepare(strategy, rules, c)
        out.append(U.edges(strategy, rules, k, keys) if len(keys) >= 2 else [[]] * len(keys))
    return out


def _per_call(res_list):
    """(kinds, ids, counts) of a batch whose groups each hold one call, from the oracle's per-call results."""
    kinds = [kd for r in res_list for kd, _ in r]
    ids = [i if kd != U.NONE else 0 for r in res_list for kd, i in r]
    counts = [max([i for kd, i in r if kd != U.NONE], default=-1) + 1 for r in res_list]
    return kinds, ids, counts


@pytest.mark.parametrize("strategy,rules", TWO_BIT)
@pytest.mark.parametrize("k", [0, 1, 2])
def test_seeded_batches_in_both_forms(fg, monkeypatch, strategy, rules, k):
    """The seeded batches of tests/test_umi_assign.py (lengths 1..33, dash variants, duplicates, single-key and empty
    calls), every call with two or more keys forced into the enumeration form, then into the all-pairs form."""
    groups = batch(100 * strategy + 10 * rules + k, strategy, rules, k)
    calls = [c for g in groups for c in g]
    want = U.assign_groups(strategy, rules, k, groups)
    want_edges = _oracle_edges(strategy, rules, k, calls)
    assert sum(len(U.prepare(strategy, rules, c)[0]) >= 2 for c in calls) >= 20
    for got, got_edges in _forms(fg, monkeypatch, strategy, rules, k, lambda r: (r.assign(groups), r.edges(calls))):
        assert got == want
        assert got_edges == want_edges


@pytest.mark.parametrize("n_keys,L,k,strategy,rules", [
    (900, 12, 1, U.ADJACENCY, U.UNMAPPED), (4000, 32, 1, U.ADJACENCY, U.MAPPED),
    (16000, 12, 1, U.ADJACENCY, U.UNMAPPED), (30000, 12, 1, U.EDIT, U.UNMAPPED),
    (9000, 12, 2, U.ADJACENCY, U.UNMAPPED), (2500, 32, 2, U.PAIRED, U.UNMAPPED), (1100, 31, 2, U.ADJACENCY, U.MAPPED)])
def test_large_calls_in_both_forms(fg, monkeypatch, n_keys, L, k, strategy, rules):
    """Calls of 900 to 30 000 keys in the all-pairs form (many CTAs and tiles of one call) and in the enumeration
    form: the same capture lists and molecules, equal to U.edges_enum (k = 1) or the numpy reference (k = 2)."""
    umis = S.twobit_call(n_keys + L + k, strategy, rules, n_keys, L)
    keys, _ = U.prepare(strategy, rules, umis)
    assert len(keys) == n_keys
    want_edges = U.edges_enum(strategy, rules, k, keys) if k == 1 else S.capture_lists(strategy, rules, k, keys)
    assert sum(map(len, want_edges)) > n_keys // 20
    want = S.assign_call(strategy, rules, k, umis, want_edges)
    want = ([kd for kd, _ in want], [i if kd != U.NONE else 0 for kd, i in want])
    for (kinds, ids, _), got_edges in _forms(fg, monkeypatch, strategy, rules, k,
                                             lambda r: (r.assign([[umis]]), r.edges([umis])[0])):
        assert got_edges == want_edges
        assert (kinds, ids) == want


@pytest.mark.parametrize("strategy,rules", TWO_BIT)
@pytest.mark.parametrize("k", [1, 2])
def test_several_enumeration_calls_in_one_batch(fg, monkeypatch, strategy, rules, k):
    """Three calls past the product's enumeration threshold in one fgb_umi_assign, among all-pairs, edge-free,
    single-key and empty calls of three groups: each enumeration call sorts and searches its own slice of the batch's
    sorted table.  Then every call alone: the same molecules (mapped ids shifted by the earlier calls of its group)."""
    groups = S.interleaved_batch(40 + 10 * strategy + rules + k, strategy, rules, k)
    assert S.n_enum_calls(strategy, rules, k, groups) == 3
    want = S.assign_groups(strategy, rules, k, groups)
    monkeypatch.delenv("FGB_UMI_ENUM_MIN_KEYS", raising=False)
    run = _Run(fg, strategy, rules, k)
    try:
        got = run.assign(groups)
        assert got == want
        kinds, ids, _ = got
        u = 0
        for g in groups:
            base = 0
            for c in g:
                ak, ai, _ = run.assign([[c]])
                bk, bi = kinds[u:u + len(c)], ids[u:u + len(c)]
                assert ak == bk
                if rules == U.MAPPED:
                    ai = [i + base if kd != U.NONE else 0 for kd, i in zip(ak, ai)]
                    base = max([base] + [i + 1 for kd, i in zip(bk, bi) if kd != U.NONE])
                assert ai == bi
                u += len(c)
    finally:
        run.close()


BYTE_SIZES = [(129, 8), (255, 33), (256, 33), (257, 33), (383, 64), (384, 64), (385, 64), (1023, 40), (1024, 40),
              (1025, 40), (6015, 8), (6016, 8), (6017, 8)]


@pytest.mark.parametrize("strategy", [U.EDIT, U.PAIRED])
def test_byte_comparator_past_one_tile(fg, strategy):
    """Mapped edit and mapped paired calls of 128 m - 1, 128 m and 128 m + 1 keys (m up to 47) and UMIs of 8 to 64
    bases: several CTAs per call, several tiles and a short last tile.  Edges against the numpy reference, each call
    alone; molecules against the oracle's rules over those edges, all calls in one batch."""
    calls = [S.byte_call(n + L, strategy, n, L) for n, L in BYTE_SIZES]
    tables = [U.prepare(strategy, U.MAPPED, c)[0] for c in calls]
    assert [len(t) for t in tables] == [n for n, _ in BYTE_SIZES]
    want_edges = [S.capture_lists_by_k(strategy, U.MAPPED, (0, 1, 2, 3), t) for t in tables]
    for k in range(4):
        run = _Run(fg, strategy, U.MAPPED, k)
        try:
            for c, by_k, (n, L) in zip(calls, want_edges, BYTE_SIZES):
                assert run.edges([c])[0] == by_k[k], (n, L, k)
            want = _per_call([S.assign_call(strategy, U.MAPPED, k, c, by_k[k]) for c, by_k in zip(calls, want_edges)])
            assert run.assign([[c] for c in calls]) == want
        finally:
            run.close()


@pytest.mark.parametrize("strategy,rules", TWO_BIT)
@pytest.mark.parametrize("k", [0, 1, 2])
def test_long_and_mixed_length_keys_in_both_forms(fg, monkeypatch, strategy, rules, k):
    """31- and 32-base keys (the top BitEnc bits) and, under the unmapped rules, calls of 1..5 bases whose BitEncs
    collide across lengths, one of them past the enumeration threshold: both forms and the product's thresholds, one
    group of several calls."""
    calls = [S.twobit_call(31 + k, strategy, rules, 600, 31), S.twobit_call(32 + k, strategy, rules, 1100, 32)]
    if rules == U.UNMAPPED:
        calls += [S.mixed_call(5 + k, strategy, 300), S.mixed_call(6 + k, strategy, 1200)]
    tables = [U.prepare(strategy, rules, c)[0] for c in calls]
    want_edges = [S.capture_lists(strategy, rules, k, t) for t in tables]
    want = S.assign_groups(strategy, rules, k, [calls])
    for got, got_edges in _forms(fg, monkeypatch, strategy, rules, k,
                                 lambda r: (r.assign([calls]), r.edges(calls)), settings=(ENUM, ALL_PAIRS, None)):
        assert got_edges == want_edges
        assert got == want


def _kept(group, synth, seed, paired, umi_length):
    hdr, b, off = synth.mapped_templates(2, molecules=5, mean_family=3.0, umi_length=umi_length, paired_umis=paired,
                                         amplicon_molecules=1500, umi_error_rate=0.03, seed=seed)
    keep, begin = group.group_by_position(b, off, hdr)
    kb, koff = group.compact(b, off, keep)
    recs = [kb[int(koff[i]):int(koff[i + 1])].tobytes() for i in range(len(koff) - 1)]
    return kb, koff, begin, recs


@pytest.mark.parametrize("strategy,umi_length", [("adjacency", 8), ("paired", 6)])
def test_grouper_flushes_two_amplicon_sites(fg, strategy, umi_length):
    """Two amplicon inputs through two add_groups and one flush: two calls past the enumeration threshold in one
    device phase, against the oracle grouper fed the same two batches."""
    from fgumi_b200 import group, synth
    s = U.STRATEGIES[strategy]
    og = G.Grouper(G.Config(strategy=s, edits=1, rules=U.UNMAPPED))
    g = group.ReadGrouper(0, strategy, 1, allow_unmapped=True, n_threads=4)
    try:
        for seed in (21, 22):
            kb, koff, begin, recs = _kept(group, synth, seed, strategy == "paired", umi_length)
            og.add_groups(recs, begin)
            g.add_groups(kb, koff, begin)
        pending = og.pending()
        big = [c for gr in pending for c in gr if len(U.prepare(s, U.UNMAPPED, c)[0]) > S.enum_min_keys(1)]
        assert len(big) >= 2
        c = og.cfg
        want = og.flush(U.assign_groups(c.assign_strategy, c.rules, c.assign_edits, pending, c.assign_min_len, enum=True))
        assert g.flush() == want
    finally:
        g.close()
