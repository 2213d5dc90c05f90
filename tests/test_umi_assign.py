"""fgb_umi_assign on the H100 against oracle/umi_oracle.py: exact kinds, ids and per-group MI counts on seeded batches
(UMI lengths 1..33, mixed case, N and other bytes, dash variants, paired input prefixed and raw, single-key, empty
and multi-call groups), one large call on each side of the all-pairs / enumeration crossover, batch splitting, and
the error cases."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import umi_oracle as U      # noqa: E402
from tests import umi_cases             # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = {U.IDENTITY: "identity", U.EDIT: "edit", U.ADJACENCY: "adjacency", U.PAIRED: "paired"}
RULES = {U.MAPPED: "mapped", U.UNMAPPED: "unmapped"}


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as g
    g.build()
    import fgumi_b200
    return fgumi_b200


def batch(seed, strategy, rules, k, n_groups=60):
    rng = random.Random(seed)
    groups = []
    for _ in range(n_groups):
        L = rng.choice([1, 6, 8, 12, 20, 31, 32, 33])
        ncalls = rng.choice([1, 1, 2, 4])
        g = []
        for _ in range(ncalls):
            r = rng.random()
            if r < 0.05:
                g.append([])
            else:
                c = umi_cases.noisy_call(rng, strategy, rules, k, length=L, max_umis=rng.choice([5, 40, 120]))
                g.append(c[:1] * 3 if r < 0.12 else c)
        # a batch fails as a whole on a call the reference would fail: keep such calls out of these batches
        if all(umi_cases.oracle_ok(strategy, rules, k, c) is not None for c in g):
            groups.append(g)
    return groups


def check(fg, strategy, rules, k, groups, min_len=None):
    a = fg.UmiAssigner(0, NAMES[strategy], k, RULES[rules], min_umi_length=min_len, n_threads=4)
    try:
        res = a.assign(groups)
    finally:
        a.close()
    kinds, ids, counts = U.assign_groups(strategy, rules, k, groups, min_len)
    assert res.kinds.tolist() == kinds
    assert res.ids.tolist() == ids
    assert res.mi_counts.tolist() == counts
    return res


@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
@pytest.mark.parametrize("strategy", [U.IDENTITY, U.EDIT, U.ADJACENCY, U.PAIRED])
@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_assign_matches_oracle(fg, strategy, rules, k):
    if strategy == U.IDENTITY and k:
        pytest.skip("identity takes edits = 0 only")
    check(fg, strategy, rules, k, batch(100 * strategy + 10 * rules + k, strategy, rules, k))


def test_mi_strings(fg):
    groups = [[["AAAA-CCCC", "CCCC-AAAA", "AAAA-CCCA"]], [["GGGG-TTTT"]]]
    res = check(fg, U.PAIRED, U.UNMAPPED, 1, [[[u.encode() for u in c] for c in g] for g in groups])
    assert res.mi_strings(10) == ["10/A", "10/B", "10/A", "11/A"]


def _big_call(n_keys, L, seed):
    rng = np.random.default_rng(seed)
    codes = np.unique(rng.integers(0, 4 ** L, size=int(n_keys * 1.05), dtype=np.int64))[:n_keys]
    rng.shuffle(codes)
    digits = (codes[:, None] >> (2 * np.arange(L))[None, :]) & 3
    txt = np.frombuffer(b"ACGT", np.uint8)[digits]
    umis = [bytes(r) for r in txt]
    reps = rng.integers(1, 4, size=len(umis))          # counts 1..3: the count rule keeps some edges, drops others
    return [u for u, r in zip(umis, reps) for _ in range(r)]


@pytest.mark.parametrize("n_keys,L,k,strategy", [(200_000, 12, 1, U.ADJACENCY), (200_000, 12, 1, U.EDIT),
                                                 (900, 12, 1, U.ADJACENCY), (6_000, 10, 2, U.ADJACENCY),
                                                 (20_000, 10, 2, U.ADJACENCY)])
def test_large_call_against_enumeration_oracle(fg, n_keys, L, k, strategy):
    umis = _big_call(n_keys, L, n_keys + k)
    a = fg.UmiAssigner(0, NAMES[strategy], k, "unmapped", n_threads=8)
    try:
        res = a.assign([[umis]])
    finally:
        a.close()
    want = U.assign_call(strategy, U.UNMAPPED, k, umis, enum=True)
    assert res.kinds.tolist() == [kd for kd, _ in want]
    assert res.ids.tolist() == [i for _, i in want]


@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
def test_split_batch_changes_nothing(fg, rules):
    groups = batch(77 + rules, U.ADJACENCY, rules, 1, n_groups=40)
    a = fg.UmiAssigner(0, "adjacency", 1, RULES[rules])
    try:
        whole = a.assign(groups)
        cut = len(groups) // 3
        p1, p2 = a.assign(groups[:cut]), a.assign(groups[cut:])
    finally:
        a.close()
    assert np.array_equal(whole.kinds, np.concatenate([p1.kinds, p2.kinds]))
    assert np.array_equal(whole.ids, np.concatenate([p1.ids, p2.ids]))
    assert np.array_equal(whole.mi_counts, np.concatenate([p1.mi_counts, p2.mi_counts]))


@pytest.mark.parametrize("strategy,rules,k,groups,min_len,what", [
    (U.ADJACENCY, U.MAPPED, 1, [[[b"ACGT", b"AC"]]], None, "Multiple UMI lengths"),
    (U.PAIRED, U.MAPPED, 1, [[[b"AC-GT"]], [[b"ACGT"]]], None, "call 1"),
    (U.PAIRED, U.UNMAPPED, 1, [[[b"A-C-GT"]]], None, "not a paired UMI"),
    (U.IDENTITY, U.MAPPED, 0, [[[b"AAAAAA"], [b"AAAA"]]], 5, "shorter length"),
])
def test_errors(fg, strategy, rules, k, groups, min_len, what):
    a = fg.UmiAssigner(0, NAMES[strategy], k, RULES[rules], min_umi_length=min_len)
    try:
        with pytest.raises(fg.lib.FgbError) as e:
            a.assign(groups)
    finally:
        a.close()
    assert e.value.status == fg.lib.FGB_ERR_INVALID_ARG
    assert what in str(e.value)


def _dash_variants(rng, umis):
    """Move the dash of some UMIs: distinct strings, one BitEnc (the unmapped rules' last-index-wins case)."""
    out = []
    for u in umis:
        if rng.random() < 0.3 and len(u) > 2:
            b = u.replace("-", "")
            j = rng.randrange(1, len(b))
            u = b[:j] + "-" + b[j:]
        out.append(u)
    return out


def _edge_call(seed, strategy, rules, k, n_mol, L):
    rng = random.Random(seed)
    umis = [u.decode() for u in umi_cases.noisy_call(rng, strategy, rules, k, length=L, max_umis=40)]
    from fgumi_b200 import synth
    paired = strategy == U.PAIRED
    big = synth.umi_families(n_mol, L, mean_family=2.0, error_rate=0.03, paired=paired, seed=seed)
    if rules == U.UNMAPPED and strategy != U.IDENTITY:
        big = _dash_variants(rng, big)
    if paired and rules == U.MAPPED:
        big = [U.umi_for_read(u.encode(), rng.random() < 0.5, strategy, rules, k).decode() for u in big]
    return [u.encode() for u in (big if n_mol else umis)]


@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
@pytest.mark.parametrize("strategy", [U.EDIT, U.ADJACENCY, U.PAIRED])
@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_device_edges_equal_oracle(fg, strategy, rules, k):
    """fgb_umi_edges against the oracle's brute-force capture lists as sets: small calls (all-pairs form, both
    comparators) and, for the 2-bit comparator at k <= 2, calls past the enumeration threshold (against
    U.edges_enum) with duplicate BitEncs where the rules allow them."""
    a = fg.UmiAssigner(0, NAMES[strategy], k, RULES[rules])
    try:
        cases = [(s, 0, L) for s, L in ((1, 6), (2, 8), (3, 12), (4, 4), (5, 2))]
        if not U.uses_bytes(strategy, rules) and k <= 2:
            cases.append((6, 9000 if k <= 1 else 20000, 12 if strategy != U.PAIRED else 6))
        for seed, n_mol, L in cases:
            umis = _edge_call(seed * 10 + k, strategy, rules, k, n_mol, L)
            try:
                keys, _ = U.prepare(strategy, rules, umis)
            except U.UmiError:
                continue
            got = a.edges(umis)
            assert len(got) == len(keys)
            if len(keys) < 2:
                assert all(not r for r in got)
                continue
            want = U.edges_enum(strategy, rules, k, keys) if n_mol else U.edges(strategy, rules, k, keys)
            assert got == want, (seed, len(keys))
            if n_mol:
                assert len(keys) >= (1000 if k <= 1 else 8000)
    finally:
        a.close()


@pytest.mark.parametrize("strategy,rules,L", [(U.ADJACENCY, U.MAPPED, 12), (U.PAIRED, U.UNMAPPED, 6),
                                              (U.ADJACENCY, U.UNMAPPED, 12)])
def test_large_call_enumeration_assign(fg, strategy, rules, L):
    """Assignments of calls past the enumeration threshold: mapped adjacency, unmapped paired, and dash variants
    (several keys per BitEnc) in unmapped adjacency."""
    umis = _edge_call(77, strategy, rules, 1, 12000, L)
    a = fg.UmiAssigner(0, NAMES[strategy], 1, RULES[rules], n_threads=8)
    try:
        res = a.assign([[umis]])
    finally:
        a.close()
    keys, _ = U.prepare(strategy, rules, umis)
    assert len(keys) >= 1000
    want = U.assign_call(strategy, rules, 1, umis, enum=True)
    assert res.kinds.tolist() == [kd for kd, _ in want]
    assert res.ids.tolist() == [i for _, i in want]
