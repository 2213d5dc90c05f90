"""tests/umi_shapes.py on the CPU: its capture lists against the oracle's brute force (U.edges) and neighbour enumeration
(U.edges_enum), its assignments against U.assign_groups, and its generators against what they claim to build."""
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import umi_oracle as U       # noqa: E402
from tests import umi_cases               # noqa: E402
from tests import umi_shapes as S         # noqa: E402

TWO_BIT = [(U.ADJACENCY, U.MAPPED), (U.ADJACENCY, U.UNMAPPED), (U.EDIT, U.UNMAPPED), (U.PAIRED, U.UNMAPPED)]


def _calls(strategy, rules, seed):
    """Calls of up to ~300 keys: the seeded noisy calls, and the generators' shapes that fit the rules."""
    rng = random.Random(seed)
    out = [umi_cases.noisy_call(rng, strategy, rules, 1, length=L, max_umis=m)
           for L, m in ((1, 30), (6, 120), (12, 120), (31, 80), (32, 80), (33, 60))]
    if U.uses_bytes(strategy, rules):
        out += [S.byte_call(seed + n, strategy, n, L) for n, L in ((127, 8), (129, 33), (257, 40), (300, 64))]
    else:
        out += [S.twobit_call(seed + n, strategy, rules, n, L) for n, L in ((150, 12), (257, 31), (300, 32))]
        if rules == U.UNMAPPED:
            out.append(S.mixed_call(seed, strategy, 300))
    return out


@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
@pytest.mark.parametrize("strategy", [U.EDIT, U.ADJACENCY, U.PAIRED])
def test_reference_equals_brute_force(strategy, rules):
    n = 0
    for c in _calls(strategy, rules, 10 * strategy + rules):
        try:
            keys, _ = U.prepare(strategy, rules, c)
        except U.UmiError:
            continue
        got = S.capture_lists_by_k(strategy, rules, (0, 1, 2, 3), keys)
        for k in range(4):
            assert got[k] == U.edges(strategy, rules, k, keys), (len(keys), k)
            n += sum(map(len, got[k]))
    assert n > 200                              # the calls have edges to find


@pytest.mark.parametrize("strategy,rules", TWO_BIT)
@pytest.mark.parametrize("k", [0, 1, 2])
def test_reference_equals_enumeration(strategy, rules, k):
    for c in _calls(strategy, rules, 100 + 10 * strategy + rules):
        try:
            keys, _ = U.prepare(strategy, rules, c)
        except U.UmiError:
            continue
        assert S.capture_lists(strategy, rules, k, keys) == U.edges_enum(strategy, rules, k, keys), len(keys)


@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
@pytest.mark.parametrize("strategy", [U.IDENTITY, U.EDIT, U.ADJACENCY, U.PAIRED])
def test_assign_groups_equals_oracle(strategy, rules):
    for k in (0, 1, 2):
        calls = [c for c in umi_cases.calls(7 * strategy + rules + k, strategy, rules, k, 60)
                 if umi_cases.oracle_ok(strategy, rules, k, c) is not None]
        groups = [calls[i:i + 1 + i % 4] for i in range(0, len(calls), 4)]
        assert S.assign_groups(strategy, rules, k, groups) == U.assign_groups(strategy, rules, k, groups)


# ---- the generators -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("strategy", [U.EDIT, U.PAIRED])
def test_byte_calls(strategy):
    for n, L in ((129, 8), (255, 33), (256, 40), (257, 64), (1023, 8), (6017, 8)):
        c = S.byte_call(n, strategy, n, L)
        keys, _ = U.prepare(strategy, U.MAPPED, c)
        assert len(keys) == n
        assert {len(k.s) for k in keys} == {L + (strategy == U.PAIRED)}
        assert len(c) > n                       # counts above 1 exist, so the count rule drops some edges
    if strategy == U.EDIT:
        return
    # the dash moves within one length, and some edges are found only through the query's reversed form between
    # keys whose dashes differ (building the reversed form around the other key's dash would lose them)
    keys, _ = U.prepare(U.PAIRED, U.MAPPED, S.byte_call(3, U.PAIRED, 300, 33))
    assert len({k.s.index(b"-") for k in keys}) >= 3
    rev_only = [(a, b) for a in keys for b in keys
                if U.count_mismatches(a.s, b.s) > 1 and U.count_mismatches(U.reverse_paired(a.s), b.s) <= 1
                and a.s.index(b"-") != b.s.index(b"-")]
    assert len(rev_only) >= 5


@pytest.mark.parametrize("strategy,rules", TWO_BIT)
@pytest.mark.parametrize("L", [31, 32])
def test_twobit_calls(strategy, rules, L):
    c = S.twobit_call(L, strategy, rules, 500, L)
    keys, _ = U.prepare(strategy, rules, c)
    assert len(keys) == 500 and {k.len for k in keys} == {L}
    top = [k.bits >> (2 * L - 2) for k in keys]
    assert len(set(top)) == 4                   # the last base takes every value, in BitEnc bits 2L - 2 and 2L - 1
    assert sum(map(len, S.capture_lists(strategy, rules, 1, keys))) > 0
    if rules == U.UNMAPPED and strategy != U.EDIT:
        assert not all(k.last for k in keys)   # several keys per BitEnc


@pytest.mark.parametrize("strategy", [U.ADJACENCY, U.EDIT, U.PAIRED])
def test_mixed_length_calls(strategy):
    for n in (300, 1200):
        c = S.mixed_call(n, strategy, n)
        keys, _ = U.prepare(strategy, U.UNMAPPED, c)
        assert len(keys) == n and {k.len for k in keys} == {1, 2, 3, 4, 5}
        lens_of = {}
        for k in keys:
            lens_of.setdefault(k.bits, set()).add(k.len)
        assert lens_of[0] >= {1, 2, 3}          # A, AA, AAA: one BitEnc
        assert sum(len(v) > 1 for v in lens_of.values()) >= 20
    assert n >= S.enum_min_keys(1)


@pytest.mark.parametrize("strategy,rules", TWO_BIT)
@pytest.mark.parametrize("k", [1, 2])
def test_interleaved_batches(strategy, rules, k):
    groups = S.interleaved_batch(5, strategy, rules, k, n_groups=3, n_enum=3)
    assert len(groups) == 3 and S.n_enum_calls(strategy, rules, k, groups) == 3
    sizes = []
    for g in groups:
        assert sum(len(U.prepare(strategy, rules, c)[0]) >= S.enum_min_keys(k) for c in g) == 1
        assert [] in g
        per_call = [U.prepare(strategy, rules, c)[0] for c in g if c]
        assert any(len(keys) == 1 for keys in per_call)                          # a single-key call
        assert any(2 <= len(keys) < 128 for keys in per_call)                    # small all-pairs calls
        assert any(len(keys) == 12 and not any(S.capture_lists(strategy, rules, k, keys)) for keys in per_call)
        sizes += [len(keys) for keys in per_call if len(keys) >= S.enum_min_keys(k)]
    assert len(set(sizes)) == 3
