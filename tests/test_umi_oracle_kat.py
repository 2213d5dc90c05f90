"""oracle/umi_oracle.py pinned by ports of the reference's own known-answer tests (fgumi 0.2.0):
crates/fgumi-umi/src/assigner.rs (tests module), src/lib/umi/parallel_assigner.rs (tests module),
crates/fgumi-umi/src/lib.rs (MoleculeId) and src/lib/commands/group.rs (test_umi_for_read_*, test_truncate_umis_*).
Each test keeps the reference's name.  Not ported: the BK-tree / n-gram index internals (the restatement has no index;
test_adjacency_index_vs_linear_produces_same_results and test_bktree_vs_ngram_same_results become the linear vs
enumeration check in tests/test_umi_host.py, plus the index-threshold cases below, which must give the linear
answer), the UnionFind internals, the thread-count / determinism-across-runs cases (one answer by construction) and the
proptest properties, which are restated as seeded loops where they constrain results.  CPU only."""
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import umi_oracle as U      # noqa: E402

M, UM = U.MAPPED, U.UNMAPPED


def run(strategy, umis, k=1, rules=M):
    return U.assign_call(strategy, rules, k, [u.encode() for u in umis])


def mid(res, strip=False):
    """MoleculeId as the reference's to_string / base_id_string (lib.rs:134-141, 178-187)."""
    return [U.mi_string(U.SINGLE if strip and kd != U.NONE else kd, i, 0) for kd, i in res]


def groups(umis, res, strip=False):
    g = {}
    for u, m in zip(umis, mid(res, strip)):
        g.setdefault(m, set()).add(u)
    return sorted(map(sorted, g.values()))


def amap(umis, res):
    return dict(zip(umis, mid(res)))


def rep(u, n):
    return [u] * n


# ---- assigner.rs tests ------------------------------------------------------------------------------------
@pytest.mark.parametrize("a,b,want", [("AAAA", "AAAA", 0), ("AAAA", "AAAC", 1), ("AAAA", "CCCC", 4),
                                      ("AAAA", "AACC", 2), ("AAA", "AAAA", 1 << 64), ("", "", 0), ("A", "A", 0),
                                      ("A", "T", 1)])
def test_count_mismatches(a, b, want):
    assert U.count_mismatches(a.encode(), b.encode()) == want


UM6 = ["AAAAAA", "AAAAAT", "ACGTAC", "ACGTAC", "AAAAAA"]


def test_identity_assigner_basic():
    assert len(set(mid(run(U.IDENTITY, UM6, 0)))) == 3


def test_identity_assigner_groups_exact_matches():
    assert groups(UM6, run(U.IDENTITY, UM6, 0)) == [["AAAAAA"], ["AAAAAT"], ["ACGTAC"]]


E6 = ["AAAAAA", "AAAATT", "AAAATA", "TGCACC", "TGCACG", "GGCGGC"]


def test_simple_error_assigner_basic():
    assert len(set(mid(run(U.EDIT, E6, 1)))) == 3


def test_simple_error_assigner_groups_by_mismatches():
    umis = E6 + ["GGCGGC", "GGCGGC"]
    assert groups(umis, run(U.EDIT, umis, 1)) == [["AAAAAA", "AAAATA", "AAAATT"], ["GGCGGC"], ["TGCACC", "TGCACG"]]


def test_simple_error_assigner_groups_everything_with_high_edits():
    umis = E6 + ["GGCGGC", "GGCGGC"]
    assert len(groups(umis, run(U.EDIT, umis, 6))) == 1


def test_simple_error_with_zero_edits():
    umis = ["AAAAAA", "AAAAAA", "AAAAAT"]
    assert len(groups(umis, run(U.EDIT, umis, 0))) == 2


def test_adjacency_with_zero_edits():
    umis = ["AAAAAA", "AAAAAA", "AAAAAT"]
    assert len(groups(umis, run(U.ADJACENCY, umis, 0))) == 2


def test_adjacency_backward_capture():
    umis = rep("AAAA", 100) + rep("CCAA", 1) + rep("GGGG", 2) + rep("ACAA", 2)
    m = amap(umis, run(U.ADJACENCY, umis, 1))
    assert m["AAAA"] == m["CCAA"] == m["ACAA"]
    assert m["AAAA"] != m["GGGG"]


def test_paired_assigner_basic():
    umis = ["AAAA-CCCC", "CCCC-AAAA"]
    assert len(set(mid(run(U.PAIRED, umis), strip=True))) == 1


def test_paired_assigns_ab_and_ba_with_different_suffix():
    umis = ["AAAA-CCCC", "CCCC-AAAA"]
    res = run(U.PAIRED, umis)
    assert len(groups(umis, res)) == 2 and len(groups(umis, res, True)) == 1


def test_paired_assigns_ab_and_ba_with_errors():
    umis = rep("AAAA-CCCC", 3) + rep("CCCC-CAAA", 1) + rep("AAAA-GGGG", 3) + rep("GGGG-AAGA", 1)
    res = run(U.PAIRED, umis)
    assert len(groups(umis, res)) == 4 and len(groups(umis, res, True)) == 2


def test_paired_handles_errors_in_first_base_changing_lexical_ordering():
    umis = rep("GTGT-ACAC", 500) + rep("ACAC-GTGT", 460) + rep("GTGT-TCAC", 6) + rep("TCAC-GTGT", 6) + \
        rep("GTGT-TGAC", 1)
    res = run(U.PAIRED, umis)
    assert groups(umis, res) == [["ACAC-GTGT", "TCAC-GTGT"], ["GTGT-ACAC", "GTGT-TCAC", "GTGT-TGAC"]]
    assert len(groups(umis, res, True)) == 1


def test_paired_counts_ab_and_ba_together_when_constructing_graph():
    u1 = rep("AAAA-CCCC", 256) + rep("AAAA-CCCG", 64) + rep("CCCG-AAAA", 64)
    u2 = rep("AAAA-CCCC", 256) + rep("AAAA-CCCG", 128) + rep("CCCG-AAAA", 128)
    assert len(groups(u1, run(U.PAIRED, u1), True)) == 1
    assert len(groups(u2, run(U.PAIRED, u2), True)) == 2


def test_paired_fails_if_supplied_non_paired_umis():
    with pytest.raises(U.UmiError, match="is not a paired UMI"):
        run(U.PAIRED, ["AAAAAAAA", "GGGGGGGG"])


@pytest.mark.parametrize("umi,want", [("ACGT-TGCA", ("ACGT", "TGCA")), ("ACT-", ("ACT", "")), ("-ACT", ("", "ACT")),
                                      ("ACTACT", None), ("A-B-C", None)])
def test_paired_split(umi, want):
    if want is None:
        with pytest.raises(U.UmiError):
            U.split_paired(umi.encode())
    else:
        assert U.split_paired(umi.encode()) == tuple(x.encode() for x in want)


@pytest.mark.parametrize("umi,want", [("ACGT-TGCA", "TGCA-ACGT"), ("ACT-", "-ACT"), ("-ACT", "ACT-"),
                                      ("AAAA-TTTT", "TTTT-AAAA")])
def test_paired_reverse(umi, want):
    assert U.reverse_paired(umi.encode()) == want.encode()


@pytest.mark.parametrize("umi,want", [("ACGT-TGCA", "ACGT-TGCA"), ("TGCA-ACGT", "ACGT-TGCA"), ("ACT-", "-ACT"),
                                      ("-ACT", "-ACT"), ("AAAA-TTTT", "AAAA-TTTT")])
def test_paired_canonicalize(umi, want):
    assert U._canonical_mapped(umi.encode()) == want.encode()


def test_paired_count():
    keys, _ = U.prepare(U.PAIRED, M, [b"ACGT-TGCA", b"TGCA-ACGT", b"AAAA-TTTT", b"ACGT-TGCA"])
    assert {k.s: k.count for k in keys} == {b"ACGT-TGCA": 3, b"AAAA-TTTT": 1}


def test_paired_matches():
    def matches(a, b):   # matches_paired with k = 1: the oracle's byte comparator, count rule lifted
        keys = [U.Key(a.encode(), 0, 0, 1, 0), U.Key(b.encode(), 0, 0, 1, 1)]
        return U.accept(U.PAIRED, M, 1, keys, 0, 1)
    assert matches("ACGT-TGCA", "ACGT-TGCA") and matches("ACGT-TGCA", "TGCA-ACGT")
    assert matches("ACGT-TGCA", "ACTT-TGCA") and matches("ACGT-TGCA", "TGCA-ACTT")
    assert not matches("ACGT-TGCA", "AAAA-TTTT")


def test_paired_backward_capture():
    umis = rep("AAAA-XXXX", 100) + rep("CCAA-XXXX", 1) + rep("ACAA-XXXX", 2)
    m = dict(zip(umis, mid(run(U.PAIRED, umis), strip=True)))
    assert m["AAAA-XXXX"] == m["CCAA-XXXX"] == m["ACAA-XXXX"]


def test_empty_umi_list():
    assert run(U.IDENTITY, [], 0) == []


def test_single_umi():
    res = run(U.IDENTITY, ["ACGTACGT"], 0)
    assert len(res) == 1 and res[0][0] != U.NONE


def test_all_identical_umis():
    assert len(set(mid(run(U.IDENTITY, rep("ACGTACGT", 100), 0)))) == 1


def test_umis_with_empty_parts_in_paired():
    umis = ["ACT-", "-ACT", "ACT-"]
    assert len(groups(umis, run(U.PAIRED, umis), True)) == 1


def test_prop_properties_seeded():
    """prop_identity_assigns_duplicates_to_same_id, prop_every_umi_gets_assignment,
    prop_paired_reverse_is_reversible, prop_paired_canonicalize_is_idempotent / _matches_reverse,
    prop_adjacency_zero_edits_like_identity, prop_count_mismatches_symmetric / _self_is_zero."""
    rng = random.Random(5)
    for _ in range(300):
        u = "".join(rng.choice("ACGT") for _ in range(rng.randint(4, 12)))
        assert len(set(mid(run(U.IDENTITY, [u, u, u], 0)))) == 1
        v = "".join(rng.choice("ACGT") for _ in range(rng.randint(4, 12)))
        assert U.count_mismatches(u.encode(), v.encode()) == U.count_mismatches(v.encode(), u.encode())
        assert U.count_mismatches(u.encode(), u.encode()) == 0
        p = ("".join(rng.choice("ACGT") for _ in range(rng.randint(4, 8))) + "-" +
             "".join(rng.choice("ACGT") for _ in range(rng.randint(4, 8)))).encode()
        assert U.reverse_paired(U.reverse_paired(p)) == p
        c = U._canonical_mapped(p)
        assert U._canonical_mapped(c) == c == U._canonical_mapped(U.reverse_paired(p))
        umis = ["".join(rng.choice("ACGT") for _ in range(8)) for _ in range(rng.randint(1, 9))]
        assert all(kd != U.NONE for kd, _ in run(U.IDENTITY, umis, 0))
        assert len(set(mid(run(U.IDENTITY, umis, 0)))) == len(set(mid(run(U.ADJACENCY, umis, 0))))


@pytest.mark.parametrize("a,b,k,want", [
    ("ACGT", "ACGT", 0, True), ("ACGT", "ACGT", 1, True), ("ACGT", "ACGT", 5, True),                 # exact_match
    ("ACGT", "ACGC", 0, False), ("ACGT", "ACGC", 1, True), ("ACGT", "ACGC", 2, True),               # one_mismatch
    ("ACGT", "AATT", 0, False), ("ACGT", "AATT", 1, False), ("ACGT", "AATT", 2, True), ("ACGT", "AATT", 3, True),
    ("ACGT", "ACG", 5, False), ("ACG", "ACGT", 5, False), ("", "ACGT", 10, False),                  # different_lengths
    ("", "", 0, True), ("", "", 5, True),                                                           # empty_strings
    ("AAAA", "TTTT", 3, False), ("AAAA", "TTTT", 4, True), ("AAAA", "TTTT", 5, True),               # all_mismatches
    ("A" * 40, "TT" + "A" * 38, 1, False), ("A" * 40, "TT" + "A" * 38, 2, True),                    # early_exit_behavior
])
def test_matches_within_threshold(a, b, k, want):
    """test_matches_within_threshold_* (the mapped-edit byte comparator)."""
    keys = [U.Key(a.encode(), 0, 0, 1, 0), U.Key(b.encode(), 0, 0, 1, 1)]
    assert U.accept(U.EDIT, M, k, keys, 0, 1) == want


def test_simple_error_assigner_deterministic():
    umis = ["GGGGGG", "GGGGGC", "AAAAAA", "AAAAAC", "TTTTTT"]
    m = amap(umis, run(U.EDIT, umis, 1))
    assert m["GGGGGG"] == m["GGGGGC"] and m["AAAAAA"] == m["AAAAAC"]


def test_adjacency_equal_count_deterministic():
    umis = ["AAAAAA", "AAAAAA", "AAAGAC", "AAAGAC", "AAAAAC"]
    m = amap(umis, run(U.ADJACENCY, umis, 1))
    assert m["AAAAAA"] == m["AAAAAC"] and m["AAAAAA"] != m["AAAGAC"]


def test_adjacency_index_vs_linear_produces_same_results():
    """The reference's n-gram index (>= 100 keys, k = 1) against its linear scan: here the neighbour-enumeration form
    against the linear one, on the same 200 UMIs."""
    umis = [format(i, "b").replace("0", "A").replace("1", "C").rjust(8, "0")[:8] for i in range(200)]
    a = U.assign_call(U.ADJACENCY, M, 1, [u.encode() for u in umis])
    b = U.assign_call(U.ADJACENCY, M, 1, [u.encode() for u in umis], enum=True)
    assert a == b


@pytest.mark.parametrize("n", [8, 6])
def test_adjacency_threshold_zero_always_uses_linear(n):
    """also test_strategy_new_assigner_full_passes_threshold (n = 6)."""
    umis = rep("A" * n, 10) + ["A" * (n - 1) + "C"] + rep("T" * n, 5)
    m = amap(umis, run(U.ADJACENCY, umis, 1))
    assert m["A" * n] == m["A" * (n - 1) + "C"] and m["A" * n] != m["T" * n]


def test_paired_assigner_respects_index_threshold():
    umis = rep("AAAA-CCCC", 10) + ["AAAC-CCCC"] + rep("TTTT-GGGG", 5)
    m = dict(zip(umis, mid(run(U.PAIRED, umis))))
    assert m["AAAA-CCCC"] == m["AAAC-CCCC"] and m["AAAA-CCCC"] != m["TTTT-GGGG"]


def test_adjacency_large_dataset_with_indexing():
    umis = ["".join("ACGT"[(i >> (2 * p)) & 3] for p in range(8)) for i in range(150)]
    a = run(U.ADJACENCY, umis, 1)
    assert len(a) == 150 and a == U.assign_call(U.ADJACENCY, M, 1, [u.encode() for u in umis], enum=True)


# ---- parallel_assigner.rs tests -------------------------------------------------------------------------------
def _keys(seqs):
    ks = []
    for i, s in enumerate(seqs):
        bits, n = U.bitenc(s.encode())
        ks.append(U.Key(s.encode(), bits, n, 1, i))
    return ks


def _undirected(k, seqs):
    adj = U.edges(U.EDIT, UM, k, _keys(seqs))
    return sorted((i, j) for i, row in enumerate(adj) for j in row if i < j)


def test_discover_edges_parallel_k1():
    assert _undirected(1, ["AAAA", "AAAT", "TTTT"]) == [(0, 1)]


def test_discover_edges_parallel_k2():
    assert _undirected(2, ["AAAA", "AATT", "TTTT"]) == [(0, 1), (1, 2)]


def test_discover_edges_parallel_chain():
    assert _undirected(1, ["AAAA", "AAAT", "AATT"]) == [(0, 1), (1, 2)]


def test_generate_neighbors():
    """generate_neighbors of AA: 6 variants (k = 1); generate_neighbors_k(AA, 2): all 16 2-mers incl. itself."""
    allk = ["AA"] + [a + b for a in "ACGT" for b in "ACGT" if a + b != "AA"]
    k1 = {allk[j] for i, j in _undirected(1, allk) if i == 0}
    assert k1 == {"CA", "GA", "TA", "AC", "AG", "AT"}
    k2 = {allk[j] for i, j in _undirected(2, allk) if i == 0}
    assert len(k2) == 15 and {"CA", "CC", "TT"} <= k2


def ur(strategy, umis, k=1):
    return run(strategy, umis, k, UM)


def test_parallel_identity_basic():
    a = ur(U.IDENTITY, ["AAAA", "AAAA", "TTTT"], 0)
    assert a[0] == a[1] != a[2]


def test_parallel_identity_case_insensitive():
    a = ur(U.IDENTITY, ["ACGT", "acgt", "AcGt"], 0)
    assert a[0] == a[1] == a[2]


def test_parallel_identity_empty_and_single():
    assert ur(U.IDENTITY, [], 0) == [] and len(ur(U.IDENTITY, ["ACGT"], 0)) == 1


def test_parallel_identity_many_duplicates():
    a = ur(U.IDENTITY, rep("AAAAAA", 100) + rep("TTTTTT", 100) + rep("CCCCCC", 100), 0)
    assert len(set(a[:100])) == len(set(a[100:200])) == len(set(a[200:])) == 1
    assert len({a[0], a[100], a[200]}) == 3


def test_parallel_edit_basic():
    a = ur(U.EDIT, ["AAAA", "AAAT", "TTTT"])
    assert a[0] == a[1] != a[2]


def test_parallel_edit_k2():
    a = ur(U.EDIT, ["AAAA", "AATT", "TTTT"], 2)
    assert a[0] == a[1] == a[2]


def test_parallel_edit_transitive():
    a = ur(U.EDIT, ["AAAA", "AAAT", "AATT"])
    assert a[0] == a[1] == a[2]


def test_parallel_edit_empty_single_identical():
    assert ur(U.EDIT, []) == [] and len(ur(U.EDIT, ["ACGT"])) == 1
    a = ur(U.EDIT, ["ACGT", "ACGT", "ACGT"])
    assert a[0] == a[1] == a[2]


def test_parallel_edit_paired_umis_with_dash():
    a = ur(U.EDIT, ["ACGTACGT-TGCATGCA", "ACGTACGT-TGCATGCA", "ACGTACGT-TGCATGCT", "GGGGGGGG-CCCCCCCC"])
    assert a[0] == a[1] == a[2] != a[3]


def test_parallel_adjacency_paired_umis_with_dash():
    a = ur(U.ADJACENCY, ["ACGTACGT-TGCATGCA", "ACGTACGT-TGCATGCA", "ACGTACGT-TGCATGCT"])
    assert a[0] == a[1]


def test_parallel_edit_case_insensitive():
    a = ur(U.EDIT, ["ACGT", "acgt", "AcGt"])
    assert a[0] == a[1] == a[2]


def test_parallel_edit_invalid_umis():
    a = ur(U.EDIT, ["ACGT", "ACGN", "ACGT"])
    assert a[0] == a[2] != a[1]


def test_parallel_adjacency_basic():
    a = ur(U.ADJACENCY, ["AAAA", "AAAA", "AAAT"])
    assert a[0] == a[1] == a[2]


def test_parallel_adjacency_count_constraint():
    a = ur(U.ADJACENCY, rep("AAAA", 4) + ["AAAT"] + rep("TTTT", 4))
    assert len(set(a[:5])) == 1 and a[5] == a[6] and a[0] != a[5]


def test_parallel_adjacency_cascade():
    assert len(set(ur(U.ADJACENCY, rep("AAAA", 10) + rep("AAAT", 4) + rep("AATT", 1)))) == 1


def test_parallel_adjacency_deterministic_tiebreak():
    a = ur(U.ADJACENCY, ["AAAAAA", "AAAAAA", "AAAGAC", "AAAGAC", "AAAAAC"])
    assert a[0] == a[4]


def test_parallel_adjacency_empty_and_single():
    assert ur(U.ADJACENCY, []) == [] and len(ur(U.ADJACENCY, ["ACGT"])) == 1


def test_parallel_paired_basic():
    a = ur(U.PAIRED, ["AAAA-CCCC", "CCCC-AAAA"])
    assert {a[0][0], a[1][0]} == {U.A, U.B} and a[0][1] == a[1][1]


def test_parallel_paired_with_errors():
    a = ur(U.PAIRED, ["AAAA-CCCC", "AAAA-CCCC", "AAAT-CCCC"])
    assert all(kd in (U.A, U.B) for kd, _ in a) and len({i for _, i in a}) == 1


@pytest.mark.parametrize("umi,want", [("AAAA-CCCC", "AAAA-CCCC"), ("CCCC-AAAA", "AAAA-CCCC"), ("TTTT-AAAA", "AAAA-TTTT"),
                                      ("aaaa-cccc", "AAAA-CCCC"), ("cccc-aaaa", "AAAA-CCCC"), ("Tttt-Aaaa", "AAAA-TTTT")])
def test_parallel_paired_canonicalization(umi, want):
    """also test_parallel_paired_canonicalization_mixed_case."""
    assert U._canonical_unmapped(umi.encode()) == want.encode()
    assert U._canonical_unmapped(b"aaaa-CCCC") == U._canonical_unmapped(b"AAAA-cccc")


def test_edit_equivalence_with_sequential():
    a = ur(U.EDIT, ["AAAAAA", "AAAAAT", "AAAATT", "TTTTTT", "TTTTTA", "GGGGGG"])
    assert a[0] == a[1] == a[2] and a[3] == a[4]
    assert len({a[5], a[0], a[3]}) == 3


# ---- fgumi-umi lib.rs: MoleculeId ----------------------------------------------------------------------------
@pytest.mark.parametrize("kind,i,base,want", [(U.NONE, 0, 0, ""), (U.SINGLE, 42, 0, "42"), (U.A, 42, 0, "42/A"),
                                              (U.B, 42, 0, "42/B"), (U.SINGLE, 5, 100, "105"), (U.A, 5, 100, "105/A"),
                                              (U.B, 5, 100, "105/B"), (U.NONE, 5, 100, "")])
def test_molecule_id_to_string_with_offset(kind, i, base, want):
    assert U.mi_string(kind, i, base) == want


# ---- group.rs -----------------------------------------------------------------------------------------------
def test_umi_for_read_assigns_ab_prefixes_by_coordinates():
    r1 = U.umi_for_read(b"AAA-TTT", True, U.PAIRED, M, 1)
    r2 = U.umi_for_read(b"AAA-TTT", False, U.PAIRED, M, 1)
    assert b"AAA" in r1 and b"TTT" in r1 and b"-" in r1 and r1 != r2


def test_umi_for_read_handles_absent_umi_ends():
    left = U.umi_for_read(b"-TTT", True, U.PAIRED, M, 1)
    right = U.umi_for_read(b"AAA-", True, U.PAIRED, M, 1)
    assert b"-" in left and b"TTT" in left and b"AAA" in right and b"-" in right


def test_umi_for_read_uppercase_for_non_paired():
    assert U.umi_for_read(b"acgtacgt", True, U.IDENTITY, M, 0) == b"ACGTACGT"


def test_truncate_umis_to_minimum_length():
    t = U.truncate_umis([b"AAAAAA", b"AAAAA", b"AAAAAAA"], 5)
    assert len(t) == 3 and all(len(u) == 5 for u in t)


def test_truncate_umis_none_returns_unchanged():
    assert U.truncate_umis([b"AAAAAA", b"AAAAA"], None) == [b"AAAAAA", b"AAAAA"]


def test_truncate_umis_fails_when_too_short():
    with pytest.raises(U.UmiError):
        U.truncate_umis([b"AAAAAA", b"AAAA"], 6)
