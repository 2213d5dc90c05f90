"""The host half of UMI assignment against oracle/umi_oracle.py, with edges the oracle supplies: fgb_host_umi_prepare
(the key table the device receives), fgb_host_umi_resolve (the rules applied to the capture lists) and
fgb_host_umi_for_read, on seeded random calls of both rule families, all four strategies and k = 0..3; and the
oracle's two edge forms against each other.  CPU only."""
import ctypes as C
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import umi_oracle as U      # noqa: E402
from tests import umi_cases             # noqa: E402

STRATS = [U.IDENTITY, U.EDIT, U.ADJACENCY, U.PAIRED]
NAMES = {U.IDENTITY: "identity", U.EDIT: "edit", U.ADJACENCY: "adjacency", U.PAIRED: "paired"}


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import lib as L
    return L


def _opt(L, strategy, rules, k, min_len=None):
    return L.FgbUmiOptions(strategy, k, rules, min_len or 0, 1, 0)


def product_prepare(L, o, umis):
    from fgumi_b200.umi import KEY_DTYPE, pack_umis
    blob, off = pack_umis(umis)
    n = len(umis)
    keys = np.zeros(max(n, 1), KEY_DTYPE)
    kb = np.zeros(max(int(off[-1]), 1), np.uint8)
    key_of = np.zeros(max(n, 1), np.uint32)
    nk = C.c_uint64()
    st = L.load().fgb_host_umi_prepare(C.byref(o), blob.ctypes.data, off.ctypes.data, n, keys.ctypes.data,
                                       C.byref(nk), kb.ctypes.data, key_of.ctypes.data)
    return st, blob, off, keys[:nk.value], kb, key_of[:n]


def product_resolve(L, o, blob, off, keys, kb, key_of, adj):
    n = len(off) - 1
    eo = np.zeros(len(keys) + 1, np.uint64)
    eo[1:] = np.cumsum([len(a) for a in adj]) if len(adj) else []
    e = np.array([j for a in adj for j in a] or [0], np.uint32)
    ids = np.zeros(max(n, 1), np.uint64)
    kinds = np.zeros(max(n, 1), np.uint8)
    keys = np.ascontiguousarray(keys)
    key_of = np.ascontiguousarray(key_of)
    st = L.load().fgb_host_umi_resolve(C.byref(o), blob.ctypes.data, off.ctypes.data, n, keys.ctypes.data, len(keys),
                                       kb.ctypes.data, key_of.ctypes.data, eo.ctypes.data, e.ctypes.data,
                                       ids.ctypes.data, kinds.ctypes.data)
    assert st == 0
    return [(int(k), int(i)) for k, i in zip(kinds[:n], ids[:n])]


def check_call(L, strategy, rules, k, umis, min_len=None):
    o = _opt(L, strategy, rules, k, min_len)
    st, blob, off, keys, kb, key_of = product_prepare(L, o, umis)
    try:
        tumis = U.truncate_umis(umis, min_len)
        okeys, okey_of = U.prepare(strategy, rules, tumis)
    except U.UmiError:
        assert st == L.FGB_ERR_INVALID_ARG
        return None
    assert st == 0, umis
    got = [(bytes(kb[int(x["str_off"]):int(x["str_off"]) + int(x["str_len"])]), int(x["bits"]), int(x["len"]),
            int(x["count"]), int(x["first"]), bool(x["flags"] & 1)) for x in keys]
    want = [q.tup() for q in okeys]
    if U.uses_bytes(strategy, rules) or strategy == U.IDENTITY:   # BitEncs only matter to the 2-bit comparator
        got = [g[:1] + g[3:] for g in got]
        want = [w[:1] + w[3:] for w in want]
    assert got == want, umis
    assert [(-1 if x == 0xFFFFFFFF else int(x)) for x in key_of] == okey_of
    adj = U.edges(strategy, rules, k, okeys) if U.needs_edges(strategy, okeys) else [[] for _ in okeys]
    res = product_resolve(L, o, blob, off, keys, kb, key_of, adj)
    assert res == U.resolve(strategy, rules, tumis, okeys, okey_of, adj), umis
    return res


@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
@pytest.mark.parametrize("strategy", STRATS)
@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_prepare_resolve_random_calls(lib, strategy, rules, k):
    if strategy == U.IDENTITY and k:
        pytest.skip("identity takes edits = 0 only")
    n = 1300 if strategy == U.IDENTITY else 320     # ~10 k calls over the grid
    for i, umis in enumerate(umi_cases.calls(1000 * strategy + 10 * rules + k, strategy, rules, k, n)):
        check_call(lib, strategy, rules, k, umis, min_len=None if i % 7 else 2)


def test_prepare_errors(lib):
    o = _opt(lib, U.ADJACENCY, U.MAPPED, 1)
    assert product_prepare(lib, o, [b"ACGT", b"ACG"])[0] == lib.FGB_ERR_INVALID_ARG       # mixed base lengths
    assert product_prepare(lib, o, [b"ACGT", b"ACGN"])[0] == 0                             # the N UMI has no key
    assert product_prepare(lib, o, [b"ACGT", b"acgt", b"A-CGT"])[0] == 0                   # one key
    for rules in (U.MAPPED, U.UNMAPPED):
        o = _opt(lib, U.PAIRED, rules, 1)
        assert product_prepare(lib, o, [b"AC-GT", b"ACGT"])[0] == lib.FGB_ERR_INVALID_ARG
        assert product_prepare(lib, o, [b"A-C-GT"])[0] == lib.FGB_ERR_INVALID_ARG
    o = _opt(lib, U.IDENTITY, U.MAPPED, 0, 5)
    assert product_prepare(lib, o, [b"AAAAAA", b"AAAA"])[0] == lib.FGB_ERR_INVALID_ARG
    assert product_prepare(lib, _opt(lib, U.IDENTITY, U.MAPPED, 1), [b"A"])[0] == lib.FGB_ERR_INVALID_ARG


@pytest.mark.parametrize("strategy", STRATS)
@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
def test_umi_for_read(lib, strategy, rules):
    from fgumi_b200.umi import umi_for_read
    rng = random.Random(strategy * 2 + rules)
    for _ in range(300):
        k = rng.randint(0, 3) if strategy != U.IDENTITY else 0
        u = "".join(rng.choice("ACGTacgtN-") for _ in range(rng.randint(0, 12)))
        r1 = rng.random() < 0.5
        try:
            want = U.umi_for_read(u.encode(), r1, strategy, rules, k)
        except U.UmiError:
            with pytest.raises(Exception):
                umi_for_read(u, r1, NAMES[strategy], k, "mapped" if rules == U.MAPPED else "unmapped")
            continue
        assert umi_for_read(u, r1, NAMES[strategy], k, "mapped" if rules == U.MAPPED else "unmapped") == want


@pytest.mark.parametrize("rules", [U.MAPPED, U.UNMAPPED])
@pytest.mark.parametrize("strategy", [U.EDIT, U.ADJACENCY, U.PAIRED])
@pytest.mark.parametrize("k", [0, 1, 2])
def test_oracle_linear_equals_enumeration(strategy, rules, k):
    if U.uses_bytes(strategy, rules):
        pytest.skip("the byte comparator has no enumeration form")
    for umis in umi_cases.calls(7 + strategy * 3 + rules + 11 * k, strategy, rules, k, 150):
        try:
            keys, _ = U.prepare(strategy, rules, umis)
        except U.UmiError:
            continue
        assert U.edges(strategy, rules, k, keys) == U.edges_enum(strategy, rules, k, keys)
