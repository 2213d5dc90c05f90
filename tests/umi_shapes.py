"""UMI calls at the shapes real batches reach, and a fast exact reference for their capture lists.

`capture_lists` is the oracle's `accept` rule (oracle/umi_oracle.py) over every pair of a call's key table, in numpy
and in blocks of queries, so that calls of thousands of keys can be checked: the oracle's own `edges` is pure Python
and quadratic.  The generators are seeded and build calls with an exact number of unique keys:
  byte_call        mapped edit / mapped paired (the byte comparator): clusters of close strings, 8 to 64 bases; the
                   paired form has similar halves and a dash that moves, so that edges found only through the
                   query's reversed form exist between keys whose dashes differ
  twobit_call      the 2-bit comparator at one length (31 and 32 bases reach the top BitEnc bits)
  mixed_call       unmapped calls of 1..5 bases, where BitEncs collide across lengths (A, AA, AAA all encode to 0)
  interleaved_batch  several enumeration-size calls mixed with small, edge-free, single-key and empty calls
"""
from __future__ import annotations

import random
from typing import Dict, List, Sequence

import numpy as np

from oracle import umi_oracle as U
from tests import umi_cases

ACGT = np.frombuffer(b"ACGT", np.uint8)
_EVEN = np.uint64(0x5555555555555555)
_BLOCK_ELEMS = 1 << 22          # query block x keys (x string length for bytes) per step


def enum_min_keys(k: int) -> int:
    """The product's default enumeration threshold (unique keys of a call) for a 2-bit call at k <= 2."""
    return 1000 if k <= 1 else 8000


# ---- the reference -------------------------------------------------------------------------------------------------
def _lists(r: np.ndarray, c: np.ndarray, n_rows: int) -> List[List[int]]:
    """Pairs (row, col), rows ascending and cols ascending within a row -> one list of cols per row."""
    vals = c.tolist()
    cuts = np.searchsorted(r, np.arange(1, n_rows)).tolist()
    out, lo = [], 0
    for hi in cuts + [len(vals)]:
        out.append(vals[lo:hi])
        lo = hi
    return out


def capture_lists_by_k(strategy: int, rules: int, ks: Sequence[int], keys: Sequence[U.Key]) -> Dict[int, List[List[int]]]:
    """{k: capture lists} for a call's key table (U.prepare), every k from one pass over the pairs.  The same lists as
    U.edges: ascending key indices per key."""
    n = len(keys)
    out = {k: [[] for _ in range(n)] for k in ks}
    if n < 2:
        return out
    directed = strategy in (U.ADJACENCY, U.PAIRED)
    byte = U.uses_bytes(strategy, rules)
    count = np.array([x.count for x in keys], np.int64)
    length = np.array([len(x.s) if byte else x.len for x in keys], np.int64)
    if not byte:
        bits = np.array([x.bits for x in keys], np.uint64)
        last = np.array([x.last for x in keys], bool)
    for L in np.unique(length).tolist():
        idx = np.nonzero(length == L)[0]                 # a key only meets keys of its own length
        if byte:
            s = np.frombuffer(b"".join(keys[i].s for i in idx), np.uint8).reshape(len(idx), L)
            if strategy == U.PAIRED:                      # the query's reversed form, around its own dash
                rev = np.frombuffer(b"".join(U.reverse_paired(keys[i].s) for i in idx), np.uint8).reshape(len(idx), L)
        step = max(1, _BLOCK_ELEMS // (len(idx) * (max(L, 1) if byte else 1)))
        for q0 in range(0, len(idx), step):
            qi = idx[q0:q0 + step]
            if byte:
                d = (s[q0:q0 + step, None, :] != s[None, :, :]).sum(-1, dtype=np.int32)
                if strategy == U.PAIRED:
                    d = np.minimum(d, (rev[q0:q0 + step, None, :] != s[None, :, :]).sum(-1, dtype=np.int32))
            else:
                x = bits[qi, None] ^ bits[None, idx]
                d = np.bitwise_count((x | (x >> np.uint64(1))) & _EVEN)   # a position differs when either bit does
            r, c = np.nonzero(d <= max(ks))                   # few pairs pass the distance: the rules run on those
            dist, i, j = d[r, c], qi[r], idx[c]
            ok = i != j
            if not byte:                                      # an edge (a, b), a < b, only where b is the last key
                ok &= np.where(i < j, last[j], last[i])       # of its BitEnc
            if directed:
                ok &= count[j] <= count[i] // 2 + 1
            for k in ks:
                m = ok & (dist <= k)
                if not byte and k == 1:
                    m &= dist > 0                             # k = 1 enumerates distance exactly 1
                for q, row in zip(qi.tolist(), _lists(r[m], j[m], len(qi))):
                    out[k][q] = row
    return out


def capture_lists(strategy: int, rules: int, k: int, keys: Sequence[U.Key]) -> List[List[int]]:
    return capture_lists_by_k(strategy, rules, (k,), keys)[k]


def assign_call(strategy, rules, k, umis, adj=None):
    """U.assign_call with the capture lists from `capture_lists` (or given): the oracle's key table and rules."""
    keys, key_of = U.prepare(strategy, rules, umis)
    if adj is None:
        adj = capture_lists(strategy, rules, k, keys) if U.needs_edges(strategy, keys) else [[]] * len(keys)
    return U.resolve(strategy, rules, umis, keys, key_of, adj)


def assign_groups(strategy, rules, k, groups):
    """U.assign_groups over `assign_call`: (kinds, ids, group MI counts), ids numbered as U.assign_groups does."""
    kinds, ids, counts = [], [], []
    for g in groups:
        base, mx = 0, -1
        for call in g:
            res = assign_call(strategy, rules, k, call)
            if rules == U.MAPPED:
                res = [(kd, i + base) for kd, i in res]
                base = max([base] + [i + 1 for kd, i in res if kd != U.NONE])
            for kd, i in res:
                kinds.append(kd)
                ids.append(i if kd != U.NONE else 0)
                if kd != U.NONE:
                    mx = max(mx, i)
        counts.append(mx + 1)
    return kinds, ids, counts


# ---- generators ----------------------------------------------------------------------------------------------------
def _text(codes: np.ndarray) -> List[bytes]:
    return [bytes(r) for r in ACGT[codes]]


def _clustered(rng: np.random.Generator, n: int, L: int, per_centre: int = 4) -> np.ndarray:
    """n base rows of length L in clusters: each row is a random centre with each base substituted with probability
    1.5 / L, so close pairs exist at every length."""
    centres = rng.integers(0, 4, size=(max(1, n // per_centre), L), dtype=np.uint8)
    rows = centres[rng.integers(0, len(centres), size=n)]
    hit = rng.random(rows.shape) < min(1.0, 1.5 / L)
    return np.where(hit, (rows + rng.integers(1, 4, size=rows.shape, dtype=np.uint8)) % 4, rows).astype(np.uint8)


def _take_keys(strategy, rules, pool: Sequence[bytes], n_keys: int, rng: np.random.Generator) -> List[bytes]:
    """The UMIs of `pool` whose keys (U.prepare) are among the first n_keys keys to appear, each key repeated to a
    count of 1..4, shuffled: a call with exactly n_keys unique keys."""
    keys, key_of = U.prepare(strategy, rules, pool)
    if len(keys) < n_keys:
        raise ValueError(f"pool has {len(keys)} keys, {n_keys} wanted")
    chosen = sorted(range(len(keys)), key=lambda i: keys[i].first)[:n_keys]
    want = dict(zip(chosen, rng.integers(1, 5, size=n_keys).tolist()))
    out, have = [], {}
    for u, ki in zip(pool, key_of):
        if ki in want and have.get(ki, 0) < want[ki]:
            out.append(u)
            have[ki] = have.get(ki, 0) + 1
    firsts = {ki: pool[keys[ki].first] for ki in chosen}
    for ki, c in want.items():
        out += [firsts[ki]] * (c - have[ki])
    return [out[i] for i in rng.permutation(len(out))]


def byte_call(seed: int, strategy: int, n_keys: int, L: int) -> List[bytes]:
    """A mapped edit or mapped paired call (the byte comparator) with exactly n_keys unique keys of L bases.  Paired
    UMIs are raw "X-Y" strings of L bases in all, around molecules whose halves differ in one base and whose dash sits
    within two places of the middle; half of the reads carry "Y-X".  A key's reversed form is then often close to
    another key whose dash is elsewhere."""
    rng = np.random.default_rng(seed)
    n_pool = 3 * n_keys + 64
    if strategy == U.EDIT:
        return _take_keys(U.EDIT, U.MAPPED, _text(_clustered(rng, n_pool, L)), n_keys, rng)
    h, n_mol = L // 2, max(1, n_pool // 4)
    x = rng.integers(0, 4, size=(n_mol, h), dtype=np.uint8)
    y = np.concatenate([x, rng.integers(0, 4, size=(n_mol, L - 2 * h), dtype=np.uint8)], axis=1)
    at = rng.integers(0, y.shape[1], size=n_mol)
    y[np.arange(n_mol), at] = (y[np.arange(n_mol), at] + rng.integers(1, 4, size=n_mol, dtype=np.uint8)) % 4
    mol_dash = np.clip(h + rng.integers(-2, 3, size=n_mol), 1, L - 1)
    pick = rng.integers(0, n_mol, size=n_pool)
    rows = np.concatenate([x, y], axis=1)[pick]
    hit = rng.random(rows.shape) < 1.0 / L               # about one substituted base per read
    rows = np.where(hit, (rows + rng.integers(1, 4, size=rows.shape, dtype=np.uint8)) % 4, rows).astype(np.uint8)
    dash = np.where(rng.random(n_pool) < 0.8, mol_dash[pick], np.clip(h + rng.integers(-2, 3, size=n_pool), 1, L - 1))
    pool = []
    for b, d, sw in zip(_text(rows), dash.tolist(), (rng.random(n_pool) < 0.5).tolist()):
        u = b[:d] + b"-" + b[d:]
        pool.append(U.reverse_paired(u) if sw else u)
    return _take_keys(U.PAIRED, U.MAPPED, pool, n_keys, rng)


def twobit_call(seed: int, strategy: int, rules: int, n_keys: int, L: int, dash_rate: float = 0.2) -> List[bytes]:
    """A call for the 2-bit comparator with exactly n_keys unique keys of L bases.  Under the unmapped rules a share of
    the UMIs carry a dash (several keys per BitEnc for adjacency and paired); paired UMIs are "X-Y" around a dash
    near the middle."""
    rng = np.random.default_rng(seed)
    raw = _text(_clustered(rng, 3 * n_keys + 64, L))
    pool = []
    for u, r, d in zip(raw, rng.random(len(raw)).tolist(), rng.integers(1, max(2, L), size=len(raw)).tolist()):
        if strategy == U.PAIRED:
            d = min(max(1, L // 2 + d % 3 - 1), L - 1) if L > 1 else 0
            u = u[:d] + b"-" + u[d:]
        elif rules == U.UNMAPPED and L > 1 and r < dash_rate:
            u = u[:d] + b"-" + u[d:]
        pool.append(u)
    return _take_keys(strategy, rules, pool, n_keys, rng)


def mixed_call(seed: int, strategy: int, n_keys: int) -> List[bytes]:
    """An unmapped call of UMIs of 1..5 bases with exactly n_keys unique keys.  Every length is equally likely, so
    short and long keys whose BitEncs collide (A / AA / AAA, C / CA, ...) are both present; adjacency UMIs carry a dash
    now and then, paired UMIs are "X-Y" with X or Y possibly empty."""
    rng = np.random.default_rng(seed)
    n_pool = 16 * n_keys + 2000
    lens = rng.integers(1, 6, size=n_pool)
    codes = rng.integers(0, 4, size=(n_pool, 5), dtype=np.uint8)
    pool = []
    for row, L, r, d in zip(_text(codes), lens.tolist(), rng.random(n_pool).tolist(),
                            rng.integers(0, 6, size=n_pool).tolist()):
        u = row[:L]
        if strategy == U.PAIRED or (strategy == U.ADJACENCY and r < 0.3 and L > 1):
            d = min(d, L) if strategy == U.PAIRED else 1 + d % (L - 1)
            u = u[:d] + b"-" + u[d:]
        pool.append(u)
    return _take_keys(strategy, U.UNMAPPED, pool, n_keys, rng)


def _edge_free_call(rng: random.Random, strategy: int, rules: int, k: int, L: int = 16, n: int = 12) -> List[bytes]:
    """n keys of L bases with no edge between them: every key its own molecule.  Paired UMIs get a dash in the
    middle."""
    while True:
        keys = [bytes(rng.choice(b"ACGT") for _ in range(L)) for _ in range(n)]
        if strategy == U.PAIRED:
            keys = [u[:L // 2] + b"-" + u[L // 2:] for u in keys]
        umis = [u for u in keys for _ in range(rng.randint(1, 3))]
        table, _ = U.prepare(strategy, rules, umis)
        if len(table) == n and not any(capture_lists(strategy, rules, k, table)):
            return umis


def interleaved_batch(seed: int, strategy: int, rules: int, k: int, n_groups: int = 3, n_enum: int = 3):
    """groups -> calls -> UMIs: n_enum calls past the enumeration threshold at different lengths and sizes, spread over
    the groups, each group also holding small noisy calls, an edge-free call, a single-key call and an empty call, in a
    seeded order."""
    rng = random.Random(seed)
    groups = [[] for _ in range(n_groups)]
    lengths = [10, 12, 14] if k <= 1 else [9, 10, 12]
    for e in range(n_enum):
        n_keys = enum_min_keys(k) + rng.randrange(0, enum_min_keys(k) // 2)
        L = lengths[e % len(lengths)]
        groups[e % n_groups].append(twobit_call(seed * 31 + e, strategy, rules, n_keys, L))
    for g in groups:
        L, n_small = rng.choice([6, 8, 12]), len(g) + 3 + rng.randrange(3)
        while len(g) < n_small:
            c = umi_cases.noisy_call(rng, strategy, rules, k, length=L, max_umis=rng.choice([5, 40, 120]))
            if umi_cases.oracle_ok(strategy, rules, k, c) is not None:
                g.append(c)
        free = _edge_free_call(rng, strategy, rules, k)
        g += [free, free[:1] * 3, []]
        rng.shuffle(g)
    return groups


def n_enum_calls(strategy, rules, k, groups) -> int:
    """Calls of a batch that take the enumeration form at the product's default threshold."""
    if U.uses_bytes(strategy, rules) or k > 2:
        return 0
    return sum(len(U.prepare(strategy, rules, c)[0]) >= enum_min_keys(k) for g in groups for c in g)
