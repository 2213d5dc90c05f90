"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Restatement (pure Python) of the UMI assigners exactly as `fgumi group` uses them, and of the two
input-side helpers in front of them.  Citations are relative to the fgumi 0.2.0 source tree:
  assigner.rs           crates/fgumi-umi/src/assigner.rs        (mapped data, the default)
  parallel_assigner.rs  src/lib/umi/parallel_assigner.rs        (`group --allow-unmapped`, group.rs:1073-1093)
  bitenc.rs             crates/fgumi-dna/src/bitenc.rs
  lib.rs                crates/fgumi-umi/src/lib.rs             (MoleculeId)
  group.rs              src/lib/commands/group.rs
The two rule families are NOT identical despite their doc comments, so both are restated.

Every call is split the way the product splits it: `prepare` builds the unique-key table (what the
device receives), `edges` the capture lists the device emits (brute force, or `edges_enum`, the
neighbour-enumeration form), `resolve` the order-dependent rules on the host.  `assign` strings them.
Upper-casing is ASCII only (the reference uses Unicode `to_uppercase`).
"""
from __future__ import annotations

from itertools import combinations, product
from typing import Dict, List, Optional, Sequence, Tuple

IDENTITY, EDIT, ADJACENCY, PAIRED = 0, 1, 2, 3
MAPPED, UNMAPPED = 0, 1
NONE, SINGLE, A, B = 0, 1, 2, 3              # MoleculeId variants, lib.rs:26-36
STRATEGIES = {"identity": IDENTITY, "edit": EDIT, "adjacency": ADJACENCY, "paired": PAIRED}


class UmiError(ValueError):
    """Where the reference panics (assert!) or bails: the product fails the batch instead."""


def upper(s: bytes) -> bytes:
    return s.upper()                          # ASCII only: bytes.upper() leaves other bytes alone


# ---- bitenc.rs:32-90 from_umi_str: ACGT in either case, '-' skipped, anything else or > 32 bases -> None
_CODE = {ord(c): i for i, c in enumerate("ACGT")}
_CODE.update({ord(c): i for i, c in enumerate("acgt")})


def bitenc(s: bytes) -> Optional[Tuple[int, int]]:
    bits, n = 0, 0
    for b in s:
        c = _CODE.get(b)
        if c is not None:
            if n >= 32:
                return None
            bits |= c << (2 * n)
            n += 1
        elif b != ord("-"):
            return None
    return bits, n


def hamming2(a: int, b: int) -> int:           # bitenc.rs:111-125
    d = a ^ b
    return bin(((d & 0xAAAAAAAAAAAAAAAA) >> 1) | (d & 0x5555555555555555)).count("1")


def count_mismatches(a: bytes, b: bytes) -> int:   # assigner.rs:644-649
    if len(a) != len(b):
        return 1 << 64
    return sum(x != y for x, y in zip(a, b))


def split_paired(u: bytes) -> Tuple[bytes, bytes]:  # assigner.rs:1663-1678 (`split('-').count() == 2`)
    parts = u.split(b"-")
    if len(parts) != 2:
        raise UmiError(f"UMI {u!r} is not a paired UMI")
    return parts[0], parts[1]


def reverse_paired(u: bytes) -> bytes:           # assigner.rs:1695-1703
    a, b = split_paired(u)
    return b + b"-" + a


# ---- input side, group.rs:300-364 --------------------------------------------------------------
def umi_for_read(umi: bytes, is_r1_earlier: bool, strategy: int, rules: int, edits: int) -> bytes:
    if strategy != PAIRED:
        return upper(umi)                      # :301-308
    a, b = split_paired(umi)                   # :311-317 bails on != 2 segments
    if rules == UNMAPPED:
        return upper(umi)                      # :320-322 ParallelPairedAssigner: no prefixes
    lo, hi = b"a" * (edits + 1), b"b" * (edits + 1)   # assigner.rs:1621-1628
    if is_r1_earlier:
        return lo + b":" + a + b"-" + hi + b":" + b   # :330-337
    return hi + b":" + a + b"-" + lo + b":" + b       # :339-345


def truncate_umis(umis: Sequence[bytes], min_len: Optional[int]) -> List[bytes]:
    if not min_len or not umis:              # an empty call never gets here (group.rs:436-438)
        return list(umis)
    m = min((len(u) for u in umis), default=0)
    if m < min_len:                           # :357-360 bails
        raise UmiError(f"UMI found that had shorter length than expected ({m} < {min_len})")
    return [u[:min_len] for u in umis]


# ---- the key table ---------------------------------------------------------------------------------
class Key:
    __slots__ = ("s", "bits", "len", "count", "first", "last")

    def __init__(self, s, bits, n, count, first):
        self.s, self.bits, self.len, self.count, self.first, self.last = s, bits, n, count, first, True

    def tup(self):
        return (self.s, self.bits, self.len, self.count, self.first, self.last)


def _count(keys_in: Sequence[Optional[bytes]]) -> Dict[bytes, List[int]]:
    d: Dict[bytes, List[int]] = {}
    for i, k in enumerate(keys_in):
        if k is None:
            continue
        if k in d:
            d[k][0] += 1
        else:
            d[k] = [1, i]
    return d


def _canonical_mapped(u: bytes) -> bytes:        # assigner.rs:1721-1736: compares the PARTS
    a, b = split_paired(u)
    return u if a <= b else b + b"-" + a


def _canonical_unmapped(u: bytes) -> bytes:      # parallel_assigner.rs:609-616: compares whole strings
    up = upper(u)
    r = reverse_paired(up)
    return r if r < up else up


def prepare(strategy: int, rules: int, umis: Sequence[bytes]) -> Tuple[List[Key], List[int]]:
    """Unique keys of one call in the order the rules number / sort them, and key_of[input] (-1 = invalid).
    Raises UmiError where the reference panics."""
    n = len(umis)
    if strategy == IDENTITY:                  # assigner.rs:857-878, parallel_assigner.rs:272-316
        ks = [upper(u) for u in umis]
        d = _count(ks)
        order = sorted(d)
    elif strategy == EDIT and rules == MAPPED:  # assigner.rs:936-1008: raw strings, case-sensitive
        ks = list(umis)
        d = _count(ks)
        order = sorted(d)
    elif strategy == EDIT:                    # parallel_assigner.rs:352-418: BitEnc of the upper-cased UMI
        ks = []
        for u in umis:
            e = bitenc(upper(u))
            ks.append(None if e is None else e)
        d = _count(ks)
        order = sorted(d, key=lambda e: d[e][1])     # first appearance
        keys = [Key(upper(umis[d[e][1]]), e[0], e[1], d[e][0], d[e][1]) for e in order]
        idx = {e: i for i, e in enumerate(order)}
        return keys, [-1 if k is None else idx[k] for k in ks]
    elif strategy == ADJACENCY and rules == MAPPED:   # assigner.rs:1435-1491
        ks = [bitenc(u) for u in umis]
        d = _count(ks)
        order = sorted(d, key=lambda e: (-d[e][0], umis[d[e][1]]))   # :1479 raw string of the first occurrence
        keys = [Key(umis[d[e][1]], e[0], e[1], d[e][0], d[e][1]) for e in order]
        idx = {e: i for i, e in enumerate(order)}
        if len(keys) > 1 and any(k.len != keys[0].len for k in keys):
            raise UmiError("Multiple UMI lengths")          # :1494-1502
        return keys, [-1 if k is None else idx[k] for k in ks]
    elif strategy == ADJACENCY:               # parallel_assigner.rs:454-483
        ks = [upper(u) for u in umis]
        d0 = _count(ks)
        d = {s: v for s, v in d0.items() if bitenc(s) is not None}
        order = sorted(d, key=lambda s: (-d[s][0], s))
    elif rules == MAPPED:                     # PAIRED, assigner.rs:1787-1799
        for u in umis:
            split_paired(u)
        ks = [_canonical_mapped(u) for u in umis]
        d = _count(ks)
        order = sorted(d, key=lambda s: (-d[s][0], s))
    else:                                     # PAIRED unmapped, parallel_assigner.rs:625-657
        for u in umis:
            split_paired(u)
        ks = [_canonical_unmapped(u) for u in umis]
        d0 = _count(ks)
        d = {s: v for s, v in d0.items() if bitenc(s) is not None}
        order = sorted(d, key=lambda s: (-d[s][0], s))
    keys = []
    for s in order:
        e = bitenc(s) or (0, 0)
        keys.append(Key(s, e[0], e[1], d[s][0], d[s][1]))
    if rules == UNMAPPED and strategy in (ADJACENCY, PAIRED):
        last: Dict[Tuple[int, int], int] = {}
        for i, k in enumerate(keys):          # parallel_assigner.rs:184-185: BitEnc -> index, last index wins
            last[(k.bits, k.len)] = i
        for i, k in enumerate(keys):
            k.last = last[(k.bits, k.len)] == i
    idx = {s: i for i, s in enumerate(order)}
    return keys, [idx.get(k, -1) if k is not None else -1 for k in ks]


def needs_edges(strategy: int, keys: Sequence[Key]) -> bool:
    return strategy != IDENTITY and len(keys) >= 2


def uses_bytes(strategy: int, rules: int) -> bool:
    """Mapped edit and mapped paired compare bytes; everything else compares BitEncs."""
    return rules == MAPPED and strategy in (EDIT, PAIRED)


def accept(strategy: int, rules: int, k: int, keys: Sequence[Key], i: int, j: int) -> bool:
    """Is j in i's capture list?  Edit: undirected edges; adjacency / paired: the count rule applies."""
    if i == j:
        return False
    qi, kj = keys[i], keys[j]
    if uses_bytes(strategy, rules):
        ok = count_mismatches(qi.s, kj.s) <= k          # matches_within_threshold, assigner.rs:683-730
        if not ok and strategy == PAIRED:               # matches_paired, assigner.rs:1773-1783
            ok = count_mismatches(reverse_paired(qi.s), kj.s) <= k
        if not ok:
            return False
    else:
        if qi.len != kj.len:
            return False
        dd = hamming2(qi.bits, kj.bits)
        # discover_edges_parallel_k (parallel_assigner.rs:180-242): k == 1 enumerates distance exactly 1,
        # every other k enumerates 0..=k (the UMI itself included); an edge (a, b), a < b, exists only when b
        # is the LAST key of its BitEnc (the lookup map's last index wins).  Mapped adjacency compares every
        # pair (assigner.rs:1237-1247) but its keys are unique BitEncs, so the same rule gives its edges.
        if dd > k or (dd == 0 and k == 1):
            return False
        if not ((i < j and kj.last) or (j < i and qi.last)):
            return False
    if strategy in (ADJACENCY, PAIRED) and kj.count > qi.count // 2 + 1:   # assigner.rs:1193, 1214
        return False
    return True


def edges(strategy: int, rules: int, k: int, keys: Sequence[Key]) -> List[List[int]]:
    """Brute force: every pair."""
    n = len(keys)
    return [[j for j in range(n) if accept(strategy, rules, k, keys, i, j)] for i in range(n)]


def edges_enum(strategy: int, rules: int, k: int, keys: Sequence[Key]) -> List[List[int]]:
    """Neighbour enumeration (2-bit comparator): every variant within the distance set, looked up."""
    assert not uses_bytes(strategy, rules)
    table: Dict[Tuple[int, int], List[int]] = {}
    for i, key in enumerate(keys):
        table.setdefault((key.bits, key.len), []).append(i)
    out = []
    for i, key in enumerate(keys):
        found = set()
        for dist in range(0 if k != 1 else 1, k + 1):
            for pos in combinations(range(key.len), dist):
                for subs in product(range(1, 4), repeat=dist):
                    v = key.bits
                    for p, s in zip(pos, subs):
                        v ^= s << (2 * p)
                    for j in table.get((v, key.len), ()):
                        if accept(strategy, rules, k, keys, i, j):
                            found.add(j)
        out.append(sorted(found))
    return out


# ---- resolve -------------------------------------------------------------------------------------------
def _bfs_roots(keys, adj):
    """Roots in sorted order; a child must be unassigned (assigner.rs:1182-1258, parallel_assigner.rs:506-539)."""
    n = len(keys)
    comp = [-1] * n
    roots = []
    for r in range(n):
        if comp[r] >= 0:
            continue
        c = len(roots)
        roots.append(r)
        comp[r] = c
        q = [r]
        while q:
            x = q.pop(0)
            for j in adj[x]:
                if comp[j] < 0:
                    comp[j] = c
                    q.append(j)
    return comp, roots


def _components(n, adj):
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for i in range(n):
        for j in adj[i]:
            a, b = find(i), find(j)
            if a != b:
                parent[max(a, b)] = min(a, b)
    return [find(i) for i in range(n)]


def resolve(strategy: int, rules: int, umis: Sequence[bytes], keys: Sequence[Key], key_of: Sequence[int],
            adj: Sequence[Sequence[int]]) -> List[Tuple[int, int]]:
    """(kind, local id) per input; mapped ids start at 0 here (the group's counter is added by the caller)."""
    n = len(umis)
    if n == 0:
        return []
    if strategy == IDENTITY:
        return [(SINGLE, key_of[i]) for i in range(n)]
    if strategy == EDIT and rules == MAPPED:           # components, numbered by their smallest string
        root = _components(len(keys), adj)
        num: Dict[int, int] = {}
        for i in range(len(keys)):
            num.setdefault(root[i], len(num))
        return [(SINGLE, num[root[key_of[i]]]) for i in range(n)]
    if strategy == EDIT:                               # parallel_assigner.rs:373-417
        if not keys:
            return [(SINGLE, i) for i in range(n)]
        root = _components(len(keys), adj)
        num, out, nxt = {}, [], 0
        for i in range(n):
            if key_of[i] < 0:
                out.append((SINGLE, nxt))
                nxt += 1
            else:
                r = root[key_of[i]]
                if r not in num:
                    num[r] = nxt
                    nxt += 1
                out.append((SINGLE, num[r]))
        return out
    if strategy == ADJACENCY and rules == MAPPED:      # assigner.rs:1470-1524
        if not keys:
            return [(NONE, 0)] * n
        if len(keys) == 1:
            return [(SINGLE, 0)] * n
        comp, _ = _bfs_roots(keys, adj)
        return [(NONE, 0) if key_of[i] < 0 else (SINGLE, comp[key_of[i]]) for i in range(n)]
    if strategy == ADJACENCY:                          # parallel_assigner.rs:475-561
        if not keys:
            return [(SINGLE, i) for i in range(n)]
        comp, roots = _bfs_roots(keys, adj)
        nxt, out = len(roots), []
        for i in range(n):
            if key_of[i] < 0:
                out.append((SINGLE, nxt))
                nxt += 1
            else:
                out.append((SINGLE, comp[key_of[i]]))
        return out
    if rules == MAPPED:                                # PAIRED, assigner.rs:1801-1860
        if len(keys) == 1:
            return [(A if u < reverse_paired(u) else B, 0) for u in umis]
        comp, roots = _bfs_roots(keys, adj)
        strand: Dict[bytes, Tuple[int, int]] = {}
        root_set = set(roots)
        for c, r in enumerate(roots):
            rs = keys[r].s
            strand[rs] = (A, c)                        # insert order matters for palindromic X-X keys
            strand[reverse_paired(rs)] = (B, c)
        for i, key in enumerate(keys):
            if i in root_set:
                continue
            c = comp[i]
            rs, cs = keys[roots[c]].s, key.s
            crev = reverse_paired(cs)
            if count_mismatches(rs, cs) < count_mismatches(rs, crev):
                strand[cs] = (A, c)
                strand[crev] = (B, c)
            else:
                strand[cs] = (B, c)
                strand[crev] = (A, c)
        return [strand.get(u, (NONE, 0)) for u in umis]
    # PAIRED unmapped, parallel_assigner.rs:651-737
    if not keys:
        return [(SINGLE, i) for i in range(n)]
    comp, _ = _bfs_roots(keys, adj)
    out = []
    for i, u in enumerate(umis):
        if key_of[i] < 0:
            out.append((NONE, 0))
        else:
            up = upper(u)
            out.append((A if up == keys[key_of[i]].s else B, comp[key_of[i]]))
    return out


def n_ids(strategy: int, rules: int, res: Sequence[Tuple[int, int]], keys) -> int:
    """IDs a MAPPED call takes from its assigner's counter (next_id calls)."""
    if not res:
        return 0
    return max((i for kd, i in res if kd != NONE), default=-1) + 1


def assign_call(strategy, rules, k, umis, min_umi_length=None, enum=False):
    umis = truncate_umis(umis, min_umi_length)
    keys, key_of = prepare(strategy, rules, umis)
    adj = (edges_enum if enum else edges)(strategy, rules, k, keys) if needs_edges(strategy, keys) else [[]] * len(keys)
    return resolve(strategy, rules, umis, keys, key_of, adj)


def assign_groups(strategy, rules, k, groups, min_umi_length=None, enum=False):
    """groups: list of groups, a group a list of calls, a call a list of UMI strings (after umi_for_read).
    Returns (kinds, ids, group_mi_count), ids local to each group.  Mapped assigners keep one counter across
    a group's calls, unmapped ones restart at 0 (group.rs:1073-1093, 382-407); MI count = max(id) + 1
    (:1126-1131)."""
    kinds, ids, counts = [], [], []
    for g in groups:
        base, mx = 0, -1
        for call in g:
            res = assign_call(strategy, rules, k, call, min_umi_length, enum)
            if rules == MAPPED:
                res = [(kd, i + base) for kd, i in res]
                # identity / edit / adjacency / paired take one id per root / component / unique key
                base = max([base] + [i + 1 for kd, i in res if kd != NONE])
            for kd, i in res:
                kinds.append(kd)
                ids.append(i if kd != NONE else 0)
                if kd != NONE:
                    mx = max(mx, i)
        counts.append(mx + 1)
    return kinds, ids, counts


def mi_string(kind: int, local_id: int, base: int) -> str:   # lib.rs:79-98
    if kind == NONE:
        return ""
    s = str(local_id + base)
    return s + ("/A" if kind == A else "/B" if kind == B else "")
