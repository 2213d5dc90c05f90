"""Consensus units of long reads, up to the ABI's 65 535-base limit, and the tile forms they reach.

The vote kernels change form with the length of a unit's rows, not only with its depth: a unit whose rows span more
than one shared-memory stage is voted straight from HBM (a direct tile) whatever its class, a unit of more than 4 096
8-position items carries no uniform-items hint (the unit is found by binary search instead of `__umulhi`), and queue
entries `(u << 16) | p0` carry positions up to 65 535.  The helpers here build seeded units that sit on those edges,
with limits read from the library (`fgb_tile_capacity_bytes`, `fgb_tile_max_reads`) rather than written down:

  long_unit        one unit: a template, 1-3 % substitutions, a few N / lowercase / IUPAC bytes, qualities 2-60, and
                   a dense-dissent stretch (~30 % of the reads disagree at each position) of a few kb
  ladder           (depth, length) rungs: the longest staged and the shortest direct length per depth, cons_len on
                   both sides of the uniform-hint edge, 65 528..65 535, units whose only dissent lies above position
                   32 767 (after a clean prefix), one- and two-unit staged tiles at the cap, and ragged units whose
                   positions lie past some reads' ends
  forms            every tile of a packed batch as (class, direct, regular, uniform hint)
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

ACGT = np.frombuffer(b"ACGT", np.uint8)
IUPAC = np.frombuffer(b"RYKMSWBDHV", np.uint8)
LOWER = np.frombuffer(b"acgtn", np.uint8)
MAX_READ_LEN = 65535            # FGB_MAX_READ_LEN: a row descriptor holds 16 bits of length
UNIFORM_MAX_ITEMS = 4096        # planner.h: the largest uniform-items hint (`__umulhi` is exact up to here)
DISSENT_LEN = 3000              # dense-dissent stretch: enough undecided positions to overflow a warp's queue
HIGH_P0 = 33000                 # first noisy position of the high-dissent rungs: above 32 767, the upper half of p0
CLEAN_Q = 60                    # quality of their clean prefix: unanimous there, so the fast pass decides it
CLASS_NAMES = {0: "general", 1: "shallow", 2: "deep"}

SHALLOW_DEPTHS = (1, 2, 3, 4)
GENERAL_DEPTHS = (5, 8, 23)
DEEP_DEPTHS = (24, 25, 64)
UNIFORM_EDGE = (32767, 32768, 32769, 32776)   # 4 096, 4 096, 4 097, 4 097 items
EDGE_DEPTHS = (1, 2, 5, 24)


def _r8(n: int) -> int:
    return (n + 7) // 8 * 8


def _r16(n: int) -> int:
    return (n + 15) // 16 * 16


def long_unit(rng, depth: int, lens: Sequence[int], dissent: Optional[Tuple[int, int]] = None, clean: int = 0
              ) -> List[Tuple[bytes, bytes]]:
    """`depth` rows of the given lengths over one template.  `dissent` = [a, b): positions where each read carries
    another A/C/G/T base with probability 0.3 (clipped to each read's length).  `clean`: positions [0, clean) carry
    the template base in every read at quality CLEAN_Q, with no noise at all."""
    assert len(lens) == depth and min(lens) >= 1 and max(lens) <= MAX_READ_LEN
    P = max(lens)
    tmpl = ACGT[rng.integers(0, 4, size=P)]
    B = np.repeat(tmpl[None, :], depth, 0)
    Q = rng.integers(2, 61, size=(depth, P), dtype=np.uint8)
    sub = rng.random((depth, P)) < rng.uniform(0.01, 0.03)
    B[sub] = ACGT[rng.integers(0, 4, size=int(sub.sum()))]
    x = rng.random((depth, P))
    B[x < 0.003] = ord("N")
    m = (x >= 0.003) & (x < 0.005)
    B[m] = LOWER[rng.integers(0, len(LOWER), size=int(m.sum()))]
    m = (x >= 0.005) & (x < 0.006)
    B[m] = IUPAC[rng.integers(0, len(IUPAC), size=int(m.sum()))]
    if dissent is not None:
        a, b = max(0, dissent[0]), min(P, dissent[1])
        if b > a:
            d = rng.random((depth, b - a)) < 0.3
            shift = rng.integers(1, 4, size=(depth, b - a))
            idx = (np.searchsorted(ACGT, tmpl[a:b])[None, :] + shift) & 3
            seg = B[:, a:b]
            seg[d] = ACGT[idx[d]]
    if clean:
        B[:, :clean] = tmpl[None, :clean]
        Q[:, :clean] = CLEAN_Q
    return [(B[r, :lens[r]].tobytes(), Q[r, :lens[r]].tobytes()) for r in range(depth)]


def default_dissent(length: int) -> Tuple[int, int]:
    """A few kb of dense dissent a quarter of the way in (the middle third of rows shorter than 4 kb)."""
    if length < 4000:
        return length // 3, 2 * length // 3
    a = length // 4
    return a, a + DISSENT_LEN


def longest_staged(depth: int, cap: int, start: int) -> int:
    """The longest length L for which `depth` regular rows of L, the first at byte `start`, fit one stage."""
    s = start % 16
    lo, hi = 1, MAX_READ_LEN
    if _r16(s + (depth - 1) * _r8(1) + 1) > cap:
        return 0
    while lo < hi:                                  # span grows with L
        mid = (lo + hi + 1) // 2
        if _r16(s + (depth - 1) * _r8(mid) + mid) <= cap:
            lo = mid
        else:
            hi = mid - 1
    return lo


def ladder(cap: int, max_reads: int) -> List[Dict]:
    """The rungs, in packing order, as specs {name, depth, lens | "staged"/"direct", dissent, direct (expected)}.
    Lengths that depend on where a unit starts ("staged": the longest that fits a stage, "direct": one more) are
    resolved by `build`.  Every staged-at-the-cap tile follows a direct unit, so that it opens a tile of its own."""
    assert max_reads >= 64 + 1
    specs: List[Dict] = []
    for d in SHALLOW_DEPTHS + GENERAL_DEPTHS + DEEP_DEPTHS:
        specs.append(dict(name=f"staged d{d}", depth=d, lens="staged", direct=False))
        specs.append(dict(name=f"direct d{d}", depth=d, lens="direct", direct=True))
    for d in EDGE_DEPTHS:
        for n in UNIFORM_EDGE:
            specs.append(dict(name=f"uniform edge d{d} L{n}", depth=d, lens=[n] * d, direct=True))
    for d in EDGE_DEPTHS:
        for n in range(MAX_READ_LEN - 7, MAX_READ_LEN + 1):
            specs.append(dict(name=f"limit d{d} L{n}", depth=d, lens=[n] * d, direct=True))
    # the warp queue fills in item order and keeps its first kWarpQueueCap entries, so queued positions above 32 767
    # need a prefix with nothing to queue: a clean prefix, then dense dissent, in each kernel class
    for d in (3, 8, 30):
        specs.append(dict(name=f"high dissent d{d}", depth=d, lens=[40000] * d, clean=HIGH_P0,
                          dissent=(HIGH_P0, HIGH_P0 + DISSENT_LEN), direct=True))
    # two units per staged tile at the cap: regular rows back to back, 1 and 2 reads per unit
    for d in (1, 2):
        n = (cap - 16) // (2 * d) // 8 * 8
        specs.append(dict(name=f"two-unit tile d{d} (a)", depth=d, lens=[n] * d, direct=False, pair="a"))
        specs.append(dict(name=f"two-unit tile d{d} (b)", depth=d, lens=[n] * d, direct=False, pair="b"))
        specs.append(dict(name=f"closer d{d}", depth=1, lens=[cap + 1000], direct=True))
    # ragged units: positions past some reads' ends, on both sides of the stage and of the uniform edge
    specs += [
        dict(name="ragged staged d2", depth=2, lens=[12000, 7001], direct=False),
        dict(name="ragged direct d3", depth=3, lens=[30001, 22000, 9003], direct=True),
        dict(name="ragged direct d4", depth=4, lens=[65535, 40000, 33000, 1200], direct=True),
        dict(name="ragged direct d8", depth=8, lens=[41000, 4000, 39999, 12345, 8, 20000, 36001, 33333], direct=True),
        dict(name="ragged direct d30", depth=30, lens=[1000 + 1337 * i for i in range(30)], direct=True),
        dict(name="ragged staged d6", depth=6, lens=[3000, 2999, 1500, 3333, 17, 800], direct=False),
    ]
    return specs


def build(rng, specs: Sequence[Dict], cap: int) -> Tuple[List[List[Tuple[bytes, bytes]]], List[Dict]]:
    """Units for `specs`, packed the way `pack_source_reads` packs them (rows at 8-byte strides).  Returns (units,
    resolved specs) where every spec has its final `lens` and `start` (byte offset of its first row)."""
    units, out = [], []
    off = 0
    for s in specs:
        s = dict(s)
        d = s["depth"]
        if s["lens"] == "staged":
            n = longest_staged(d, cap, off)
            assert n > 0, s
            s["lens"] = [n] * d
        elif s["lens"] == "direct":
            n = longest_staged(d, cap, off) + 1     # the shortest length that does not fit a stage from `off`
            s["lens"] = [n] * d
        lens = s["lens"]
        s.setdefault("dissent", default_dissent(max(lens)))
        s["start"] = off
        units.append(long_unit(rng, d, lens, s["dissent"], s.get("clean", 0)))
        out.append(s)
        off += sum(_r8(n) for n in lens)
    return units, out


def ladder_batch(fg, seed: int = 1, min_reads: int = 1):
    """(PackedBatch, units, resolved specs) of the whole ladder."""
    lib = fg.lib.load()
    cap, max_reads = int(lib.fgb_tile_capacity_bytes()), int(lib.fgb_tile_max_reads())
    units, specs = build(np.random.default_rng(seed), ladder(cap, max_reads), cap)
    return fg.pack_source_reads(units, min_reads), units, specs


def forms(fg, batch) -> set:
    """Every tile of `batch` (fg.plan_tiles) as (class, direct, regular, uniform hint present)."""
    return {f for f, _ in tile_forms(fg, batch)}


def tile_forms(fg, batch) -> List[Tuple[Tuple[str, bool, bool, bool], np.void]]:
    out = []
    for t in fg.plan_tiles(batch):
        f = int(t["flags"])
        out.append(((CLASS_NAMES[(f >> 4) & 3], bool(f & 1), bool(f & 2), (f >> 8) != 0), t))
    return out


def unit_tiles(fg, batch) -> Dict[int, Tuple[Tuple[str, bool, bool, bool], np.void]]:
    """unit index -> (form, tile) of the tile that holds it."""
    out = {}
    for form, t in tile_forms(fg, batch):
        for u in range(int(t["unit_begin"]), int(t["unit_begin"]) + int(t["n_units"])):
            out[u] = (form, t)
    return out


# ---- record-level families of long reads ---------------------------------------------------------------------------
# (kind, depth, (shortest, longest read), insert of a pair): depths 1..255 on both strands, reads of 1 kb to the limit,
# pairs whose mates overlap by tens of kb (insert shorter than the two reads) and pairs that do not meet
LONG_FAMILIES = (
    ("frag", 1, (MAX_READ_LEN, MAX_READ_LEN), None),
    ("frag", 3, (30000, MAX_READ_LEN), None),
    ("pair", 2, (40000, 50000), 60000),
    ("pair", 4, (9001, 12000), 30000),
    ("pair", 3, (MAX_READ_LEN - 3, MAX_READ_LEN), MAX_READ_LEN),
    ("frag", 24, (1000, 4001), None),
    ("pair", 6, (20000, 30000), 32000),
    ("frag", 64, (1000, 3000), None),
    ("frag", 255, (1000, 1400), None),
)


def long_family(rng, g: int, kind: str, depth: int, lens: Tuple[int, int], insert: Optional[int], r1_rev: bool):
    """One MI group of `depth` fragments or pairs with read lengths in [lens] (mixed within the family), on the
    strand `r1_rev` picks.  Reads carry the record tests' noise (tests/test_callers_at_depth.py `_read`): ~1 %
    substitutions, N and IUPAC bytes, low-quality tails."""
    from tests.test_callers_at_depth import PAD, _pair, _read, _tags
    from tests.bam_builder import make_record
    span = insert if insert is not None else lens[1]
    tmpl = ACGT[rng.integers(0, 4, size=2 * PAD + span)].tobytes()
    rx = b"ACGTAC-GTTACA"
    recs = []
    for d in range(depth):
        l1, l2 = (int(x) for x in rng.integers(lens[0], lens[1] + 1, size=2))
        tags = _tags(rng, b"%d" % g, rx)
        name = b"L%d_%d" % (g, d)
        if kind == "frag":
            ref = tmpl[PAD + span - l1:PAD + span] if r1_rev else tmpl[PAD:PAD + l1]
            s, q = _read(rng, ref, r1_rev)
            recs.append(make_record(name=name, flags=16 if r1_rev else 0, pos=1000 + (span - l1 if r1_rev else 0),
                                    seq=s, quals=q, cigar="%dM" % l1, tags=tags))
        else:
            recs += _pair(rng, name, tmpl, insert, min(l1, insert), min(l2, insert), r1_rev, False, tags)
    return recs


def long_families(seed: int, specs=LONG_FAMILIES) -> List[List[bytes]]:
    rng = np.random.default_rng(seed)
    return [long_family(rng, g, kind, depth, lens, insert, g % 2 == 1)
            for g, (kind, depth, lens, insert) in enumerate(specs)]


def flatten(groups: Sequence[Sequence[bytes]]):
    """(blob, record offsets, group offsets) as fgb_caller_add_groups takes them."""
    recs = [r for g in groups for r in g]
    blob = np.frombuffer(b"".join(recs), np.uint8)
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in recs])
    grp = np.zeros(len(groups) + 1, np.uint64)
    grp[1:] = np.cumsum([len(g) for g in groups])
    return blob, off, grp
