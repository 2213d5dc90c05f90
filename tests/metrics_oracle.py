"""Oracle of `fgumi duplex-metrics` / `simplex-metrics` (fgumi 0.2.0): a restatement in Python of
src/lib/commands/shared_metrics.rs (templates, keys, intervals, Murmur3 downsampling), duplex_metrics.rs and
simplex_metrics.rs (the per-group collectors) and crates/fgumi-metrics/src/{duplex,simplex,shared}.rs (the tables).

collect(header_text, records, duplex=..., intervals=...) -> {table name: TSV text}; a failing input raises
MetricsOracleError with the index of the record the error names.

Known deviations, as the collector has them: ds_fraction_duplexes_ideal uses scipy's binomial CDF where the
reference uses statrs 0.18's regularised beta (compared within 1e-12 relative), and duplex UMIs with equal unique
counts are ordered by UMI (the reference's order of ties is its HashMap's).
"""
from __future__ import annotations

import os
import struct
import sys
from collections import OrderedDict
from typing import Dict, List, Optional, Sequence

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import group_oracle as G   # noqa: E402
from oracle import record_oracle as R  # noqa: E402

FRACTIONS = [0.05, 0.10, 0.15, 0.20, 0.25, 0.30, 0.35, 0.40, 0.45, 0.50, 0.55, 0.60, 0.65, 0.70, 0.75, 0.80,
             0.85, 0.90, 0.95, 1.00]   # shared_metrics.rs:23-26


class MetricsOracleError(ValueError):
    def __init__(self, msg: str, record: int):
        super().__init__(msg)
        self.record = record


# ---- Murmur3 (shared_metrics.rs:129-184) ------------------------------------------------------------------------
def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & 0xFFFFFFFF


def _mix_k1(k1):
    k1 = (k1 * 0xCC9E2D51) & 0xFFFFFFFF
    return (_rotl(k1, 15) * 0x1B873593) & 0xFFFFFFFF


def murmur3_chars(units: Sequence[int], seed: int = 42) -> int:   # htsjdk Murmur3.hashUnencodedChars
    h1 = seed & 0xFFFFFFFF
    n = len(units)
    i = 1
    while i < n:
        h1 ^= _mix_k1(units[i - 1] | (units[i] << 16))
        h1 = (_rotl(h1, 13) * 5 + 0xE6546B64) & 0xFFFFFFFF
        i += 2
    if n & 1:
        h1 ^= _mix_k1(units[n - 1])
    h1 ^= (2 * n) & 0xFFFFFFFF
    h1 ^= h1 >> 16
    h1 = (h1 * 0x85EBCA6B) & 0xFFFFFFFF
    h1 ^= h1 >> 13
    h1 = (h1 * 0xC2B2AE35) & 0xFFFFFFFF
    h1 ^= h1 >> 16
    return h1 - (1 << 32) if h1 >= 1 << 31 else h1


def name_hash(name: bytes) -> int:
    s = name.decode("utf-8", errors="replace")    # String::from_utf8_lossy
    b = s.encode("utf-16-le", errors="surrogatepass")
    return murmur3_chars(struct.unpack("<%dH" % (len(b) // 2), b))


def hash_fraction_of(h: int) -> float:
    a = h if h == -2 ** 31 else abs(h)           # wrapping_abs
    return float(a) / float(2 ** 31 - 1)


def hash_fraction(name: bytes) -> float:
    return hash_fraction_of(name_hash(name))


def bucket_of(hf: float) -> int:
    for i, f in enumerate(FRACTIONS):
        if hf <= f:
            return i
    return len(FRACTIONS)


# ---- intervals (shared_metrics.rs:197-289) ----------------------------------------------------------------------
def parse_intervals(text: bytes):
    out, picard = [], False
    for line in text.decode().split("\n"):
        line = line.strip()
        if not line or line.startswith("#"):
            continue
        if line.startswith("@"):
            picard = True
            continue
        f = line.split("\t", 3)
        if len(f) < 3:
            raise ValueError("Invalid line (needs at least 3 fields): " + line)
        s, e = _i32(f[1]), _i32(f[2])
        out.append((f[0], s - 1 if picard else s, e))
    return out


def _i32(s: str) -> int:
    t = s[1:] if s[:1] in "+-" else s
    if not t or not all("0" <= c <= "9" for c in t):
        raise ValueError("Invalid position: " + s)
    v = int(s)
    if not -2 ** 31 <= v < 2 ** 31:
        raise ValueError("Invalid position: " + s)
    return v


def overlaps(ivs, ref_name: Optional[str], start: int, end: int) -> bool:
    if not ivs:
        return True
    if ref_name is None:
        return False
    return any(n == ref_name and start <= e and s < end for n, s, e in ivs)


# ---- templates (shared_metrics.rs:457-605) ----------------------------------------------------------------------
def _passes(f: int, first: bool) -> bool:
    seg = G.FIRST if first else 0x80
    return bool(f & G.PAIRED) and not f & G.UNMAPPED and not f & 0x8 and bool(f & seg) and \
        not f & G.SECONDARY and not f & G.SUPPLEMENTARY


def _ref_len(r: bytes) -> int:
    return sum(op >> 4 for op in G.cigar(r) if (op & 0xF) in (0, 2, 3, 7, 8))


def _utf8(b: bytes) -> Optional[str]:
    try:
        return b.decode("utf-8")
    except UnicodeDecodeError:
        return None


def templates(header_text: bytes, records: Sequence[bytes], ivs, first_index: int = 0, overlap=None):
    """(key, mi, rx, hash fraction, first record index) per kept template, in stream order: a generator, so that an
    error is raised where the reference's stream meets it.  overlap(ref_name, start, end), when given, replaces
    overlaps(ivs, ...) (tests/metrics_shapes.py's index for long interval lists)."""
    sq = [ln.split(b"\tSN:")[1].split(b"\t")[0].decode(errors="replace")
          for ln in header_text.split(b"\n") if ln.startswith(b"@SQ\t") and b"\tSN:" in ln]
    i = 0
    while i < len(records):
        nm = G.name(records[i])
        j = i + 1
        while j < len(records) and G.name(records[j]) == nm:
            j += 1
        recs, idx = _template_order(records, i, j, first_index)
        i0 = i
        i = j
        if len(recs) < 2:
            continue
        r1 = next((r for r in recs if _passes(G.flags(r), True)), None)
        r2 = next((r for r in recs if _passes(G.flags(r), False)), None)
        if r1 is None or r2 is None:
            continue
        name = nm.decode("utf-8", errors="replace")
        for tag in (b"MI", b"RX"):
            v = G.find_string_tag(r1, tag)
            if v is None:
                raise MetricsOracleError(f"Read '{name}' is missing the required {tag.decode()} tag", first_index + i0)
            if _utf8(v) is None:
                raise MetricsOracleError(f"Read '{name}' {tag.decode()} tag is not UTF-8", first_index + i0)
        mi, rx = G.find_string_tag(r1, b"MI").decode(), G.find_string_tag(r1, b"RX").decode()
        t1, t2 = G.ref_id(r1), G.ref_id(r2)
        if t1 < 0 or t2 < 0 or not G.cigar(r1) or not G.cigar(r2):
            continue
        s1, s2 = G.unclipped_5prime(r1), G.unclipped_5prime(r2)
        p1, p2 = struct.unpack_from("<i", r1, 4)[0] + 1, struct.unpack_from("<i", r2, 4)[0] + 1
        e1 = p1 - 1 + _ref_len(r1) if p1 - 1 >= 0 and _ref_len(r1) else None
        e2 = p2 - 1 + _ref_len(r2) if p2 - 1 >= 0 and _ref_len(r2) else None
        if t1 == t2:
            start = min(p1, p2)
            end = max(e1, e2) if e1 is not None and e2 is not None else max(p1, p2)
        else:
            start, end = p1, (e1 if e1 is not None else p1)
        rev1, rev2 = bool(G.flags(r1) & 0x10), bool(G.flags(r2) & 0x10)
        key = (t1, s1, rev1, t2, s2, rev2) if (t1, s1) <= (t2, s2) else (t2, s2, rev2, t1, s1, rev1)
        ref_name = sq[t1] if t1 < len(sq) else None
        if not (overlap(ref_name, start, end) if overlap is not None else overlaps(ivs, ref_name, start, end)):
            continue
        yield key, mi, rx, hash_fraction(nm), first_index + i0


def _template_order(records, i, j, first_index):
    r1 = r2 = None
    lists = {k: [] for k in ("r1_supp", "r2_supp", "r1_sec", "r2_sec")}
    for k in range(i, j):
        r = records[k]
        f = G.flags(r)
        is_r1 = not f & G.PAIRED or f & G.FIRST
        if f & G.SECONDARY:
            lists["r1_sec" if is_r1 else "r2_sec"].append(r)
        elif f & G.SUPPLEMENTARY:
            lists["r1_supp" if is_r1 else "r2_supp"].append(r)
        elif is_r1:
            if r1 is not None:
                raise MetricsOracleError("Multiple non-secondary, non-supplemental R1 records", first_index + k)
            r1 = r
        else:
            if r2 is not None:
                raise MetricsOracleError("Multiple non-secondary, non-supplemental R2 records", first_index + k)
            r2 = r
    recs = [r for r in (r1, r2) if r is not None]
    for k in ("r1_supp", "r2_supp", "r1_sec", "r2_sec"):
        recs += lists[k][::-1]
    return recs, None


def consensus_input(records: Sequence[bytes]) -> Optional[int]:   # validate_not_consensus_bam (:300-350)
    for i, r in enumerate(records):
        f = G.flags(r)
        if not f & G.PAIRED or not f & G.FIRST or f & G.SECONDARY or f & G.SUPPLEMENTARY:
            continue
        tags = {t for _, t, _, _ in G.aux_entries(r)}
        return i if (b"aD" in tags and b"bD" in tags) or b"cD" in tags else None
    return None


# ---- the collectors (duplex_metrics.rs:291-603, simplex_metrics.rs:221-296) -----------------------------------------
def _builder_vote(pre, post, bases, quals):
    from tests import oracle_lib as O
    return O.builder_call(pre, post, bases, quals)[:2]


def umi_consensus(umis: List[str]) -> str:   # SimpleUmiConsensusCaller::consensus (simple_umi.rs:170-193)
    if len(umis) <= 1:
        return umis[0] if umis else ""
    if any(len(u) != len(umis[0]) for u in umis):
        return umis[0]
    try:
        return R.consensus_umis(list(umis), _builder_vote)
    except AssertionError:
        raise ValueError("mixed DNA and non-DNA characters")


class Collector:
    def __init__(self, duplex: bool, duplex_umi_counts: bool):
        self.duplex = duplex
        self.cs: Dict[int, int] = {}
        self.ss: Dict[int, int] = {}
        self.ds: Dict[int, int] = {}
        self.pairs: Dict[tuple, int] = {}
        self.umi: Dict[str, list] = {}
        self.dumi: Dict[str, list] = {}
        self.collect_duplex = duplex_umi_counts


def _inc(d, k):
    d[k] = d.get(k, 0) + 1


def _record(d, umi, raw, err):
    c = d.setdefault(umi, [0, 0, 0])
    c[0] += raw
    c[1] += err
    c[2] += 1


def _base(mi: str):
    if mi.endswith("/A"):
        return mi[:-2], 1
    if mi.endswith("/B"):
        return mi[:-2], 2
    return mi, 0


def process_group(group, collectors: List[Collector], counts: List[int], duplex: bool, duplex_umi_counts: bool):
    for idx, f in enumerate(FRACTIONS):
        ds_ = [t for t in group if t[3] <= f]
        if not ds_:
            continue
        counts[idx] += len(ds_)
        c = collectors[idx]
        _inc(c.cs, len(ds_))
        ss: "OrderedDict[str, int]" = OrderedDict()
        for t in ds_:
            ss[t[1]] = ss.get(t[1], 0) + 1
        for v in ss.values():
            _inc(c.ss, v)
        fams: "OrderedDict[str, list]" = OrderedDict()   # base -> [a, b, [(mi, rx, rec)]] in stream order
        for t in ds_:
            b, k = _base(t[1])
            e = fams.setdefault(b, [0, 0, []])
            if k == 1:
                e[0] += 1
            elif k == 2:
                e[1] += 1
            e[2].append((t[1], t[2], t[4]))
        last = idx == len(FRACTIONS) - 1
        for b, (a, bb, pairs) in fams.items():
            if duplex:
                _inc(c.ds, a + bb)
                _inc(c.pairs, (max(a, bb), min(a, bb)))
            if not last:
                continue
            try:
                if duplex:
                    _duplex_umis(c, pairs, duplex_umi_counts)
                else:
                    _simplex_umis(c, pairs)
            except ValueError:
                raise MetricsOracleError("UMI consensus fails", pairs[0][2])


def _duplex_umis(c: Collector, pairs, duplex_umi_counts):   # duplex_metrics.rs:515-602
    u1, u2 = [], []
    for mi, rx, _ in pairs:
        p = rx.split("-")
        if len(p) != 2 or not p[0] or not p[1]:
            continue
        if mi.endswith("/A"):
            u1.append(p[0]); u2.append(p[1])
        elif mi.endswith("/B"):
            u1.append(p[1]); u2.append(p[0])
    cons = []
    for us in (u1, u2):
        if us:
            k = umi_consensus(us)
            _record(c.umi, k, len(us), sum(u != k for u in us))
            cons.append(k)
    if duplex_umi_counts and len(cons) == 2:
        d1, d2 = f"{cons[0]}-{cons[1]}", f"{cons[1]}-{cons[0]}"
        err = sum(1 for _, rx, _ in pairs if rx != d1 and rx != d2)
        _record(c.dumi, d1, len(u1), err)


def _simplex_umis(c: Collector, pairs):   # simplex_metrics.rs:262-293
    split = [rx.split("-") for _, rx, _ in pairs]
    for pos in range(len(split[0]) if split else 0):
        us = [p[pos] for p in split if pos < len(p) and p[pos]]
        if not us:
            continue
        k = umi_consensus(us)
        _record(c.umi, k, len(us), sum(u != k for u in us))


# ---- the text (csv 1.1 over serde; floats as ryu 1.0 writes them) ---------------------------------------------------
def fmt_float(v: float) -> str:
    """ryu's format64 layout over the shortest round-trip digits d and exponent k (v = d * 10^k; Python's repr has the
    same digits): kk = len(d) + k; k >= 0 and kk <= 16: "d000.0"; 0 < kk <= 16: a point inside d; -5 < kk <= 0:
    "0.000d"; else d[0] [. rest] "e" kk - 1."""
    from decimal import Decimal
    if v == 0:
        return "0.0"
    sign = "-" if v < 0 else ""
    t = Decimal(repr(abs(v))).as_tuple()
    digits, k = "".join(map(str, t.digits)), t.exponent
    stripped = digits.rstrip("0")
    k += len(digits) - len(stripped)
    digits = stripped.lstrip("0")
    n = len(digits)
    kk = n + k
    if 0 <= k and kk <= 16:
        s = digits + "0" * k + ".0"
    elif 0 < kk <= 16:
        s = digits[:kk] + "." + digits[kk:]
    elif -5 < kk <= 0:
        s = "0." + "0" * (-kk) + digits
    elif n == 1:
        s = digits + "e" + str(kk - 1)
    else:
        s = digits[0] + "." + digits[1:] + "e" + str(kk - 1)
    return sign + s


def _frac(a, b):
    return a / b if b > 0 else 0.0


def _table(header, rows) -> str:
    if not rows:
        return ""
    out = ["\t".join(header)]
    for r in rows:
        out.append("\t".join(fmt_float(x) if isinstance(x, float) else str(x) for x in r))
    return "\n".join(out) + "\n"


def family_size_rows(c: Collector, duplex: bool):   # duplex.rs:323-369, simplex.rs:157-210
    kinds = [c.cs, c.ss] + ([c.ds] if duplex else [])
    mx = max([max(d) if d else 0 for d in kinds])
    tot = [sum(d.values()) for d in kinds]
    rows = []
    for z in range(1, mx + 1):
        rows.append([z] + [x for k, d in enumerate(kinds) for x in (d.get(z, 0), _frac(d.get(z, 0), tot[k]), 0.0)])
    for i in range(len(rows) - 1, -1, -1):
        for k in range(len(kinds)):
            nxt = rows[i + 1][1 + 3 * k + 2] if i + 1 < len(rows) else 0.0
            rows[i][1 + 3 * k + 2] = rows[i][1 + 3 * k + 1] + nxt
    return rows


def duplex_pair_rows(c: Collector):   # duplex.rs:373-420
    total = sum(c.pairs.values())
    rows = []
    for (a, b) in sorted(c.pairs):
        ge = sum(v for (x, y), v in c.pairs.items() if x >= a and y >= b)
        rows.append([a, b, c.pairs[(a, b)], _frac(c.pairs[(a, b)], total), _frac(ge, total)])
    return rows


def ideal_fraction(sizes: List[int], min_ab: int, min_ba: int) -> float:   # duplex_metrics.rs:456-503
    from scipy.stats import binom
    if not sizes:
        return 0.0
    acc = 0.0
    for n in sizes:
        if n < min_ab + min_ba:
            continue
        upper, lower = n - min_ba, min_ab
        p = float(binom.cdf(upper, n, 0.5)) - (float(binom.cdf(lower - 1, n, 0.5)) if lower > 0 else 0.0) \
            if upper >= lower else 0.0
        acc += p
    return acc / len(sizes)


def umi_rows(d: Dict[str, list]):   # shared.rs:117-135
    raw = sum(v[0] for v in d.values())
    uniq = sum(v[2] for v in d.values())
    return [[u, v[0], v[1], v[2], _frac(v[0], raw), _frac(v[2], uniq)] for u, v in sorted(d.items())]


def collect(header_text: bytes, records: Sequence[bytes], duplex: bool = True, intervals: Optional[bytes] = None,
            min_ab_reads: int = 1, min_ba_reads: int = 1, min_reads: int = 1,
            duplex_umi_counts: bool = False, overlap=None) -> Dict[str, str]:
    if duplex and min_ab_reads < min_ba_reads:
        raise ValueError("--min-ab-reads must be >= --min-ba-reads")
    ci = consensus_input(records)
    if ci is not None:
        raise MetricsOracleError("consensus input", ci)
    ivs = parse_intervals(intervals) if intervals is not None else []
    cols = [Collector(duplex, duplex_umi_counts and f == 1.0) for f in FRACTIONS]
    counts = [0] * len(FRACTIONS)
    group, key = [], None
    for t in templates(header_text, records, ivs, overlap=overlap):
        if key != t[0] and group:
            process_group(group, cols, counts, duplex, duplex_umi_counts)
            group = []
        group.append(t)
        key = t[0]
    if group:
        process_group(group, cols, counts, duplex, duplex_umi_counts)
    return tables(cols, counts, duplex, min_ab_reads, min_ba_reads, min_reads, duplex_umi_counts)


def tables(cols: List[Collector], counts: List[int], duplex: bool, min_ab_reads: int = 1, min_ba_reads: int = 1,
           min_reads: int = 1, duplex_umi_counts: bool = False) -> Dict[str, str]:
    """The tables of the per-fraction collectors and template counts."""
    main = cols[-1]
    out = {}
    fs_head = ["family_size", "cs_count", "cs_fraction", "cs_fraction_gt_or_eq_size", "ss_count", "ss_fraction",
               "ss_fraction_gt_or_eq_size"] + (["ds_count", "ds_fraction", "ds_fraction_gt_or_eq_size"] if duplex else [])
    out["family_sizes"] = _table(fs_head, family_size_rows(main, duplex))
    if duplex:
        out["duplex_family_sizes"] = _table(["ab_size", "ba_size", "count", "fraction", "fraction_gt_or_eq_size"],
                                            duplex_pair_rows(main))
    yrows = []
    for f, c, n in zip(FRACTIONS, cols, counts):
        rows = family_size_rows(c, duplex)
        cs = sum(r[1] for r in rows)
        if duplex:
            ds = sum(r[7] for r in rows)
            dup = sum(v for (a, b), v in c.pairs.items() if a >= min_ab_reads and b >= min_ba_reads)
            sizes = [r[0] for r in rows for _ in range(r[7])]
            ss = sum(((a > 0) + (b > 0)) * v for (a, b), v in c.pairs.items())
            yrows.append([f, n, cs, ss, ds, dup, _frac(dup, ds), ideal_fraction(sizes, min_ab_reads, min_ba_reads)])
        else:
            ss = sum(r[4] for r in rows)
            reads = sum(r[0] * r[4] for r in rows)
            single = next((r[4] for r in rows if r[0] == 1), 0)
            cons = sum(r[4] for r in rows if r[0] >= min_reads)
            yrows.append([f, n, cs, ss, _frac(reads, ss), single, _frac(single, ss), cons])
    out["yield_metrics"] = _table(
        ["fraction", "read_pairs", "cs_families", "ss_families", "ds_families", "ds_duplexes", "ds_fraction_duplexes",
         "ds_fraction_duplexes_ideal"] if duplex else
        ["fraction", "read_pairs", "cs_families", "ss_families", "mean_ss_family_size", "ss_singletons",
         "ss_singleton_fraction", "ss_consensus_families"], yrows)
    urows = umi_rows(main.umi)
    out["umi_counts"] = _table(["umi", "raw_observations", "raw_observations_with_errors", "unique_observations",
                                "fraction_raw_observations", "fraction_unique_observations"], urows)
    if duplex and duplex_umi_counts:
        single = {r[0]: r[5] for r in urows}
        raw = sum(v[0] for v in main.dumi.values())
        uniq = sum(v[2] for v in main.dumi.values())
        drows = []
        for u, v in sorted(main.dumi.items(), key=lambda kv: (-kv[1][2], kv[0])):
            a, _, b = u.partition("-")
            exp = single.get(a, 0.0) * single.get(b, 0.0) if "-" in u else 0.0
            drows.append([u, v[0], v[1], v[2], _frac(v[0], raw), _frac(v[2], uniq), exp])
        out["duplex_umi_counts"] = _table(["umi", "raw_observations", "raw_observations_with_errors",
                                           "unique_observations", "fraction_raw_observations",
                                           "fraction_unique_observations", "fraction_unique_observations_expected"],
                                          drows)
    return out
