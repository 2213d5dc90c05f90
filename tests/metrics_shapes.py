"""Test helper: metrics collector inputs at the shapes users collect (fgb_metrics_*, DESIGN.md section 13).

- NamePool: unique read names whose Murmur3 downsampling bucket is chosen, so that a template joins fractions f..19
  only (murmur3_ascii / buckets_of hash fixed-length ASCII names in bulk).
- StreamBuilder: coordinate groups of given families (fam), templates interleaved across the families of a group.
- LAYOUTS / layout_template: one template in every record layout the collector must read (R2 first, secondary and
  supplementary records, clips and every CIGAR op, strands, contigs, unmapped reads, long and non-ASCII names, MI / RX
  anywhere in the aux block, records near 64 KiB); twin() is a plain template with the same ReadInfoKey.
- CountReference: a numpy restatement of the family-size, duplex-pair and yield counts (CS, SS, DS, pairs, templates
  per fraction) for streams where tests/metrics_oracle.py is too slow; its tables go through the oracle's table
  writer, and it derives the overflow count of the shared histograms (K_SMALL, K_PAIR).
- IntervalIndex: metrics_oracle.overlaps for interval lists of exome size (sorted starts, running maximum ends).
"""
from __future__ import annotations

import ctypes as C
import zlib
from typing import Dict, List, Optional, Sequence

import numpy as np

from tests import metrics_oracle as O
from tests import metrics_streams as S
from tests.bam_builder import cigar_from_string, make_record

HEADER = S.HEADER
# chr2 has no intervals in exome_intervals: a header contig between two that have them
HEADER3 = HEADER + b"@SQ\tSN:chr3\tLN:198295559\n"
K_SMALL, K_PAIR = 32, 8     # kSmall / kPair of fgumi_b200/csrc/host/metrics_device.h: the shared-histogram bounds
N_FRACTIONS = len(O.FRACTIONS)
PAIRED, FIRST, LAST, REV, MREV = S.PAIRED, S.FIRST, S.LAST, S.REV, S.MREV
UNMAPPED, MATE_UNMAPPED, SECONDARY, SUPP = 0x4, 0x8, S.SECONDARY, S.SUPP

_FR = np.array(O.FRACTIONS, np.float64)
_U32 = np.uint32


# ---- names by bucket ----------------------------------------------------------------------------------------------
def murmur3_ascii(names: np.ndarray) -> np.ndarray:
    """O.name_hash of fixed-length ASCII names, one per row of a uint8 matrix: int32 per row."""
    u = names.astype(np.uint32)
    n = u.shape[1]
    h = np.full(len(u), 42, np.uint32)

    def mix(k):
        k = k * _U32(0xCC9E2D51)
        k = (k << _U32(15)) | (k >> _U32(17))
        return k * _U32(0x1B873593)

    for i in range(1, n, 2):
        h ^= mix(u[:, i - 1] | (u[:, i] << _U32(16)))
        h = (h << _U32(13)) | (h >> _U32(19))
        h = h * _U32(5) + _U32(0xE6546B64)
    if n & 1:
        h ^= mix(u[:, n - 1])
    h ^= _U32(2 * n)
    h ^= h >> _U32(16)
    h *= _U32(0x85EBCA6B)
    h ^= h >> _U32(13)
    h *= _U32(0xC2B2AE35)
    h ^= h >> _U32(16)
    return h.view(np.int32)


def buckets_of(hashes: np.ndarray) -> np.ndarray:
    """O.bucket_of(O.hash_fraction_of(h)) per hash: the first fraction the hash fraction does not exceed."""
    h = hashes.astype(np.int64)
    a = np.where(h == -2 ** 31, h, np.abs(h))    # wrapping_abs keeps i32::MIN
    return np.searchsorted(_FR, a / float(2 ** 31 - 1), side="left")


class NamePool:
    """Unique fixed-length ASCII read names by bucket: take(b) hands out the next unused name of bucket b.  The
    candidates, prefix + a zero-padded counter, are hashed 64 Ki at a time; each bucket holds about 5 % of them."""

    def __init__(self, prefix: bytes = b"q", width: int = 11):
        self.prefix, self.width, self.next = prefix, width, 0
        self.free: List[List[bytes]] = [[] for _ in range(N_FRACTIONS)]
        self.pos = [0] * N_FRACTIONS

    def _fill(self, count: int = 1 << 16):
        k = np.arange(self.next, self.next + count, dtype=np.int64)
        self.next += count
        digits = (k[:, None] // 10 ** np.arange(self.width - 1, -1, -1, dtype=np.int64)) % 10 + ord("0")
        pre = np.frombuffer(self.prefix, np.uint8)[None, :].repeat(count, 0)
        names = np.concatenate([pre, digits.astype(np.uint8)], 1)
        b = buckets_of(murmur3_ascii(names))
        for bucket in range(N_FRACTIONS):
            self.free[bucket] += [r.tobytes() for r in names[b == bucket]]

    def take(self, bucket: int, n: Optional[int] = None):
        want = 1 if n is None else n
        while len(self.free[bucket]) - self.pos[bucket] < want:
            self._fill()
        p = self.pos[bucket]
        self.pos[bucket] = p + want
        out = self.free[bucket][p:p + want]
        return out[0] if n is None else out


# ---- families and coordinate groups -------------------------------------------------------------------------------
def umi_pair(base: bytes):
    """Two 6-base UMIs fixed by the MI base: RX is "X-Y" on /A and bare MIs, "Y-X" on /B."""
    x = zlib.crc32(base)
    u = bytes(b"ACGT"[(x >> (2 * i)) & 3] for i in range(12))
    return u[:6], u[6:]


def fam(base: bytes, n_a: int = 0, n_b: int = 0, n_0: int = 0, bucket=0):
    """A family: n_a templates of base/A, n_b of base/B and n_0 of the bare base.  bucket: one bucket for all, or a
    sequence with one per template (the /A templates, then /B, then bare)."""
    sufs = [b"/A"] * n_a + [b"/B"] * n_b + [b""] * n_0
    bks = [bucket] * len(sufs) if isinstance(bucket, int) else list(bucket)
    assert len(bks) == len(sufs)
    return [(base, s, b) for s, b in zip(sufs, bks)]


class StreamBuilder:
    """A grouped stream: group() appends one coordinate group (its own position) of families, their templates
    interleaved one per family in turn, in the style of metrics_streams.pair."""

    def __init__(self, prefix: bytes = b"q", start: int = 1000):
        self.pool = NamePool(prefix)
        self.records: List[bytes] = []
        self.pos = start
        self.n_groups = 0

    def group(self, families: Sequence[Sequence[tuple]], ref: Optional[int] = None, pos: Optional[int] = None):
        ref = self.n_groups % 2 if ref is None else ref
        if pos is None:
            pos, self.pos = self.pos, self.pos + 500
        self.n_groups += 1
        fams = [list(f) for f in families if f]
        for i in range(max((len(f) for f in fams), default=0)):
            for f in fams:
                if i < len(f):
                    base, suf, bucket = f[i]
                    x, y = umi_pair(base)
                    rx = y + b"-" + x if suf == b"/B" else x + b"-" + y
                    self.records += S.pair(self.pool.take(bucket), base + suf, rx, ref1=ref, pos1=pos, pos2=pos + 200)
        return self


def boundary_stream(buckets=range(N_FRACTIONS), prefix=b"b"):
    """Every shared-histogram boundary in every given bucket: SS sizes 1, 7, 8, 31, 32, 33 on /A, /B and bare; DS
    sizes 0, 31, 32, 33; pairs (7, 0), (7, 7), (8, 0), (8, 7), (8, 8), (31, 31), (32, 1); CS groups of 31, 32 and 33;
    and families whose size crosses 32 (or ab crosses 8) between two fractions."""
    sb = StreamBuilder(prefix)
    mi = [0]

    def base():
        mi[0] += 1
        return b"%d" % mi[0]

    for b in buckets:
        for n in (1, 7, 8, 31, 32, 33):
            for kw in ("n_a", "n_b", "n_0"):
                sb.group([fam(base(), bucket=b, **{kw: n})])
        for a, bb in ((16, 15), (16, 16), (17, 16), (7, 0), (7, 7), (8, 0), (8, 7), (8, 8), (31, 31), (32, 1)):
            sb.group([fam(base(), a, bb, bucket=b)])
        sb.group([fam(base(), n_0=3, bucket=b)])                      # DS size 0
        for n in (31, 32, 33):                                           # CS groups of several families
            sb.group([fam(base(), n // 3, n // 3, bucket=b), fam(base(), n_0=n - 2 * (n // 3), bucket=b)])
        if b + 1 < N_FRACTIONS:                                        # sizes that cross the bounds at fraction b + 1
            sb.group([fam(base(), 32, bucket=[b] * 31 + [b + 1])])
            sb.group([fam(base(), 8, 7, bucket=[b] * 7 + [b + 1] + [b] * 7)])
            sb.group([fam(base(), 20, 13, bucket=[b + 1] + [b] * 32)])
    return sb.records


def worst_case_overflow(n_groups, prefix=b"w"):
    sb = StreamBuilder(prefix)
    for g in range(n_groups):
        sb.group([fam(b"%d" % (4 * g + k + 1), 8, bucket=0) for k in range(4)])
    return sb.records



# ---- template layouts ---------------------------------------------------------------------------------------------
_FILL = [(b"XS", "i", 5), (b"AS", "C", 7), (b"XZ", "Z", b"filler")]
_BARR = [(b"BC", "Bc", [-1, 2, 3]), (b"BS", "Bs", [1, -2, 3, 4, 5]), (b"BF", "Bf", [0.5]), (b"BI", "BI", [7] * 9)]


def _tags(mi, rx, place="end"):
    t = [(b"RX", "Z", rx), (b"MI", "Z", mi)]
    return {"start": t[::-1] + _FILL, "middle": _FILL[:2] + t[:1] + _FILL[2:] + t[1:], "end": _FILL + t,
            "after_b": _BARR + t}[place]


def _read(name, first, ref, pos, cigar="20M", rev=False, mref=0, mpos=1, tags=(), extra=0, l_seq=None):
    """One record at 1-based pos; SEQ as long as the CIGAR's query unless l_seq is given."""
    ops = cigar_from_string(cigar) if cigar else []
    q = sum(op >> 4 for op in ops if (op & 0xF) in (0, 1, 4, 7, 8))
    n = q if l_seq is None else l_seq
    flags = PAIRED | (FIRST if first else LAST) | (REV if rev else 0) | extra
    return make_record(name, flags, ref, pos - 1, cigar=ops, mate_ref_id=mref, mate_pos=mpos - 1,
                       seq=bytes(b"ACGT"[i % 4] for i in range(n)), tags=tags)


def _decoy(mi, rx):
    """Tags of the records other than R1: another family's MI and another RX, so that reading them instead of R1's
    changes the tables."""
    return [(b"MI", "Z", mi + b"9"), (b"RX", "Z", rx[::-1] + b"T")]


def layout_template(layout: str, name: bytes, mi: bytes, rx: bytes, pos: int = 100_000) -> List[bytes]:
    """The records of one template in `layout` (LAYOUTS); R1 carries MI and RX, every other record decoy tags."""
    p1, p2 = pos, pos + 150
    d = _decoy(mi, rx)
    tg = _tags(mi, rx)

    def r1(**kw):
        a = dict(ref=0, pos=p1, mref=0, mpos=p2, tags=tg)
        a.update(kw)
        return _read(name, True, **a)

    def r2(**kw):
        a = dict(ref=0, pos=p2, rev=True, mref=0, mpos=p1, tags=d)
        a.update(kw)
        return _read(name, False, **a)

    def extra(first, flag, k):
        return _read(name, first, 0, p1 + 7 * k, "10M", tags=d, extra=flag)

    if layout == "plain":
        return [r1(), r2()]
    if layout == "r2_first":
        return [r2(), r1()]
    if layout == "secondary_before":
        return [extra(True, SECONDARY, 1), r1(), r2()]
    if layout == "supplementary_after":
        return [r1(), r2(), extra(False, SUPP, 1)]
    if layout == "mixed_extras":
        return [extra(True, SUPP, 1), r2(), extra(False, SECONDARY, 2), r1(), extra(True, SECONDARY, 3)]
    if layout.startswith("run_"):   # a k-record QNAME run: extras split around R2-then-R1
        k = int(layout[4:])
        ex = [extra(i % 2 == 0, SECONDARY if i % 3 else SUPP, i + 1) for i in range(k - 2)]
        return ex[:len(ex) // 2] + [r2(), r1()] + ex[len(ex) // 2:]
    if layout == "lone":
        return [r1()]
    if layout == "clips":
        return [r1(cigar="2H3S15M"), r2(cigar="15M4S1H")]
    if layout == "ops":
        return [r1(cigar="1S5M2I3D4N5=3X5M"), r2(cigar="3H10M1D2I10M3X3S")]
    if layout == "ops_reverse_r1":
        return [r1(cigar="4S6M200N10M", rev=True), r2(cigar="2S18=", rev=False)]
    if layout == "r1_reverse":
        return [r1(rev=True), r2(rev=False)]
    if layout == "cross_contig_12":
        return [r1(ref=0, mref=1), r2(ref=1, mref=0)]
    if layout == "cross_contig_21":
        return [r1(ref=1, mref=0), r2(ref=0, mref=1)]
    if layout == "cross_contig_21_reverse":
        return [r2(ref=0, mref=1, rev=False), r1(ref=1, mref=0, rev=True, cigar="5S15M")]
    if layout == "unmapped_mate":
        return [r1(extra=MATE_UNMAPPED), r2(extra=UNMAPPED)]
    if layout == "unmapped_r1":
        return [r1(extra=UNMAPPED), r2(extra=MATE_UNMAPPED)]
    if layout == "tid_minus1":
        return [r1(), r2(ref=-1)]
    if layout == "no_cigar":
        return [r1(cigar=""), r2()]
    if layout.startswith("tags_"):   # MI / RX at the start, middle or end of the aux block, or after B arrays
        return [r1(tags=_tags(mi, rx, layout[5:]), cigar="21M"), r2(cigar="21M")]
    if layout.startswith("big_"):    # R1 of exactly the given size, its MI / RX after a large B array
        size = int(layout[4:])
        rec = r1(cigar="21001M", tags=[(b"PD", "Bc", [])] + tg)
        pad = size - len(rec)
        assert pad >= 0
        return [r1(cigar="21001M", tags=[(b"PD", "Bc", [1] * pad)] + tg), r2(cigar="9M")]
    raise ValueError(layout)


LAYOUTS = (["plain", "r2_first", "secondary_before", "supplementary_after", "mixed_extras"] +
           [f"run_{k}" for k in range(3, 9)] +
           ["lone", "clips", "ops", "ops_reverse_r1", "r1_reverse", "cross_contig_12", "cross_contig_21",
            "cross_contig_21_reverse", "unmapped_mate", "unmapped_r1", "tid_minus1", "no_cigar", "tags_start",
            "tags_middle", "tags_end", "tags_after_b", "big_65535", "big_65536", "big_65541"])
# names of 1 to 254 bytes, odd and even lengths, valid and invalid UTF-8 (the host's bucket path)
LAYOUT_NAMES = [b"a", b"bc", b"x" * 7, b"y" * 100, b"z" * 253, b"w" * 254, b"r\xc3\xa9ad", b"\xff\xfe", b"a\xe2\x82",
                "名前".encode(), b"\xf0\x9f\x98\x80x"]


def twin(name: bytes, mi: bytes, rx: bytes, key) -> List[bytes]:
    """A plain template (R1 then R2, 20M, no extras) whose ReadInfoKey is `key` (O.templates' 1-based form)."""
    t1, s1, rev1, t2, s2, rev2 = key
    a = _read(name, True, t1, s1 - 19 if rev1 else s1, rev=rev1, mref=t2, mpos=1, tags=_tags(mi, rx))
    b = _read(name, False, t2, s2 - 19 if rev2 else s2, rev=rev2, mref=t1, mpos=1, tags=_tags(mi, rx))
    return [a, b]


def layout_stream(pool: NamePool, layouts=LAYOUTS, names=LAYOUT_NAMES, buckets=range(N_FRACTIONS)):
    """Every layout and every name, each template followed by its twin (the same MI base on the other strand, the
    ReadInfoKey the oracle computes for it): a right key makes a CS group of 2, a wrong one splits it."""
    recs, k = [], 0
    cases = [(ly, None) for ly in layouts] + [("plain", nm) for nm in names] + [("r2_first", nm) for nm in names]
    for i, (ly, nm) in enumerate(cases):
        bucket = list(buckets)[i % len(list(buckets))]
        name = nm if nm is not None else pool.take(bucket)
        base = b"%d" % (7000 + i)
        x, y = umi_pair(base)
        t = layout_template(ly, name, base + b"/A", x + b"-" + y, pos=100_000 + 1000 * i)
        recs += t
        kept = list(O.templates(HEADER, t, []))
        if kept:
            recs += twin(pool.take(bucket), base + b"/B", y + b"-" + x, kept[0][0])
            k += 1
    return recs


# ---- the count-only reference -------------------------------------------------------------------------------------
class CountReference:
    """The family-size, duplex-pair and yield counts of kept templates in stream order, with numpy: group ids (a new
    id where the ReadInfoKey changes), MI bases, suffix kinds (0 bare, 1 /A, 2 /B) and buckets.  collectors() fills
    O.Collector objects (cs, ss, ds, pairs per fraction) and template counts for O.tables."""

    def __init__(self, group: np.ndarray, base: np.ndarray, kind: np.ndarray, bucket: np.ndarray):
        self.n = len(group)
        self.bucket = np.asarray(bucket, np.int64)
        _, self.gi = np.unique(np.asarray(group, np.int64), return_inverse=True)
        fam_key = self.gi.astype(np.int64) * (int(np.max(base, initial=0)) + 1) + np.asarray(base, np.int64)
        _, self.fi = np.unique(fam_key, return_inverse=True)
        self.kind = np.asarray(kind, np.int64)
        self.si = self.fi * 3 + self.kind
        self.n_groups = int(self.gi.max()) + 1 if self.n else 0
        self.n_families = int(self.fi.max()) + 1 if self.n else 0

    @classmethod
    def from_templates(cls, tpls):
        """From O.templates() tuples (key, mi, rx, hash fraction, first record)."""
        group, base, kind, bucket, ids, gid, last = [], [], [], [], {}, -1, None
        for key, mi, _, hf, _ in tpls:
            if key != last:
                gid += 1
                last = key
            b, k = O._base(mi)
            group.append(gid)
            base.append(ids.setdefault(b, len(ids)))
            kind.append(k)
            bucket.append(O.bucket_of(hf))
        return cls(np.array(group, np.int64), np.array(base, np.int64), np.array(kind, np.int64),
                   np.array(bucket, np.int64))

    @classmethod
    def from_host_templates(cls, header: bytes, bodies: np.ndarray, rec_off: np.ndarray, intervals=None):
        """From fgb_host_metrics_templates' kept templates (the template rules test_metrics_shapes.py pins against the
        oracle), MI text read from each R1: for streams of bench size, where O.templates is slow."""
        t = host_template_array(header, bodies, rec_off, intervals)
        t = t[t["status"] == 2]
        key = np.stack([t[f].astype(np.int64) for f in ("ref1", "start1", "strand1", "ref2", "start2", "strand2")], 1)
        group = np.concatenate([[0], np.cumsum(np.any(key[1:] != key[:-1], 1))]) if len(t) else np.zeros(0, np.int64)
        start = rec_off[t["r1"]].astype(np.int64) + t["mi_off"]
        raw = bodies.tobytes()
        ids, base, kind = {}, np.zeros(len(t), np.int64), np.zeros(len(t), np.int64)
        for i, (s, n) in enumerate(zip(start.tolist(), t["mi_len"].tolist())):
            b, k = O._base(raw[s:s + n].decode())
            base[i] = ids.setdefault(b, len(ids))
            kind[i] = k
        return cls(group, base, kind, t["bucket"].astype(np.int64))

    @staticmethod
    def _hist(sizes: np.ndarray) -> Dict[int, int]:
        v, c = np.unique(sizes[sizes > 0], return_counts=True)
        return dict(zip(v.tolist(), c.tolist()))

    def fraction(self, f: int):
        """(CS sizes, SS sizes, DS sizes of the families present, (ab, ba) arrays, templates) at fraction index f."""
        m = self.bucket <= f
        cs = np.bincount(self.gi[m], minlength=self.n_groups)
        ss = np.bincount(self.si[m], minlength=3 * self.n_families)
        present = np.bincount(self.fi[m], minlength=self.n_families) > 0
        a = ss[1::3][present]
        b = ss[2::3][present]
        return cs[cs > 0], ss[ss > 0], (a + b), np.maximum(a, b), np.minimum(a, b), int(m.sum())

    def collectors(self, duplex: bool = True):
        cols, counts = [], []
        for f in range(N_FRACTIONS):
            cs, ss, ds, ab, ba, n = self.fraction(f)
            c = O.Collector(duplex, False)
            c.cs, c.ss = self._hist(cs), self._hist(ss)
            if duplex:
                c.ds = {int(v): int(k) for v, k in zip(*np.unique(ds, return_counts=True))}   # size 0 too
                pv, pc = np.unique(ab.astype(np.int64) << 32 | ba, return_counts=True)
                c.pairs = {(int(v >> 32), int(v & 0xFFFFFFFF)): int(k) for v, k in zip(pv, pc)}
            cols.append(c)
            counts.append(n)
        return cols, counts

    def tables(self, duplex: bool = True, **opts) -> Dict[str, str]:
        """family_sizes, duplex_family_sizes (duplex) and yield_metrics as O.tables writes them."""
        cols, counts = self.collectors(duplex)
        out = O.tables(cols, counts, duplex, **opts)
        return {k: v for k, v in out.items() if k in ("family_sizes", "duplex_family_sizes", "yield_metrics")}

    def overflow(self) -> int:
        """Entries the family pass appends to its overflow list: per fraction, every CS, SS and DS size >= K_SMALL and
        every (ab, ba) with ab >= K_PAIR (a DS family counts its sizes and its pair in both modes)."""
        n = 0
        for f in range(N_FRACTIONS):
            cs, ss, ds, ab, _, _ = self.fraction(f)
            n += int((cs >= K_SMALL).sum() + (ss >= K_SMALL).sum() + (ds >= K_SMALL).sum() + (ab >= K_PAIR).sum())
        return n


def oracle_job(args):
    """O.collect(header, records, duplex=..., **opts) of one (header, records, duplex, opts) tuple: for worker
    processes."""
    header, records, duplex, opts = args
    return O.collect(header, records, duplex=duplex, **opts)


def expected_stats(header: bytes, records, intervals: Optional[bytes] = None, overlap=None) -> Dict[str, int]:
    """stats() counts that follow from the oracle's templates: kept, outside (kept but for the intervals), groups,
    ds_families (group, MI base) and overflow."""
    ivs = O.parse_intervals(intervals) if intervals is not None else []
    kept = list(O.templates(header, records, ivs, overlap=overlap))
    every = sum(1 for _ in O.templates(header, records, []))
    ref = CountReference.from_templates(kept)
    return {"kept": len(kept), "outside": every - len(kept) if (ivs or overlap) else 0, "groups": ref.n_groups,
            "ds_families": ref.n_families, "overflow": ref.overflow()}


def host_template_array(header: bytes, bodies: np.ndarray, rec_off: np.ndarray, intervals=None) -> np.ndarray:
    """fgb_host_metrics_templates as a numpy structured array (one row per QNAME run)."""
    from fgumi_b200 import lib as L
    lib = L.load()
    bodies = np.ascontiguousarray(bodies, np.uint8)
    rec_off = np.ascontiguousarray(rec_off, np.uint64)
    n = len(rec_off) - 1
    out = (L.FgbMetricsTemplate * max(n, 1))()
    nt, bad = C.c_uint64(), C.c_uint64()
    st = lib.fgb_host_metrics_templates(header, len(header), intervals, len(intervals) if intervals is not None else 0,
                                        bodies.ctypes.data, rec_off.ctypes.data, n, out, n, C.byref(nt), C.byref(bad))
    assert st == L.FGB_OK, st
    fields = [f for f, _ in L.FgbMetricsTemplate._fields_ if f != "reserved"]
    kinds = {C.c_int32: "<i4", C.c_uint32: "<u4", C.c_uint8: "u1", C.c_uint64: "<u8"}
    dt = np.dtype({"names": fields,
                   "formats": [kinds[dict(L.FgbMetricsTemplate._fields_)[f]] for f in fields],
                   "offsets": [getattr(L.FgbMetricsTemplate, f).offset for f in fields],
                   "itemsize": C.sizeof(L.FgbMetricsTemplate)})
    return np.frombuffer(out, dt, count=nt.value).copy()


# ---- intervals ----------------------------------------------------------------------------------------------------
class IntervalIndex:
    """O.overlaps(ivs, ...) for long interval lists: per contig name, the starts sorted and the running maximum of the
    ends.  [s, e) meets the template span iff s < end and start <= e: among the intervals with s < end (a prefix of
    the sorted starts), the largest end decides."""

    def __init__(self, ivs):
        self.any = bool(ivs)
        by: Dict[str, list] = {}
        for n, s, e in ivs:
            by.setdefault(n, []).append((s, e))
        self.idx = {}
        for n, v in by.items():
            a = np.array(sorted(v), np.int64)
            self.idx[n] = (a[:, 0].copy(), np.maximum.accumulate(a[:, 1]))

    def __call__(self, ref_name: Optional[str], start: int, end: int) -> bool:
        if not self.any:
            return True
        if ref_name is None or ref_name not in self.idx:
            return False
        s, mx = self.idx[ref_name]
        k = int(np.searchsorted(s, end, side="left"))
        return k > 0 and int(mx[k - 1]) >= start


def interval_text(ivs, picard: bool = False, header: bytes = HEADER3) -> bytes:
    """BED (0-based starts) or Picard interval-list text (the header, then 1-based starts) of (name, start, end)."""
    if picard:
        return header + b"".join(b"%s\t%d\t%d\t+\tiv%d\n" % (n.encode(), s + 1, e, i) for i, (n, s, e) in enumerate(ivs))
    return b"".join(b"%s\t%d\t%d\n" % (n.encode(), s, e) for n, s, e in ivs)


def exome_stream(seed: int, n_groups: int = 2000):
    """Templates on chr1..chr3 of HEADER3 with their insert spans (contig name, 1-based start, end): same-contig pairs
    in groups of 1 to 3, and R1-only inserts of pairs whose mate is on another contig."""
    rng = np.random.default_rng(seed)
    pool = NamePool(b"e")
    recs, spans = [], []
    pos = np.sort(rng.choice(np.arange(10_000, 100_000_000, 1000), n_groups, replace=False))
    for g in range(n_groups):
        ref, p = int(rng.integers(0, 3)), int(pos[g])
        cross = rng.random() < 0.15
        ref2 = (ref + 1 + int(rng.integers(0, 2))) % 3 if cross else ref
        p2 = p + int(rng.integers(0, 400))
        base = b"%d" % (g + 1)
        x, y = umi_pair(base)
        for k in range(int(rng.integers(1, 4))):
            suf = b"/A" if k % 2 == 0 else b"/B"
            rx = x + b"-" + y if suf == b"/A" else y + b"-" + x
            recs += S.pair(pool.take(int(rng.integers(0, N_FRACTIONS))), base + suf, rx, ref1=ref, pos1=p, ref2=ref2,
                           pos2=p2)
        name = "chr%d" % (ref + 1)
        spans.append((name, p, p + 19 if cross else max(p, p2) + 19))
    return recs, spans


def exome_intervals(seed: int, spans, n: int = 200_000):
    """About n intervals (name, 0-based start, end), unsorted, by a seeded rule: random exome-like intervals on chr1
    and chr3 (none on chr2), nested and overlapping runs, duplicates, contigs absent from the header, and per template
    span an interval that just meets or just misses it (end == start, end == start - 1, start == end - 1,
    start == end) or a long interval holding a nested one that ends before it."""
    rng = np.random.default_rng(seed)
    out = []
    for name, s, e in spans:
        if name == "chr2":
            continue
        r = int(rng.integers(0, 7))
        if r == 0:
            out.append((name, s - 50, s))            # end == start: meets
        elif r == 1:
            out.append((name, s - 50, s - 1))        # end == start - 1: misses
        elif r == 2:
            out.append((name, e - 1, e + 40))        # start == end - 1: meets
        elif r == 3:
            out.append((name, e, e + 40))            # start == end: misses
        elif r == 4:                                 # a long interval over the span, a nested one ending before it
            out += [(name, s - 5000, e + 5000), (name, s - 100, s - 60)]
        elif r == 5:                                 # the long interval ends one before the span: every one misses
            out += [(name, s - 5000, s - 1), (name, s - 100, s - 60), (name, s - 3, s - 2)]
    k = n - len(out)
    n_rand = k * 8 // 10
    starts = rng.integers(0, 100_000_000, n_rand)
    lens = rng.integers(1, 300, n_rand)
    names = np.where(rng.random(n_rand) < 0.5, "chr1", "chr3")
    out += [(str(a), int(b), int(b + c)) for a, b, c in zip(names, starts, lens)]
    for _ in range((k - n_rand) // 4):                # nested and overlapping runs
        b = int(rng.integers(0, 100_000_000))
        nm = "chr1" if rng.random() < 0.5 else "chr3"
        out += [(nm, b, b + 2000), (nm, b + 10, b + 50), (nm, b + 1500, b + 2600)]
    dup = rng.choice(len(out), (k - n_rand) // 8, replace=False)
    out += [out[int(i)] for i in dup]
    out += [("chrZ", int(b), int(b) + 100) for b in rng.integers(0, 100_000_000, n - len(out))]
    order = rng.permutation(len(out))
    return [out[int(i)] for i in order]


# ---- ideal fraction -----------------------------------------------------------------------------------------------
def binom_interval_half(lower: int, upper: int, n: int) -> float:
    """binom_interval_half of metrics_host.cpp restated: P(lower <= A <= upper) for A ~ Binomial(n, 0.5), the terms
    relative to the mode's by the ratio recurrence, the interval's over all of them."""
    m = n // 2
    total, inside, t = 1.0, (1.0 if lower <= m <= upper else 0.0), 1.0
    k = m
    while k < n and t > 0:
        t *= (n - k) / (k + 1)
        total += t
        inside += t if lower <= k + 1 <= upper else 0.0
        k += 1
    t, k = 1.0, m
    while k > 0 and t > 0:
        t *= k / (n - k + 1)
        total += t
        inside += t if lower <= k - 1 <= upper else 0.0
        k -= 1
    return inside / total


def ideal_fraction_ratio(sizes, min_ab: int, min_ba: int) -> float:
    """O.ideal_fraction with binom_interval_half in place of scipy's CDF."""
    acc = 0.0
    for n in sizes:
        if n >= min_ab + min_ba:
            acc += binom_interval_half(min_ab, n - min_ba, n) if n - min_ba >= min_ab else 0.0
    return acc / len(sizes) if sizes else 0.0
