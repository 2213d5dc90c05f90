"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Restatement (pure Python) of `fgumi group` around the UMI assignment, record bytes in, record bytes out, in the
single-threaded order of the reference.  Citations are relative to the fgumi 0.2.0 source tree:
  group.rs    src/lib/commands/group.rs              (filter, orientation split, UMIs, per-group processing)
  grouper.rs  src/lib/grouper.rs                     (RecordPositionGrouper, build_templates_from_records)
  bam.rs      src/lib/unified_pipeline/bam.rs        (compute_group_key_from_raw)
  base.rs     src/lib/unified_pipeline/base.rs       (GroupKey)
  read_info   src/lib/read_info.rs                   (LibraryIndex)
  template    src/lib/template.rs                    (Template::from_records)
  cigar.rs    crates/fgumi-raw-bam/src/cigar.rs      (unclipped 5' positions)
  tags.rs     crates/fgumi-raw-bam/src/tags.rs       (update_string_tag)
  lib.rs      crates/fgumi-umi/src/lib.rs            (validate_umi, MoleculeId)
The assignment itself is oracle/umi_oracle.py.  Library, cell and QNAME are compared as bytes where the reference
compares their hashes (the same answer barring a collision).
"""
from __future__ import annotations

import struct
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

from oracle import umi_oracle as U

PAIRED, UNMAPPED, MATE_UNMAPPED, REVERSE, MATE_REVERSE, FIRST = 0x1, 0x4, 0x8, 0x10, 0x20, 0x40
QC_FAIL, SECONDARY, SUPPLEMENTARY = 0x200, 0x100, 0x800
I32_MAX = 2 ** 31 - 1

STATS = ("total_records", "accepted_records", "discarded_non_pf", "discarded_poor_alignment", "discarded_ns_in_umi",
         "discarded_umi_too_short", "position_groups", "groups_dropped", "next_mi", "records_out")


class GroupError(ValueError):
    """Where the reference fails the command (or panics): the product fails the call."""

    def __init__(self, msg, record=None):
        super().__init__(msg)
        self.record = record


# ---- record fields --------------------------------------------------------------------------------------------
def flags(r: bytes) -> int:
    return struct.unpack_from("<H", r, 14)[0]


def ref_id(r: bytes) -> int:
    return struct.unpack_from("<i", r, 0)[0]


def name(r: bytes) -> bytes:
    return r[32:32 + r[8] - 1] if r[8] else b""


def cigar(r: bytes) -> List[int]:
    n = struct.unpack_from("<H", r, 12)[0]
    return list(struct.unpack_from("<%dI" % n, r, 32 + r[8]))


def aux_off(r: bytes) -> int:
    n_cig = struct.unpack_from("<H", r, 12)[0]
    l_seq = struct.unpack_from("<I", r, 16)[0]
    return 32 + r[8] + 4 * n_cig + (l_seq + 1) // 2 + l_seq


_FIXED = {ord(c): n for c, n in (("A", 1), ("c", 1), ("C", 1), ("s", 2), ("S", 2), ("i", 4), ("I", 4), ("f", 4))}


def tag_value_size(t: int, data: bytes) -> Optional[int]:   # fields.rs:289-310
    if t in _FIXED:
        return _FIXED[t]
    if t in (ord("Z"), ord("H")):
        z = data.find(b"\0")
        return None if z < 0 else z + 1
    if t == ord("B"):
        if len(data) < 5 or data[0] not in _FIXED or data[0] == ord("A"):
            return None
        return 5 + struct.unpack_from("<I", data, 1)[0] * _FIXED[data[0]]
    return None


def aux_entries(r: bytes):
    """(offset in r, tag, type, value size) of each aux entry, stopping where the walk cannot go on."""
    a = aux_off(r)
    p = a
    while p + 3 <= len(r):
        size = tag_value_size(r[p + 2], r[p + 3:])
        yield p, r[p:p + 2], r[p + 2], size
        if size is None:
            return
        p += 3 + size


def find_string_tag(r: bytes, tag: bytes) -> Optional[bytes]:
    """The first entry of `tag`, if it is a Z string."""
    for p, t, vt, size in aux_entries(r):
        if t == tag:
            return r[p + 3:p + 2 + size] if vt == ord("Z") and size is not None else None
    return None


def unclipped_5prime(r: bytes) -> int:   # cigar.rs:201-228 (1-based), 470-508
    f = flags(r)
    if f & UNMAPPED:
        return 0
    ops = cigar(r)
    if not ops:
        return I32_MAX
    pos = struct.unpack_from("<i", r, 4)[0] + 1
    if not f & REVERSE:
        clipped = 0
        for op in ops:
            if op & 0xF in (4, 5):
                clipped += op >> 4
            else:
                break
        return pos - clipped
    ref_len = trailing = 0
    saw = False
    for op in ops:
        if op & 0xF in (0, 2, 3, 7, 8):
            ref_len += op >> 4
            trailing = 0
            saw = True
        elif op & 0xF in (4, 5) and saw:
            trailing += op >> 4
    return pos + ref_len + trailing - 1


def _parse_int(s: bytes) -> int:   # str::parse::<i32>().unwrap_or(0)
    if not s or not s.isdigit() or int(s) > I32_MAX:
        return 0
    return int(s)


def mate_unclipped_5prime(mate_pos0: int, mate_reverse: bool, mc: bytes) -> int:   # cigar.rs:276-306, 514-573
    pos = mate_pos0 + 1
    start = 0
    if not mate_reverse:
        clipped = 0
        for i, c in enumerate(mc):
            if chr(c).isdigit():
                continue
            if c in b"SH":
                clipped += _parse_int(mc[start:i])
                start = i + 1
            else:
                break
        return pos - clipped
    ref_len = trailing = 0
    saw = False
    for i, c in enumerate(mc):
        if chr(c).isdigit():
            continue
        num = _parse_int(mc[start:i])
        start = i + 1
        if c in b"MDN=X":
            ref_len += num
            trailing = 0
            saw = True
        elif c in b"SH" and saw:
            trailing += num
    return pos + ref_len + trailing - 1


def _utf8(b: bytes) -> bool:
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


# ---- position grouping ----------------------------------------------------------------------------------------
def library_index(header_text: bytes) -> Dict[bytes, int]:
    """LibraryIndex::from_header (read_info.rs:104-131): RG ID -> library number; libraries numbered from 1 in order
    of first appearance, an RG without LB is library "unknown" = 0."""
    lib_of_name = {b"unknown": 0}
    out = {}
    for line in header_text.split(b"\n"):
        line = line.rstrip(b"\r")
        if not line.startswith(b"@RG\t"):
            continue
        rid, lb = None, b"unknown"
        for f in line.split(b"\t")[1:]:
            if f.startswith(b"ID:"):
                rid = f[3:]
            elif f.startswith(b"LB:"):
                lb = f[3:]
        if rid is None:
            continue
        if lb not in lib_of_name:
            lib_of_name[lb] = len(lib_of_name)
        out[rid] = lib_of_name[lb]
    return out


def position_key(r: bytes, libs: Dict[bytes, int], cell_tag: Optional[bytes]):
    """compute_group_key_from_raw (bam.rs:415-499) + GroupKey::position_key (base.rs:1375-1436); None for a
    secondary or supplementary record."""
    f = flags(r)
    if f & (SECONDARY | SUPPLEMENTARY):
        return None
    rg = find_string_tag(r, b"RG")
    lib = libs.get(rg, 0) if rg is not None else 0
    cell = find_string_tag(r, cell_tag) if cell_tag else None
    own = (ref_id(r), unclipped_5prime(r), 1 if f & REVERSE else 0)
    mc = find_string_tag(r, b"MC")
    if mc is not None and not _utf8(mc):
        mc = None
    if f & PAIRED and not f & MATE_UNMAPPED and mc is not None:
        mate = (struct.unpack_from("<i", r, 20)[0],
                mate_unclipped_5prime(struct.unpack_from("<i", r, 24)[0], bool(f & MATE_REVERSE), mc),
                1 if f & MATE_REVERSE else 0)
        lo, hi = (own, mate) if own <= mate else (mate, own)
    else:
        lo, hi = own, (I32_MAX, I32_MAX, 255)
    return lo + hi + (lib, cell)


def group_by_position(records: Sequence[bytes], header_text: bytes = b"", cell_tag: Optional[bytes] = b"CB"):
    """RecordPositionGrouper (grouper.rs:406-588): (keep, group_begin over the kept records)."""
    libs = library_index(header_text)
    keep, begin = [], []
    cur = last = None
    kept = 0
    for i, r in enumerate(records):
        k = position_key(r, libs, cell_tag)
        if k is None:
            keep.append(0)
            continue
        f = flags(r)
        mc = find_string_tag(r, b"MC")
        if f & PAIRED and not f & (UNMAPPED | MATE_UNMAPPED) and (mc is None or not _utf8(mc)):   # :452-475
            raise GroupError("RecordPositionGrouper requires MC tags on paired-end reads", record=i)
        keep.append(1)
        same = cur is not None and (k == cur or name(last) == name(r))
        if not same:
            begin.append(kept)
            cur = k
        last = r
        kept += 1
    begin.append(kept)
    return keep, begin


# ---- per position group -----------------------------------------------------------------------------------------
@dataclass
class Config:
    strategy: int = U.ADJACENCY
    edits: int = 1
    rules: int = U.MAPPED              # UNMAPPED = --allow-unmapped
    min_umi_length: Optional[int] = None
    min_map_q: int = 1
    include_non_pf: bool = False
    no_umi: bool = False
    umi_tag: bytes = b"RX"
    assign_tag: bytes = b"MI"
    first_mi: int = 0

    def check(self):   # group.rs:723-757
        if self.strategy == U.PAIRED and (self.min_umi_length or self.no_umi):
            raise GroupError("paired strategy with --min-umi-length or --no-umi")
        if self.strategy == U.IDENTITY and self.edits and not self.no_umi:
            raise GroupError("edits must be 0 with the identity strategy")

    @property
    def assign_strategy(self):
        return U.IDENTITY if self.no_umi else self.strategy

    @property
    def assign_edits(self):
        return 0 if self.no_umi else self.edits

    @property
    def assign_min_len(self):
        return None if self.no_umi else self.min_umi_length


def build_templates(records: Sequence[bytes]):
    """build_templates_from_records (grouper.rs:596-651) + Template::from_records (template.rs:159-273):
    [(name, r1, r2)], primary reads only."""
    out = []
    i = 0
    while i < len(records):
        nm = name(records[i])
        j = i + 1
        while j < len(records) and name(records[j]) == nm:
            j += 1
        r1 = r2 = None
        for r in records[i:j]:
            f = flags(r)
            if f & (SECONDARY | SUPPLEMENTARY):
                continue
            if not f & PAIRED or f & FIRST:
                if r1 is not None:
                    raise GroupError("Multiple non-secondary, non-supplemental R1 records")
                r1 = r
            else:
                if r2 is not None:
                    raise GroupError("Multiple non-secondary, non-supplemental R2 records")
                r2 = r
        out.append((nm, r1, r2))
        i = j
    return out


def validate_umi(u: bytes):   # lib.rs:323-333: None for an upper-case N, else the number of ACGT (either case)
    n = 0
    for c in u:
        if c == ord("N"):
            return None
        if c in b"ACGTacgt":
            n += 1
    return n


def filter_template(r1, r2, cfg: Config, m: List[int]) -> bool:
    """filter_template_raw (group.rs:113-262); m: [total, accepted, non_pf, poor_alignment, ns_in_umi, too_short],
    counted per primary read of the template."""
    reads = [r for r in (r1, r2) if r is not None]
    n = len(reads)
    m[0] += n
    if not reads:
        m[3] += n
        return False
    if all(flags(r) & UNMAPPED for r in reads) and cfg.rules != U.UNMAPPED:
        m[3] += n
        return False
    for r in reads:
        f = flags(r)
        if not cfg.include_non_pf and f & QC_FAIL:
            m[2] += n
            return False
        if not f & UNMAPPED and r[9] < cfg.min_map_q:
            m[3] += n
            return False
    for r in reads:
        check_mq = not flags(r) & MATE_UNMAPPED
        check_umi = not cfg.no_umi
        mq = umi = None
        a = aux_off(r)
        p = a
        while p + 3 <= len(r):   # :167-221, one walk
            t, vt = r[p:p + 2], r[p + 2]
            if check_umi and t == cfg.umi_tag and vt == ord("Z"):
                z = r.find(b"\0", p + 3)
                if z < 0:
                    break
                umi = r[p + 3:z]
                p = z + 1
                if not check_mq or mq is not None:
                    break
                continue
            if check_mq and t == b"MQ":
                fmt = {ord("C"): "<B", ord("c"): "<b", ord("S"): "<H", ord("s"): "<h", ord("I"): "<I",
                       ord("i"): "<i"}.get(vt)
                mq = struct.unpack_from(fmt, r, p + 3)[0] if fmt and p + 3 + struct.calcsize(fmt) <= len(r) else None
            size = tag_value_size(vt, r[p + 3:])
            if size is None:
                break
            p += 3 + size
            if (not check_umi or umi is not None) and (not check_mq or mq is not None):
                break
        if check_mq and mq is not None and (mq & 0xFF) < cfg.min_map_q:   # `mq as u8`
            m[3] += n
            return False
        if cfg.no_umi:
            continue
        if umi is None:
            m[3] += n
            return False
        bases = validate_umi(umi)
        if bases is None:
            m[4] += n
            return False
        if cfg.min_umi_length and bases < cfg.min_umi_length:
            m[5] += n
            return False
    m[1] += n
    return True


def is_r1_earlier(r1: bytes, r2: bytes) -> bool:   # group.rs:268-279
    if ref_id(r1) != ref_id(r2):
        return ref_id(r1) < ref_id(r2)
    return unclipped_5prime(r1) <= unclipped_5prime(r2)


def orientation(r1, r2):   # group.rs:282-293
    return (r1 is None or not flags(r1) & REVERSE, r2 is None or not flags(r2) & REVERSE)


def prepare_group(records: Sequence[bytes], cfg: Config):
    """Everything of process_and_write_position_group (group.rs:1460-1522) before the assigner runs:
    (templates that pass, calls as lists of template indices, UMIs per call, dropped, filter counts)."""
    m = [0] * 6
    tpls = [t for t in build_templates(records) if filter_template(t[1], t[2], cfg, m)]
    if not tpls:
        return tpls, [], [], False, m
    if cfg.assign_strategy != U.PAIRED:   # split by orientation, sub-groups in (bool, bool) order (:382-407)
        subs: Dict[Tuple[bool, bool], List[int]] = {}
        for i, (_, r1, r2) in enumerate(tpls):
            subs.setdefault(orientation(r1, r2), []).append(i)
        calls = [subs[k] for k in sorted(subs)]
    else:
        calls = [list(range(len(tpls)))]
    umis = []
    for call in calls:
        cu = []
        for i in call:
            _, r1, r2 = tpls[i]
            if cfg.no_umi:
                cu.append(b"")
                continue
            u = find_string_tag(r1 if r1 is not None else r2, cfg.umi_tag)
            if u is None or not _utf8(u):   # "Missing UMI tag" / "Invalid UTF-8 in UMI": the group is dropped
                return tpls, calls, [], True, m
            early = is_r1_earlier(r1, r2) if r1 is not None and r2 is not None else True
            try:
                cu.append(U.umi_for_read(u, early, cfg.assign_strategy, cfg.rules, cfg.assign_edits))
            except U.UmiError:   # :311-317 bails: the group is dropped (:1512-1522)
                return tpls, calls, [], True, m
        umis.append(cu)
    return tpls, calls, umis, False, m


def update_string_tag(rec: bytes, tag: bytes, value: bytes) -> bytes:   # tags.rs:694-721
    for p, t, vt, size in aux_entries(rec):
        if t == tag and size is not None:
            if size - 1 == len(value):   # end - start - 4 == new length: overwrite, the type byte stays
                return rec[:p + 3] + value + rec[p + 3 + len(value):]
            return rec[:p] + tag + b"Z" + value + b"\0" + rec[p + 3 + size:]
        if t == tag or size is None:
            break
    return rec + tag + b"Z" + value + b"\0"


def vec_index(kind: int, i: int):   # lib.rs:112-119; None sorts first
    if kind == U.NONE:
        return (0, 0)
    return (1, i if kind == U.SINGLE else 2 * i + (kind == U.B))


class Grouper:
    """The grouper over a stream of position groups: add_groups, pending (the UMI batch), flush."""

    def __init__(self, cfg: Config):
        cfg.check()
        self.cfg = cfg
        self.queue = []
        self.stats = [0] * len(STATS)
        self.stats[8] = cfg.first_mi
        self.family_sizes: Dict[int, int] = {}
        self.group_sizes: Dict[int, int] = {}

    def add_groups(self, records: Sequence[bytes], group_begin: Sequence[int]):
        prepped = [prepare_group(records[group_begin[g]:group_begin[g + 1]], self.cfg)
                   for g in range(len(group_begin) - 1)]   # raises before anything is queued
        for tpls, calls, umis, dropped, m in prepped:
            for k in range(6):
                self.stats[k] += m[k]
            self.stats[6] += 1
            self.stats[7] += dropped
            if tpls and not dropped:
                self.queue.append((tpls, calls, umis))

    def pending(self):
        """groups -> calls -> UMIs, as umi_oracle.assign_groups takes them."""
        return [umis for _, _, umis in self.queue]

    def assign(self):
        c = self.cfg
        return U.assign_groups(c.assign_strategy, c.rules, c.assign_edits, self.pending(), c.assign_min_len)

    def flush(self, assignment=None) -> bytes:
        """The ConsensusOutput-style stream ([u32 block_size][record]...) of every queued group (group.rs:1524-1592,
        1650-1682).  assignment: (kinds, ids, group_mi_count) in the order of pending(); the oracle's own if None."""
        kinds, ids, counts = assignment if assignment is not None else self.assign()
        out = bytearray()
        u = 0
        for gi, (tpls, calls, _) in enumerate(self.queue):
            mol = [None] * len(tpls)
            for call in calls:
                for t in call:
                    mol[t] = (kinds[u], ids[u])
                    u += 1
            order = sorted(range(len(tpls)), key=lambda t: (vec_index(*mol[t]), tpls[t][0]))
            fams = []
            for t in order:
                v = vec_index(*mol[t])
                if fams and fams[-1][0] == v:
                    fams[-1][1] += 1
                else:
                    fams.append([v, 1])
            fams = [n for v, n in fams if v[0]]
            for n in fams:
                self.family_sizes[n] = self.family_sizes.get(n, 0) + 1
            if fams:
                self.group_sizes[len(fams)] = self.group_sizes.get(len(fams), 0) + 1
            base = self.stats[8]
            self.stats[8] += counts[gi]
            for t in order:
                _, r1, r2 = tpls[t]
                kind, i = mol[t]
                for r in (r1, r2):
                    if r is None:
                        continue
                    if kind != U.NONE:
                        r = update_string_tag(r, self.cfg.assign_tag, U.mi_string(kind, i, base).encode())
                    out += struct.pack("<I", len(r)) + r
                    self.stats[9] += 1
        self.queue = []
        return bytes(out)


def grouping_metrics(stats: Sequence[int], family_sizes: Dict[int, int]) -> dict:
    """build_grouping_metrics (group.rs:670-716)."""
    m = dict(total_records=stats[0], accepted_records=stats[1], discarded_non_pf=stats[2],
             discarded_poor_alignment=stats[3], discarded_ns_in_umi=stats[4], discarded_umi_too_short=stats[5])
    total = sum(family_sizes.values())
    m.update(total_families=total, unique_molecule_ids=total, avg_reads_per_molecule=0.0,
             median_reads_per_molecule=0, min_reads_per_molecule=0, max_reads_per_molecule=0)
    if total:
        m["avg_reads_per_molecule"] = stats[1] / total
    if family_sizes:
        sizes = sorted(family_sizes.items())
        cum = 0
        for s, c in sizes:
            cum += c
            if cum >= total // 2:
                m["median_reads_per_molecule"] = s
                break
        m["min_reads_per_molecule"] = sizes[0][0]
        m["max_reads_per_molecule"] = sizes[-1][0]
    return m


def group_stream(records: Sequence[bytes], header_text: bytes, cfg: Config, cell_tag: Optional[bytes] = b"CB"):
    """The whole of `group` on a record stream: (output stream, grouper)."""
    keep, begin = group_by_position(records, header_text, cell_tag)
    g = Grouper(cfg)
    g.add_groups([r for r, k in zip(records, keep) if k], begin)
    return g.flush(), g
