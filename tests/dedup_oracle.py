"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Restatement (pure Python) of `fgumi dedup` around the UMI assignment, record bytes in, record bytes out, in the
single-threaded order of the reference, on top of oracle/group_oracle.py (records, aux walk, position keys,
update_string_tag) and oracle/umi_oracle.py (the assigners).  Citations are relative to the fgumi 0.2.0 source tree:
  dedup.rs    src/lib/commands/dedup.rs              (filter, UMIs, scores, duplicate marking, metrics)
  grouper.rs  src/lib/grouper.rs                     (RecordPositionGrouper::with_secondary_supplementary)
  bam.rs      src/lib/unified_pipeline/bam.rs        (the default key of secondary / supplementary records)
  template    src/lib/template.rs                    (Template::from_records)
"""
from __future__ import annotations

import os
import struct
import sys
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import group_oracle as G   # noqa: E402
from oracle import umi_oracle as U     # noqa: E402

DUPLICATE = 0x400
I32_MAX = G.I32_MAX
DEFAULT_KEY = (I32_MAX, I32_MAX, 255, I32_MAX, I32_MAX, 255, 0, None)   # GroupKey::default() (base.rs:1453-1466)

STATS = ("total_templates", "unique_templates", "duplicate_templates", "total_reads", "unique_reads",
         "duplicate_reads", "secondary_reads", "supplementary_reads", "missing_tc_tag", "total_records",
         "accepted_records", "discarded_non_pf", "discarded_poor_alignment", "discarded_ns_in_umi",
         "discarded_umi_too_short", "position_groups", "next_mi", "records_out")


class DedupError(ValueError):
    """Where the reference fails the command: the product fails the call."""


# ---- position grouping with secondary and supplementary records ---------------------------------------------------
def group_by_position(records: Sequence[bytes], header_text: bytes = b"", cell_tag: Optional[bytes] = b"CB"):
    """RecordPositionGrouper::with_secondary_supplementary (grouper.rs:437-444, 488-547): every record kept; a secondary
    or supplementary record has the default key (bam.rs:431-435) and is not MC-checked.  (keep, group_begin)."""
    libs = G.library_index(header_text)
    begin = []
    cur = last = None
    for i, r in enumerate(records):
        f = G.flags(r)
        k = G.position_key(r, libs, cell_tag)
        if k is None:
            k = DEFAULT_KEY
        elif f & G.PAIRED and not f & (G.UNMAPPED | G.MATE_UNMAPPED):
            mc = G.find_string_tag(r, b"MC")
            if mc is None or not G._utf8(mc):
                raise G.GroupError("RecordPositionGrouper requires MC tags on paired-end reads", record=i)
        same = cur is not None and (k == cur or G.name(last) == G.name(r))
        if not same:
            begin.append(i)
            cur = k
        last = r
    begin.append(len(records))
    return [1] * len(records), begin


# ---- templates, filter, score ----------------------------------------------------------------------------------------
@dataclass
class Template:
    name: bytes
    r1: Optional[bytes]
    r2: Optional[bytes]
    records: List[bytes]   # Template::from_records order


def build_templates(records: Sequence[bytes]) -> List[Template]:
    """build_templates_from_records + Template::from_records (template.rs:159-330): R1, R2, R1 supplementaries, R2
    supplementaries, R1 secondaries, R2 secondaries, each list reversed; secondary wins over supplementary."""
    out = []
    i = 0
    while i < len(records):
        nm = G.name(records[i])
        j = i + 1
        while j < len(records) and G.name(records[j]) == nm:
            j += 1
        r1 = r2 = None
        lists = {k: [] for k in ("r1_supp", "r2_supp", "r1_sec", "r2_sec")}
        for r in records[i:j]:
            f = G.flags(r)
            is_r1 = not f & G.PAIRED or f & G.FIRST
            if f & G.SECONDARY:
                lists["r1_sec" if is_r1 else "r2_sec"].append(r)
            elif f & G.SUPPLEMENTARY:
                lists["r1_supp" if is_r1 else "r2_supp"].append(r)
            elif is_r1:
                if r1 is not None:
                    raise DedupError("Multiple non-secondary, non-supplemental R1 records")
                r1 = r
            else:
                if r2 is not None:
                    raise DedupError("Multiple non-secondary, non-supplemental R2 records")
                r2 = r
        recs = [r for r in (r1, r2) if r is not None]
        for k in ("r1_supp", "r2_supp", "r1_sec", "r2_sec"):
            recs += lists[k][::-1]
        out.append(Template(nm, r1, r2, recs))
        i = j
    return out


def read_score(r: bytes) -> int:
    """score_template's per-read term (dedup.rs:233-246)."""
    if len(r) < 32:
        return 0
    n_cig = struct.unpack_from("<H", r, 12)[0]
    l_seq = struct.unpack_from("<I", r, 16)[0]
    qo = 32 + r[8] + 4 * n_cig + (l_seq + 1) // 2
    if qo >= len(r):
        return 0
    return sum(min(q, 15) for q in r[qo:qo + min(l_seq, len(r) - qo)])


def score_template(t: Template) -> int:   # dedup.rs:230-249
    return sum(read_score(r) for r in (t.r1, t.r2) if r is not None)


@dataclass
class Config:
    strategy: int = U.ADJACENCY
    edits: int = 1
    min_umi_length: Optional[int] = None
    min_map_q: int = 0
    include_non_pf: bool = False
    no_umi: bool = False
    remove_duplicates: bool = False
    umi_tag: bytes = b"RX"
    assign_tag: bytes = b"MI"
    first_mi: int = 0

    def check(self):   # dedup.rs:913-921
        if self.strategy == U.PAIRED and (self.min_umi_length or self.no_umi):
            raise DedupError("paired strategy with --min-umi-length or --no-umi")

    @property
    def assign_strategy(self):   # :923-931
        return U.IDENTITY if self.no_umi else self.strategy

    @property
    def assign_edits(self):   # :940-947
        return 0 if self.no_umi or self.strategy == U.IDENTITY else self.edits

    @property
    def assign_min_len(self):
        return None if self.no_umi else self.min_umi_length


def filter_template(t: Template, cfg: Config, m: List[int]) -> bool:
    """filter_template (dedup.rs:257-402); m: [total, accepted, non_pf, poor_alignment, ns_in_umi, too_short], counted
    per template."""
    reads = [r for r in (t.r1, t.r2) if r is not None]
    m[0] += 1
    if not reads or all(G.flags(r) & G.UNMAPPED for r in reads):
        m[3] += 1
        return False
    for r in reads:
        f = G.flags(r)
        if not cfg.include_non_pf and f & G.QC_FAIL:
            m[2] += 1
            return False
        if not f & G.UNMAPPED and r[9] < cfg.min_map_q:
            m[3] += 1
            return False
    for r in reads:
        check_mq = not G.flags(r) & G.MATE_UNMAPPED
        mq, umi = aux_mq_umi(r, check_mq, not cfg.no_umi, cfg.umi_tag)
        if check_mq and mq is not None and mq < cfg.min_map_q:   # signed (:363-372)
            m[3] += 1
            return False
        if cfg.no_umi:
            continue
        if umi is None:
            m[3] += 1
            return False
        bases = G.validate_umi(umi)
        if bases is None:
            m[4] += 1
            return False
        if cfg.min_umi_length and bases < cfg.min_umi_length:
            m[5] += 1
            return False
    m[1] += 1
    return True


def aux_mq_umi(r: bytes, check_mq: bool, check_umi: bool, umi_tag: bytes):
    """The one aux walk of dedup.rs:306-361: (MQ as a signed integer or None, the UMI or None)."""
    mq = umi = None
    p = G.aux_off(r)
    while p + 3 <= len(r):
        t, vt = r[p:p + 2], r[p + 2]
        if check_umi and t == umi_tag and vt == ord("Z"):
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
        size = G.tag_value_size(vt, r[p + 3:])
        if size is None:
            break
        p += 3 + size
        if (not check_umi or umi is not None) and (not check_mq or mq is not None):
            break
    return mq, umi


def set_flags(r: bytes, f: int) -> bytes:
    return r[:14] + struct.pack("<H", f) + r[16:]


def clear_duplicate(t: Template) -> Template:   # dedup.rs:706-716
    recs = [set_flags(r, G.flags(r) & ~DUPLICATE) for r in t.records]
    k = 0
    r1 = r2 = None
    if t.r1 is not None:
        r1, k = recs[0], 1
    if t.r2 is not None:
        r2 = recs[k]
    return Template(t.name, r1, r2, recs)


def umi_for_template(t: Template, cfg: Config) -> bytes:
    """assign_umi_groups_for_indices (dedup.rs:500-526): R1's UMI else R2's, through umi_for_read."""
    if cfg.no_umi:
        return b""
    u = G.find_string_tag(t.r1 if t.r1 is not None else t.r2, cfg.umi_tag)
    if u is None:
        raise DedupError("No UMI tag found")
    if not G._utf8(u):
        raise DedupError("Invalid UTF-8")
    early = G.is_r1_earlier(t.r1, t.r2) if t.r1 is not None and t.r2 is not None else True
    try:
        return U.umi_for_read(u, early, cfg.assign_strategy, U.MAPPED, cfg.assign_edits)
    except U.UmiError as e:
        raise DedupError(str(e))


def prepare_group(records: Sequence[bytes], cfg: Config):
    """process_position_group up to the assigner (dedup.rs:684-719): (templates that pass, calls as lists of template
    indices, UMIs per call, filter counts).  Raises DedupError where the reference fails the command."""
    m = [0] * 6
    tpls = [clear_duplicate(t) for t in build_templates(records) if filter_template(t, cfg, m)]
    if not tpls:
        return tpls, [], [], m
    if cfg.assign_strategy != U.PAIRED:   # orientation sub-groups in (bool, bool) order (:550-573)
        subs: Dict[tuple, List[int]] = {}
        for i, t in enumerate(tpls):
            subs.setdefault(G.orientation(t.r1, t.r2), []).append(i)
        calls = [subs[k] for k in sorted(subs)]
    else:
        calls = [list(range(len(tpls)))]
    umis = [[umi_for_template(tpls[i], cfg) for i in call] for call in calls]
    return tpls, calls, umis, m


def representative(scores: Sequence[int]) -> int:
    """mark_duplicates_in_family (dedup.rs:598-657) on a family in sorted order: the index it keeps."""
    n = len(scores)
    if n <= 1:
        return 0
    if n == 2:
        return 0 if scores[0] >= scores[1] else 1
    if n == 3:
        s0, s1, s2 = scores
        if s0 >= s1 and s0 >= s2:
            return 0
        if s1 >= s0 and s1 >= s2:
            return 1
        return 2
    return sorted(range(n), key=lambda i: -scores[i])[0]   # a stable sort by score descending


def has_tag(r: bytes, tag: bytes) -> bool:   # find_tag_type: an entry of any type
    for _, t, _, _ in G.aux_entries(r):
        if t == tag:
            return True
    return False


class Deduper:
    """The deduper over a stream of position groups: add_groups, pending (the UMI batch), flush."""

    def __init__(self, cfg: Config):
        cfg.check()
        self.cfg = cfg
        self.queue = []
        self.stats = [0] * len(STATS)
        self.stats[16] = cfg.first_mi
        self.family_sizes: Dict[int, int] = {}
        self.later_representatives = 0   # families whose kept template is not the first in (MI, QNAME) order

    def add_groups(self, records: Sequence[bytes], group_begin: Sequence[int]):
        prepped = [prepare_group(records[group_begin[g]:group_begin[g + 1]], self.cfg)
                   for g in range(len(group_begin) - 1)]   # raises before anything is queued
        for tpls, calls, umis, m in prepped:
            for k in range(6):
                self.stats[9 + k] += m[k]
            self.stats[15] += 1
            if tpls:
                self.queue.append((tpls, calls, umis))

    def pending(self):
        return [umis for _, _, umis in self.queue]

    def assign(self):
        c = self.cfg
        return U.assign_groups(c.assign_strategy, U.MAPPED, c.assign_edits, self.pending(), c.assign_min_len)

    def scores(self):
        """Template scores in the order of the pending batch."""
        return [score_template(tpls[t]) for tpls, calls, _ in self.queue for call in calls for t in call]

    def flush(self, assignment=None, scores=None) -> bytes:
        """The output stream ([u32 block_size][record]...) of every queued group (dedup.rs:721-806, 1080-1110).
        assignment: (kinds, ids, group_mi_count) and scores in the order of pending(); the oracle's own if None."""
        kinds, ids, counts = assignment if assignment is not None else self.assign()
        scores = scores if scores is not None else self.scores()
        out = bytearray()
        u = 0
        s = self.stats
        for gi, (tpls, calls, _) in enumerate(self.queue):
            mol = [None] * len(tpls)
            sc = [0] * len(tpls)
            for call in calls:
                for t in call:
                    mol[t] = (kinds[u], ids[u])
                    sc[t] = scores[u]
                    u += 1
            order = sorted(range(len(tpls)), key=lambda t: (G.vec_index(*mol[t]), tpls[t].name))
            dup = [False] * len(tpls)
            fams = []
            for t in order:
                v = G.vec_index(*mol[t])
                if fams and fams[-1][0] == v:
                    fams[-1][1].append(t)
                else:
                    fams.append([v, [t]])
            for v, members in fams:
                if not v[0]:
                    continue   # unassigned (:751-754)
                self.family_sizes[len(members)] = self.family_sizes.get(len(members), 0) + 1
                keep = representative([sc[t] for t in members])
                self.later_representatives += keep != 0
                s[1] += 1
                for x, t in enumerate(members):
                    if x != keep:
                        dup[t] = True
                        s[2] += 1
            base = s[16]
            s[16] += counts[gi]
            for t in order:
                kind, i = mol[t]
                s[0] += 1
                for r in tpls[t].records:
                    f = G.flags(r)
                    s[3] += 1
                    if dup[t]:
                        s[5] += 1
                        r = set_flags(r, f | DUPLICATE)
                    if f & G.SECONDARY:
                        s[6] += 1
                    if f & G.SUPPLEMENTARY:
                        s[7] += 1
                    if f & (G.SECONDARY | G.SUPPLEMENTARY) and not has_tag(r, b"tc"):
                        s[8] += 1
                    if dup[t] and self.cfg.remove_duplicates:
                        continue
                    if kind != U.NONE:
                        r = G.update_string_tag(r, self.cfg.assign_tag, U.mi_string(kind, i, base).encode())
                    out += struct.pack("<I", len(r)) + r
                    s[17] += 1
        s[4] = s[3] - s[5]
        self.queue = []
        return bytes(out)


def dedup_metrics(stats: Sequence[int]) -> dict:
    """DedupMetricsOutput (dedup.rs:122-150)."""
    names = ("total_templates", "unique_templates", "duplicate_templates", "duplicate_rate", "total_reads",
             "unique_reads", "duplicate_reads", "secondary_reads", "supplementary_reads", "missing_tc_tag")
    d = dict(zip(STATS, stats))
    d["duplicate_rate"] = d["duplicate_templates"] / d["total_templates"] if d["total_templates"] else 0.0
    return {k: d[k] for k in names}


def dedup_stream(records: Sequence[bytes], header_text: bytes, cfg: Config, cell_tag: Optional[bytes] = b"CB"):
    """The whole of `dedup` on a record stream: (output stream, deduper)."""
    _, begin = group_by_position(records, header_text, cell_tag)
    d = Deduper(cfg)
    d.add_groups(records, begin)
    return d.flush(), d
