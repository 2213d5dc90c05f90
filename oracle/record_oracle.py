"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Record-level restatement (pure Python, small cases only) of the HOST side of fgumi's consensus
callers: raw BAM record decoding, source-read preparation, CIGAR grouping, the group / orphan rules
and consensus-record assembly.  The per-position vote itself is delegated to the C++ oracle
(oracle/liboracle.so).  Only tests/ may import this.  Citations are relative to the fgumi 0.2.0 source tree.

Parity status: the reference has no golden outputs and cannot be built here, so byte-level parity
with the fgumi binary is "parity unpinned"; this file is checked against the reference's own
known-answer unit tests where they exist (tests/test_record_oracle_kat.py).
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# ---- fgumi-raw-bam/src/fields.rs:240-265 -------------------------------------------------------
PAIRED, PROPER_PAIR, UNMAPPED, MATE_UNMAPPED = 0x1, 0x2, 0x4, 0x8
REVERSE, MATE_REVERSE, FIRST_SEGMENT, LAST_SEGMENT = 0x10, 0x20, 0x40, 0x80
SECONDARY, QC_FAIL, DUPLICATE, SUPPLEMENTARY = 0x100, 0x200, 0x400, 0x800

BAM_BASE_TO_ASCII = b"=ACMGRSVTWYHKDBN"            # sequence.rs:9-11
SEQ_CODES = [15] * 256                              # sequence.rs:18-35
for _i, _b in enumerate(BAM_BASE_TO_ASCII):
    SEQ_CODES[_b] = _i
    SEQ_CODES[ord(chr(_b).lower())] = _i

# ops: 0 M,1 I,2 D,3 N,4 S,5 H,6 P,7 =,8 X ; cigar.rs:50-70 (BAM_CIGAR_TYPE = 0x3C1A7)
def consumes_query(op: int) -> bool:
    return (0x3C1A7 >> ((op & 0xF) << 1)) & 1 != 0


def consumes_ref(op: int) -> bool:
    return (0x3C1A7 >> ((op & 0xF) << 1)) & 2 != 0


class Rec:
    """RawRecordView, fgumi-raw-bam/src/fields.rs:6-23 + accessors."""

    def __init__(self, b: bytes):
        self.b = bytes(b)
        (self.ref_id, self.pos, self.l_read_name, self.mapq, self.bin, self.n_cigar, self.flags,
         self.l_seq, self.mate_ref_id, self.mate_pos, self.tlen) = struct.unpack_from("<iiBBHHHIiii", self.b, 0)

    @property
    def name(self) -> bytes:                         # fields.rs:393-396
        l = self.l_read_name
        return self.b[32:32 + l - 1] if l > 1 else b""

    def cigar_ops(self) -> List[int]:                # cigar.rs:82-101
        if self.n_cigar == 0:
            return []
        s = 32 + self.l_read_name
        e = s + 4 * self.n_cigar
        if e > len(self.b):
            return []
        return list(struct.unpack_from("<%dI" % self.n_cigar, self.b, s))

    def seq_offset(self) -> int:                     # fields.rs:488-492
        return 32 + self.l_read_name + 4 * self.n_cigar

    def sequence(self) -> bytearray:                 # sequence.rs:148-173 (scalar semantics)
        off = self.seq_offset()
        out = bytearray(self.l_seq)
        for i in range(self.l_seq):
            byte = self.b[off + i // 2]
            out[i] = BAM_BASE_TO_ASCII[byte >> 4 if i % 2 == 0 else byte & 0xF]
        return out

    def quals(self) -> bytearray:                    # fields.rs:497-502
        off = self.seq_offset() + (self.l_seq + 1) // 2
        return bytearray(self.b[off:off + self.l_seq])

    def aux(self) -> bytes:                          # fields.rs:449-483
        off = 32 + self.l_read_name + 4 * self.n_cigar + (self.l_seq + 1) // 2 + self.l_seq
        return self.b[off:] if off <= len(self.b) else b""

    def find_string(self, tag: bytes) -> Optional[bytes]:   # tags.rs:13-48
        aux = self.aux()
        p = 0
        fixed = {ord("A"): 1, ord("c"): 1, ord("C"): 1, ord("s"): 2, ord("S"): 2, ord("i"): 4,
                 ord("I"): 4, ord("f"): 4}
        while p + 3 <= len(aux):
            t, vt = aux[p:p + 2], aux[p + 2]
            if t == tag:
                if vt != ord("Z"):
                    return None
                end = aux.find(b"\0", p + 3)
                return None if end < 0 else aux[p + 3:end]
            if vt in fixed:
                size = fixed[vt]
            elif vt in (ord("Z"), ord("H")):
                end = aux.find(b"\0", p + 3)
                if end < 0:
                    break
                size = end - (p + 3) + 1
            elif vt == ord("B"):
                if len(aux) - (p + 3) < 5:
                    break
                es = fixed.get(aux[p + 3], 0)
                if es == 0:
                    break
                size = 5 + struct.unpack_from("<I", aux, p + 4)[0] * es
            else:
                break
            p += 3 + size
        return None


# ---- cigar helpers -----------------------------------------------------------------------------
def reference_length(ops: Sequence[int]) -> int:      # cigar.rs:137-150
    return sum(op >> 4 for op in ops if consumes_ref(op & 0xF))


def simplify_cigar(ops: Sequence[int]) -> List[Tuple[int, int]]:   # noodles_compat.rs:10-55
    out: List[Tuple[int, int]] = []
    for raw in ops:
        ln, t = raw >> 4, raw & 0xF
        if t > 8:
            continue
        kind = 0 if t in (4, 7, 8, 5) else t          # S, =, X, H -> M
        if out and out[-1][0] == kind:
            out[-1] = (kind, out[-1][1] + ln)
        else:
            out.append((kind, ln))
    return out


def is_cigar_prefix(a, b) -> bool:                    # fgumi-sam clipper.rs:2425-2448
    if len(a) > len(b):
        return False
    last = max(len(a) - 1, 0)
    for i, (op_a, len_a) in enumerate(a):
        op_b, len_b = b[i]
        if op_a != op_b:
            return False
        if i == last:
            if len_a > len_b:
                return False
        elif len_a != len_b:
            return False
    return True


def _parse_leading_clips(cigar: str) -> int:          # cigar.rs:514-536
    clipped, num_start = 0, 0
    for i, c in enumerate(cigar):
        if c.isdigit():
            continue
        try:
            num = int(cigar[num_start:i])
        except ValueError:
            num = 0
        if c in "SH":
            clipped += num
            num_start = i + 1
        else:
            break
    return clipped


def _parse_ref_len_and_trailing_clips(cigar: str) -> Tuple[int, int]:   # cigar.rs:544-573
    ref_len = trailing = num_start = 0
    saw = False
    for i, c in enumerate(cigar):
        if c.isdigit():
            continue
        try:
            num = int(cigar[num_start:i])
        except ValueError:
            num = 0
        num_start = i + 1
        if c in "MDN=X":
            ref_len += num
            trailing = 0
            saw = True
        elif c in "SH" and saw:
            trailing += num
    return ref_len, trailing


def is_fr_pair(r: Rec) -> bool:                       # overlap.rs:15-62
    f = r.flags
    if not f & PAIRED:
        return False
    if f & UNMAPPED or f & MATE_UNMAPPED:
        return False
    if r.ref_id != r.mate_ref_id:
        return False
    rev, mrev = bool(f & REVERSE), bool(f & MATE_REVERSE)
    if rev == mrev:
        return False
    start = r.pos + 1
    mstart = r.mate_pos + 1
    if rev:
        ref_len = reference_length(r.cigar_ops())
        end = start + max(ref_len - 1, 0)
        pos5, neg5 = mstart, end
    else:
        pos5, neg5 = start, start + r.tlen
    return pos5 < neg5


def _read_pos_at_ref(ops, start1, target, at_or_past: bool) -> int:   # overlap.rs:148-204
    ref_pos, read_pos = start1, 0
    for op in ops:
        t, ln = op & 0xF, op >> 4
        if t in (0, 7, 8):
            for _ in range(ln):
                read_pos += 1
                if ref_pos == target:
                    return read_pos if at_or_past else max(read_pos - 1, 0)
                ref_pos += 1
        elif t in (1, 4):
            read_pos += ln
        elif t in (2, 3):
            for _ in range(ln):
                if ref_pos == target:
                    return 0
                ref_pos += 1
    return 0


def num_bases_extending_past_mate(r: Rec) -> int:     # overlap.rs:65-136
    if not is_fr_pair(r):
        return 0
    mc = r.find_string(b"MC")
    if mc is None:
        return 0
    try:
        mc_s = mc.decode("utf-8")
    except UnicodeDecodeError:
        return 0
    ops = r.cigar_ops()
    this_pos, m_pos = r.pos + 1, r.mate_pos + 1
    read_length = sum(op >> 4 for op in ops if consumes_query(op & 0xF))
    if r.flags & REVERSE:
        mate_us = m_pos - _parse_leading_clips(mc_s)
        if this_pos <= mate_us:
            return _read_pos_at_ref(ops, this_pos, mate_us, False)
        lead = 0
        for op in ops:
            if op & 0xF == 4:
                lead += op >> 4
            elif op & 0xF == 5:
                pass
            else:
                break
        return max(lead - (this_pos - mate_us), 0)
    ref_len = reference_length(ops)
    aln_end = this_pos + ref_len - 1
    rl, tc = _parse_ref_len_and_trailing_clips(mc_s)
    mate_ue = m_pos + rl + tc - 1
    if aln_end >= mate_ue:
        past = _read_pos_at_ref(ops, this_pos, mate_ue, True)
        return max(read_length - past, 0)
    trail = 0
    for op in reversed(ops):
        if op & 0xF == 4:
            trail += op >> 4
        elif op & 0xF == 5:
            pass
        else:
            break
    return max(trail - (mate_ue - aln_end), 0)


# ---- fgumi-dna/src/dna.rs:30-60 ----------------------------------------------------------------
_COMP = {ord("A"): ord("T"), ord("a"): ord("T"), ord("T"): ord("A"), ord("t"): ord("A"),
         ord("C"): ord("G"), ord("c"): ord("G"), ord("G"): ord("C"), ord("g"): ord("C")}


def reverse_complement(seq: bytes) -> bytearray:
    return bytearray(_COMP.get(b, b) for b in reversed(seq))


# ---- vanilla_caller.rs --------------------------------------------------------------------------
@dataclass
class VanillaOptions:                                 # vanilla_caller.rs:284-341
    tag: bytes = b"MI"
    error_rate_pre_umi: int = 45
    error_rate_post_umi: int = 40
    min_input_base_quality: int = 10
    min_reads: int = 2
    produce_per_base_tags: bool = True
    trim: bool = False
    min_consensus_base_quality: int = 40
    cell_tag: Optional[bytes] = None


@dataclass
class SourceRead:                                     # vanilla_caller.rs:129-146
    original_idx: int
    bases: bytearray
    quals: bytearray
    simplified_cigar: list
    flags: int


def find_quality_trim_point(quals: Sequence[int], trim_qual: int) -> int:   # vanilla_caller.rs:780-804
    length = len(quals)
    if trim_qual < 1 or length == 0:
        return 0
    score = max_score = 0
    trim_point = length
    for i in range(length - 1, -1, -1):
        score += trim_qual - quals[i]
        if score < 0:
            break
        if score > max_score:
            max_score = score
            trim_point = i
    return trim_point


def truncate_simplified_cigar(cigar, query_length: int):     # vanilla_caller.rs:816-851
    result, remaining = [], query_length
    for kind, ln in cigar:
        if remaining == 0:
            break
        if kind in (0, 1, 4, 7, 8):
            take = min(ln, remaining)
            result.append((kind, take))
            remaining -= take
        else:
            result.append((kind, ln))
    return result


def create_source_read(r: Rec, idx: int, mate_clip: int, opt: VanillaOptions) -> Optional[SourceRead]:
    """vanilla_caller.rs:863-955"""
    neg = bool(r.flags & REVERSE)
    min_bq = opt.min_input_base_quality
    bases, quals = r.sequence(), r.quals()
    read_len = len(bases)
    if len(quals) == 0 or len(quals) != read_len:
        return None
    if all(q == 0xFF for q in quals):
        return None
    if neg:
        bases = reverse_complement(bases)
        quals = bytearray(reversed(quals))
    trim_to = find_quality_trim_point(quals, min_bq) if opt.trim else read_len
    for i in range(trim_to):
        if quals[i] < min_bq:
            bases[i] = ord("N")
            quals[i] = 2
    clip_position = max(read_len - mate_clip, 0)
    final_len = min(clip_position, trim_to)
    while final_len > 0 and bases[final_len - 1] == ord("N"):
        final_len -= 1
    if final_len == 0:
        return None
    bases, quals = bases[:final_len], quals[:final_len]
    simp = simplify_cigar(r.cigar_ops())
    if neg:
        simp = list(reversed(simp))
    simp = truncate_simplified_cigar(simp, final_len)
    return SourceRead(idx, bases, quals, simp, r.flags)


_KIND_ORD = {0: 0, 1: 1, 2: 2, 3: 3, 4: 4, 5: 5, 6: 6, 7: 7, 8: 8}


def _cmp_cigar(a, b) -> int:                          # vanilla_caller.rs:77-105
    for (ka, la), (kb, lb) in zip(a, b):
        if la != lb:
            return -1 if la < lb else 1
        if _KIND_ORD[ka] != _KIND_ORD[kb]:
            return -1 if _KIND_ORD[ka] < _KIND_ORD[kb] else 1
    return (len(a) > len(b)) - (len(a) < len(b))


def select_most_common_alignment_group(indexed) -> List[int]:     # vanilla_caller.rs:47-119
    if len(indexed) < 2:
        return [i for i, _, _ in indexed]
    groups: List[Tuple[list, List[int]]] = []
    for idx, _len, cigar in indexed:
        found = False
        for gc, members in groups:
            if is_cigar_prefix(cigar, gc):
                members.append(idx)
                found = True
        if not found:
            groups.append((list(cigar), [idx]))
    # Iterator::max_by returns the LAST maximum; key: size asc, then cmp_cigar(b, a)
    best = None
    for g in groups:
        if best is None:
            best = g
            continue
        c = (len(g[1]) > len(best[1])) - (len(g[1]) < len(best[1]))
        if c == 0:
            c = _cmp_cigar(best[0], g[0])             # cmp(g, best) = cmp_cigar(best.cigar, g.cigar)
        if c >= 0:
            best = g
    return list(best[1]) if best else []


def filter_by_alignment(srs: List[SourceRead]):       # vanilla_caller.rs:961-1013
    if len(srs) < 2:
        return srs, 0
    indexed = [(i, len(sr.bases), sr.simplified_cigar) for i, sr in enumerate(srs)]
    indexed.sort(key=lambda t: -t[1])                 # stable sort, descending length
    keep = set(select_most_common_alignment_group(indexed))
    kept = [sr for i, sr in enumerate(srs) if i in keep]
    return kept, len(srs) - len(keep)


# ---- simple_umi.rs ------------------------------------------------------------------------------
def consensus_umis(umis: List[str], vote) -> str:     # simple_umi.rs:65-122, 236-245
    if not umis:
        return ""
    if len(umis) == 1:
        return umis[0]
    first = umis[0]
    n = len(first)
    assert all(len(s) == n for s in umis)
    out = []
    for i in range(n):
        col = [s[i] for s in umis]
        dna = [c for c in col if c.upper() in "ACGTN"]
        if len(dna) == len(col):
            b, _q = vote(90, 90, "".join(col).encode(), [20] * len(col))
            out.append(b)
        elif not dna:
            assert all(c == first[i] for c in col)
            out.append(first[i])
        else:
            raise AssertionError("mix of DNA and non-DNA characters")
    return "".join(out)


# ---- raw-bam builder.rs / tags.rs encoders -------------------------------------------------------
def pack_sequence(bases: bytes) -> bytes:             # sequence.rs:183-209
    out = bytearray()
    for i in range(0, len(bases) - 1, 2):
        out.append((SEQ_CODES[bases[i]] << 4) | SEQ_CODES[bases[i + 1]])
    if len(bases) % 2:
        out.append(SEQ_CODES[bases[-1]] << 4)
    return bytes(out)


def tag_string(tag: bytes, v: bytes) -> bytes:        # tags.rs:512-519
    return tag + b"Z" + v + b"\0"


def tag_int(tag: bytes, v: int) -> bytes:             # tags.rs:533-553
    if -128 <= v <= 127:
        return tag + b"c" + struct.pack("<b", v)
    if 0 <= v <= 255:
        return tag + b"C" + struct.pack("<B", v)
    if 0 <= v <= 65535:
        return tag + b"S" + struct.pack("<H", v)
    if -32768 <= v <= 32767:
        return tag + b"s" + struct.pack("<h", v)
    return tag + b"i" + struct.pack("<i", v)


def tag_float(tag: bytes, v) -> bytes:                # tags.rs:557-563
    return tag + b"f" + struct.pack("<f", v)


def tag_i16_array(tag: bytes, vals) -> bytes:         # tags.rs:573-586
    return tag + b"Bs" + struct.pack("<I", len(vals)) + struct.pack("<%dh" % len(vals), *vals)


def tag_phred33(tag: bytes, quals) -> bytes:          # tags.rs:656-667
    return tag + b"Z" + bytes(min(q + 33, 255) for q in quals) + b"\0"


def unmapped_record(name: bytes, flag: int, bases: bytes, quals: bytes) -> bytearray:   # builder.rs:90-142
    assert len(name) < 255
    out = bytearray(struct.pack("<iiBBHHHIiii", -1, -1, len(name) + 1, 0, 4680, 0, flag, len(bases),
                                -1, -1, 0))
    out += name + b"\0"
    out += pack_sequence(bases)
    out += bytes(quals) if (quals or not bases) else b"\xff" * len(bases)
    return out


def with_block_size(rec: bytes) -> bytes:             # builder.rs:224-230
    return struct.pack("<I", len(rec)) + bytes(rec)


# ---- the simplex caller -------------------------------------------------------------------------
@dataclass
class Stats:                                          # caller.rs:238-286
    total_reads: int = 0
    consensus_reads: int = 0
    filtered_reads: int = 0
    rejections: Dict[str, int] = field(default_factory=dict)

    def reject(self, reason: str, n: int):
        self.filtered_reads += n
        self.rejections[reason] = self.rejections.get(reason, 0) + n


class VanillaCallerOracle:
    """VanillaUmiConsensusCaller::consensus_reads, vanilla_caller.rs:1042-1499."""

    def __init__(self, prefix: str, rg: str, opt: VanillaOptions, vote_fn, builder_fn, track_rejects: bool = False):
        self.prefix, self.rg, self.opt = prefix, rg, opt
        self.stats = Stats()
        self.vote = vote_fn           # (rows, opt) -> (bases, quals, depths, errors)
        self.builder_call = builder_fn
        # vanilla_caller.rs:371-374: raw bytes of every rejected read, in the order the reject sites run.  (The one
        # site whose order the reference leaves open is the alignment filter's: it iterates a HashSet<usize>,
        # vanilla_caller.rs:964, 1193-1196; here -- and in the product -- ascending original index.)
        self.track_rejects = track_rejects
        self.rejected_reads: List[bytes] = []

    def consensus_reads(self, records: List[bytes]) -> Tuple[bytes, int]:
        if not records:
            return b"", 0
        recs = [Rec(b) for b in records]
        umi = recs[0].find_string(self.opt.tag)
        if umi is None:
            raise ValueError("Missing UMI tag")
        return self._process_group(umi.decode("utf-8", "replace"), recs)

    def _process_group(self, umi: str, recs: List[Rec]):
        st, opt = self.stats, self.opt
        st.total_reads += len(recs)
        reads = [r for r in recs if not (r.flags & SECONDARY) and not (r.flags & SUPPLEMENTARY)]
        if self.track_rejects:                           # filter_reads, :745-757
            self.rejected_reads += [r.b for r in recs if (r.flags & SECONDARY) or (r.flags & SUPPLEMENTARY)]
        if len(recs) - len(reads):
            st.reject("SecondaryOrSupplementary", len(recs) - len(reads))
        if not reads:
            return b"", 0
        if len(reads) < opt.min_reads:
            st.reject("InsufficientReads", len(reads))
            if self.track_rejects:                       # :1061-1063
                self.rejected_reads += [r.b for r in reads]
            return b"", 0
        frag = [r for r in reads if not r.flags & PAIRED]
        r1 = [r for r in reads if r.flags & PAIRED and r.flags & FIRST_SEGMENT]
        r2 = [r for r in reads if r.flags & PAIRED and not r.flags & FIRST_SEGMENT and r.flags & LAST_SEGMENT]
        out, count = bytearray(), 0
        ok, _, rec = self._subgroup(umi, "Fragment", frag)
        if ok:
            st.consensus_reads += 1
            out += rec
            count += 1
        ok1, n1, rec1 = self._subgroup(umi, "R1", r1)
        surv1 = self._last_surviving
        ok2, n2, rec2 = self._subgroup(umi, "R2", r2)
        surv2 = self._last_surviving
        if ok1 and ok2:
            st.consensus_reads += 2
            out += rec1 + rec2
            count += 2
        elif ok1:
            st.reject("OrphanConsensus", n1)
            if self.track_rejects:                       # :1095-1099
                self.rejected_reads += surv1
        elif ok2:
            st.reject("OrphanConsensus", n2)
            if self.track_rejects:                       # :1101-1105
                self.rejected_reads += surv2
        return bytes(out), count

    def _subgroup(self, umi: str, read_type: str, group: List[Rec]):
        st, opt = self.stats, self.opt
        track = self.track_rejects
        self._last_surviving: List[bytes] = []
        if not group:
            return False, 0, b""
        if len(group) < opt.min_reads:
            st.reject("InsufficientReads", len(group))
            if track:                                    # :1137-1142
                self.rejected_reads += [r.b for r in group]
            return False, 0, b""
        clips = [num_bases_extending_past_mate(r) for r in group]
        srs, zero = [], 0
        for i, (r, c) in enumerate(zip(group, clips)):
            sr = create_source_read(r, i, c, opt)
            if sr is None:
                zero += 1
                if track:                                # :1170-1174 (zero_length_indices, ascending)
                    self.rejected_reads.append(r.b)
            else:
                srs.append(sr)
        if zero:
            st.reject("ZeroLengthAfterTrimming", zero)
        if len(srs) < opt.min_reads:
            if srs:
                st.reject("InsufficientReads", len(srs))
                if track:                                # :1180-1184
                    self.rejected_reads += [group[s.original_idx].b for s in srs]
            return False, 0, b""
        before = [s.original_idx for s in srs]
        srs, n_rej = filter_by_alignment(srs)
        if n_rej:
            st.reject("MinorityAlignment", n_rej)
        if track:                                        # :1193-1197 (a HashSet in the reference: ascending here)
            kept_idx = {s.original_idx for s in srs}
            self.rejected_reads += [group[i].b for i in sorted(before) if i not in kept_idx]
        if len(srs) < opt.min_reads:
            if srs:
                st.reject("InsufficientReads", len(srs))
                if track:                                # :1205-1209
                    self.rejected_reads += [group[s.original_idx].b for s in srs]
            return False, 0, b""
        if track:                                        # :1216-1220 surviving_reads (what the orphan rule forwards)
            self._last_surviving = [group[s.original_idx].b for s in srs]
        bases, quals, depths, errors = self.vote([(bytes(s.bases), bytes(s.quals)) for s in srs], opt)
        raws = [group[s.original_idx] for s in srs]
        return True, len(srs), self._record(umi, read_type, raws, bases, quals, depths, errors)

    def _record(self, umi, read_type, raws, bases, quals, depths, errors) -> bytes:
        """build_consensus_record_into, vanilla_caller.rs:1365-1473"""
        opt = self.opt
        name = f"{self.prefix}:{umi}".encode()
        flag = UNMAPPED
        if read_type == "R1":
            flag |= PAIRED | FIRST_SEGMENT | MATE_UNMAPPED
        elif read_type == "R2":
            flag |= PAIRED | LAST_SEGMENT | MATE_UNMAPPED
        rec = unmapped_record(name, flag, bases, quals)
        rec += tag_string(b"RG", self.rg.encode())
        max_d = max(depths) if len(depths) else 0
        min_d = min(depths) if len(depths) else 0
        tot_e, tot_d = int(sum(int(e) for e in errors)), int(sum(int(d) for d in depths))
        # `total_errors as f32 / total_depth as f32`
        rate = (np.float32(tot_e) / np.float32(tot_d)) if tot_d > 0 else np.float32(0.0)
        rec += tag_int(b"cD", int(max_d)) + tag_int(b"cM", int(min_d)) + tag_float(b"cE", rate)
        if opt.produce_per_base_tags:
            rec += tag_i16_array(b"cd", [min(int(d), 32767) for d in depths])
            rec += tag_i16_array(b"ce", [min(int(e), 32767) for e in errors])
        rec += tag_string(b"MI", umi.encode())
        if opt.cell_tag is not None and raws:
            v = raws[0].find_string(opt.cell_tag)
            if v is not None:
                rec += tag_string(opt.cell_tag, v)
        umis = [r.find_string(b"RX") for r in raws]
        umis = [u.decode("utf-8", "replace") for u in umis if u is not None]
        if umis:
            rx = consensus_umis(umis, lambda pre, post, b, q: self.builder_call(pre, post, b, q)[:2])
            rec += tag_string(b"RX", rx.encode())
        return with_block_size(rec)


# =================================================================================================
# Duplex caller — crates/fgumi-consensus/src/duplex_caller.rs
# =================================================================================================
@dataclass
class SsCons:                                          # VanillaConsensusRead, vanilla_caller.rs:152-176
    bases: bytes
    quals: bytes
    depths: list
    errors: list
    source_rows: list                                  # [(bases, quals)] of the SourceReads used


@dataclass
class DuplexCons:                                      # DuplexConsensusRead
    bases: bytes
    quals: bytes
    errors: list
    ab: SsCons
    ba: Optional[SsCons]
    is_ba_only: bool = False


class DuplexCallerOracle:
    """DuplexConsensusCaller::consensus_reads, duplex_caller.rs:2206-2250 + process_group :1719-2202."""

    def __init__(self, prefix: str, rg: str, min_reads=(1, 1, 1), pre=45, post=40, min_input_q=10,
                 per_base=True, trim=False, cell_tag: Optional[bytes] = None, vote_fn=None,
                 builder_fn=None, duplex_job_fn=None):
        self.prefix, self.rg = prefix, rg
        self.min_total, self.min_xy, self.min_yx = min_reads
        self.per_base, self.cell_tag = per_base, cell_tag
        # ss_options, duplex_caller.rs:397-412: min_reads 1, min_consensus_base_quality MIN_PHRED
        self.ss_opt = VanillaOptions(error_rate_pre_umi=pre, error_rate_post_umi=post,
                                     min_input_base_quality=min_input_q, min_reads=1,
                                     produce_per_base_tags=per_base, trim=trim,
                                     min_consensus_base_quality=2, cell_tag=cell_tag)
        self.vote, self.builder_call, self.duplex_job = vote_fn, builder_fn, duplex_job_fn
        self.stats = Stats()

    # ---- consensus_reads :2206-2250 + partition_records_by_strand :576-630 ----
    def consensus_reads(self, records: List[bytes]) -> Tuple[bytes, int]:
        self.stats.total_reads += len(records)
        if not records:
            return b"", 0
        base_mi, a, b = self.partition_records_by_strand([Rec(b) for b in records])
        return self._process_group(base_mi, a, b)

    @staticmethod
    def partition_records_by_strand(recs):               # :576-630
        base_mi, a, b = None, [], []
        for r in recs:
            mi = r.find_string(b"MI")
            if mi is None:
                raise ValueError("missing MI tag")
            if base_mi is None:
                base_mi = (mi[:-2] if len(mi) >= 2 else mi).decode("utf-8", "replace")
            if len(mi) >= 2 and mi[-2:] == b"/A":
                a.append(r)
            elif len(mi) >= 2 and mi[-2:] == b"/B":
                b.append(r)
            else:
                raise ValueError("MI tag without /A or /B suffix")
        return base_mi, a, b

    @staticmethod
    def are_all_same_strand(rs) -> bool:                 # :771-780 (empty and single: true)
        return len({bool(r.flags & REVERSE) for r in rs}) <= 1

    @staticmethod
    def _r1(r):
        return bool(r.flags & PAIRED) and bool(r.flags & FIRST_SEGMENT)

    @staticmethod
    def _r2(r):
        return bool(r.flags & PAIRED) and bool(r.flags & LAST_SEGMENT)

    def _min_ok(self, na, nb):                         # :731-749 / :753-769
        xy, yx = (na, nb) if na >= nb else (nb, na)
        return self.min_total <= xy + yx and self.min_xy <= xy and self.min_yx <= yx

    def _consensus_call(self, srs: List[SourceRead]) -> Optional[SsCons]:   # vanilla_caller.rs:628-668
        if not srs or len(srs) < self.ss_opt.min_reads:
            return None
        rows = [(bytes(s.bases), bytes(s.quals)) for s in srs]
        b, q, d, e = self.vote(rows, self.ss_opt)
        return SsCons(b, q, d, e, rows)

    def _duplex_consensus(self, a: Optional[SsCons], b: Optional[SsCons], with_sources: bool):
        """duplex_consensus :838-1015 via the C++ oracle's arms."""
        if a is not None and b is not None:
            src = (a.source_rows + b.source_rows) if with_sources else []
            st, ob, oq, oe = self.duplex_job(a, b, src)
            if st == 0:
                n = len(ob)
                ab = SsCons(a.bases[:n], a.quals[:n], a.depths[:n], a.errors[:n], [])
                ba = SsCons(b.bases[:n], b.quals[:n], b.depths[:n], b.errors[:n], [])
                return DuplexCons(ob, oq, oe, ab, ba, False)
            if st == 1:
                return DuplexCons(a.bases, a.quals, list(a.errors), a, None, False)
            if st == 2:
                return DuplexCons(b.bases, b.quals, list(b.errors), b, None, True)
            return None
        one, ba_only = (a, False) if a is not None else (b, True)
        if one is None:
            return None
        # len = own length; the strand is kept only if it has depth somewhere (:852-853)
        if not any(d > 0 for d in one.depths):
            return None
        return DuplexCons(one.bases, one.quals, list(one.errors), one, None, ba_only)

    def _process_group(self, base_mi: str, a: List[Rec], b: List[Rec]):
        st = self.stats
        if not a and not b:
            return b"", 0
        na = sum(1 for r in a if self._r1(r))
        nb = sum(1 for r in b if self._r1(r))
        if not self._min_ok(na, nb):
            st.reject("InsufficientReads", len(a) + len(b))
            return b"", 0
        cell = None
        if self.cell_tag is not None:
            first = a[0] if a else (b[0] if b else None)
            if first is not None:
                v = first.find_string(self.cell_tag)
                cell = v if v is not None else None
        ab_r1 = [r for r in a if self._r1(r)]; ab_r2 = [r for r in a if self._r2(r)]
        ba_r1 = [r for r in b if self._r1(r)]; ba_r2 = [r for r in b if self._r2(r)]

        same_strand = self.are_all_same_strand
        if a and b:
            if not same_strand(ab_r1 + ba_r2) or not same_strand(ab_r2 + ba_r1):
                st.reject("PotentialCollision", len(a) + len(b))
                return b"", 0
        x_raws, y_raws = ab_r1 + ba_r2, ab_r2 + ba_r1

        def sources(raws):
            out = []
            for i, r in enumerate(raws):
                sr = create_source_read(r, i, num_bases_extending_past_mate(r), self.ss_opt)
                if sr is not None:
                    out.append(sr)
            return out
        fx, _ = filter_by_alignment(sources(x_raws))
        fy, _ = filter_by_alignment(sources(y_raws))
        f_ab_r1 = [s for s in fx if s.flags & FIRST_SEGMENT]
        f_ba_r2 = [s for s in fx if not s.flags & FIRST_SEGMENT]
        f_ab_r2 = [s for s in fy if not s.flags & FIRST_SEGMENT]
        f_ba_r1 = [s for s in fy if s.flags & FIRST_SEGMENT]
        raws_ab_r1 = [x_raws[s.original_idx] for s in f_ab_r1]
        raws_ba_r2 = [x_raws[s.original_idx] for s in f_ba_r2]
        raws_ab_r2 = [y_raws[s.original_idx] for s in f_ab_r2]
        raws_ba_r1 = [y_raws[s.original_idx] for s in f_ba_r1]
        c_ab_r1, c_ab_r2 = self._consensus_call(f_ab_r1), self._consensus_call(f_ab_r2)
        c_ba_r1, c_ba_r2 = self._consensus_call(f_ba_r1), self._consensus_call(f_ba_r2)
        out = bytearray()
        pattern = (c_ab_r1 is not None, c_ab_r2 is not None, c_ba_r1 is not None, c_ba_r2 is not None)
        if pattern == (True, True, True, True):
            d1 = self._duplex_consensus(c_ab_r1, c_ba_r2, True)       # :1999-2004
            d2 = self._duplex_consensus(c_ab_r2, c_ba_r1, True)       # :2008-2012
            if d1 is not None and d2 is not None:
                if self._cons_min_ok(d1) and self._cons_min_ok(d2):
                    out += self._record(d1, "R1", base_mi, raws_ab_r1, raws_ba_r2, True, cell)
                    out += self._record(d2, "R2", base_mi, raws_ab_r2, raws_ba_r1, False, cell)
                    st.consensus_reads += 1
                    return bytes(out), 2
                st.reject("InsufficientReads", len(a) + len(b))
                return b"", 0
        elif pattern == (True, True, False, False):
            if self.min_yx == 0:
                d1 = self._duplex_consensus(c_ab_r1, None, False)
                d2 = self._duplex_consensus(c_ab_r2, None, False)
                if d1 is not None and d2 is not None:
                    out += self._record(d1, "R1", base_mi, raws_ab_r1, [], True, cell)
                    out += self._record(d2, "R2", base_mi, raws_ab_r2, [], False, cell)
                    st.consensus_reads += 1
                    return bytes(out), 2
        elif pattern == (False, False, True, True):
            if self.min_yx == 0:
                d1 = self._duplex_consensus(None, c_ba_r2, False)
                d2 = self._duplex_consensus(None, c_ba_r1, False)
                if d1 is not None and d2 is not None:
                    out += self._record(d1, "R1", base_mi, [], raws_ba_r2, True, cell)
                    out += self._record(d2, "R2", base_mi, [], raws_ba_r1, False, cell)
                    st.consensus_reads += 1
                    return bytes(out), 2
        st.reject("InsufficientReads", len(a) + len(b))
        return b"", 0

    def _cons_min_ok(self, d: DuplexCons) -> bool:     # :753-769
        na = max(d.ab.depths) if len(d.ab.depths) else 0
        nb = (max(d.ba.depths) if len(d.ba.depths) else 0) if d.ba is not None else 0
        return self._min_ok(int(na), int(nb))

    def _record(self, d: DuplexCons, read_type, umi, raws_a, raws_b, first_of_pair, cell) -> bytes:
        """duplex_read_into :1048-1285 (methylation off)."""
        flag = UNMAPPED                                   # :1064-1076: a fragment carries no pair flags
        if read_type in ("R1", "R2"):
            flag |= PAIRED | MATE_UNMAPPED | (FIRST_SEGMENT if read_type == "R1" else LAST_SEGMENT)
        rec = unmapped_record(f"{self.prefix}:{umi}".encode(), flag, d.bases, d.quals)
        rec += tag_string(b"MI", umi.encode())
        if self.cell_tag is not None and cell is not None:
            rec += tag_string(self.cell_tag, cell)
        rec += tag_string(b"RG", self.rg.encode())

        def strand_metrics(s: Optional[SsCons]):
            if s is None:
                return 0, 0, np.float32(0.0)
            mx = int(max(s.depths)) if len(s.depths) else 0
            mn = int(min(s.depths)) if len(s.depths) else 0
            td, te = int(sum(int(x) for x in s.depths)), int(sum(int(x) for x in s.errors))
            return mx, mn, (np.float32(te) / np.float32(td)) if td > 0 else np.float32(0.0)
        amx, amn, aer = strand_metrics(d.ab)
        rec += tag_int(b"aD", amx) + tag_float(b"aE", aer) + tag_int(b"aM", amn)
        if self.per_base:
            rec += tag_string(b"ac", d.ab.bases)
            rec += tag_i16_array(b"ad", [min(int(x), 32767) for x in d.ab.depths])
            rec += tag_i16_array(b"ae", [min(int(x), 32767) for x in d.ab.errors])
            rec += tag_phred33(b"aq", d.ab.quals)
        bmx, bmn, ber = strand_metrics(d.ba)
        rec += tag_int(b"bD", bmx) + tag_float(b"bE", ber) + tag_int(b"bM", bmn)
        if self.per_base and d.ba is not None:
            rec += tag_string(b"bc", d.ba.bases)
            rec += tag_i16_array(b"bd", [min(int(x), 32767) for x in d.ba.depths])
            rec += tag_i16_array(b"be", [min(int(x), 32767) for x in d.ba.errors])
            rec += tag_phred33(b"bq", d.ba.quals)
        n = len(d.bases)
        comb = [(int(d.ab.depths[i]) if i < len(d.ab.depths) else 0) +
                (int(d.ba.depths[i]) if (d.ba is not None and i < len(d.ba.depths)) else 0) for i in range(n)]
        cmx, cmn = (max(comb) if comb else 0), (min(comb) if comb else 0)
        td, te = sum(comb), int(sum(int(x) for x in d.errors))
        cer = (np.float32(te) / np.float32(td)) if td > 0 else np.float32(0.0)
        rec += tag_int(b"cD", cmx) + tag_float(b"cE", cer) + tag_int(b"cM", cmn)
        umis = []
        for r in list(raws_a) + list(raws_b):
            rx = r.find_string(b"RX")
            if rx is None:
                continue
            s = rx.decode("utf-8", "replace")
            if bool(r.flags & FIRST_SEGMENT) == first_of_pair:
                umis.append(s)
            else:
                umis.append("-".join(reversed(s.split("-"))))
        if umis:
            rx = consensus_umis(umis, lambda pre, post, b, q: self.builder_call(pre, post, b, q)[:2])
            rec += tag_string(b"RX", rx.encode())
        return with_block_size(rec)


# =================================================================================================
# CODEC caller — crates/fgumi-consensus/src/codec_caller.rs
# =================================================================================================
def _enc(op_type: int, ln: int) -> int:
    return (ln << 4) | op_type


def _consumes_read(t: int) -> bool:                    # cigar.rs:75-77 (M, I, =, X)
    return t in (0, 1, 7, 8)


def _upgrade_clipping(ops, clip_amount, from_start):   # cigar.rs:579-655
    if from_start:
        hard = soft = skip = 0
        for op in ops:
            if op & 0xF == 5:
                hard += op >> 4; skip += 1
            else:
                break
        for op in ops[skip:]:
            if op & 0xF == 4:
                soft += op >> 4; skip += 1
            else:
                break
        up = min(soft, max(clip_amount - hard, 0))
        res = [_enc(5, hard + up)]
        if soft - up > 0:
            res.append(_enc(4, soft - up))
        return res + list(ops[skip:]), 0
    hard = soft = skip = 0
    for op in reversed(ops):
        if op & 0xF == 5:
            hard += op >> 4; skip += 1
        else:
            break
    end_idx = len(ops) - skip
    for op in reversed(ops[:end_idx]):
        if op & 0xF == 4:
            soft += op >> 4; skip += 1
        else:
            break
    up = min(soft, max(clip_amount - hard, 0))
    res = list(ops[:len(ops) - skip])
    if soft - up > 0:
        res.append(_enc(4, soft - up))
    res.append(_enc(5, hard + up))
    return res, 0


def _clip_start(ops, clip_amount):                     # cigar.rs:658-757
    hard = soft = skip = 0
    for op in ops:
        if op & 0xF == 5:
            hard += op >> 4; skip += 1
        else:
            break
    for op in ops[skip:]:
        if op & 0xF == 4:
            soft += op >> 4; skip += 1
        else:
            break
    post = list(ops[skip:])
    read_clipped = ref_clipped = 0
    new_ops, idx = [], 0
    while idx < len(post):
        op = post[idx]; t, ln = op & 0xF, op >> 4
        if read_clipped == clip_amount and not new_ops and t == 2:
            ref_clipped += ln; idx += 1
            continue
        if read_clipped >= clip_amount:
            break
        is_read, is_ref = _consumes_read(t), consumes_ref(t)
        if is_read and ln > clip_amount - read_clipped:
            if t == 1:
                read_clipped += ln
            else:
                rem_clip = clip_amount - read_clipped
                read_clipped += rem_clip
                if is_ref:
                    ref_clipped += rem_clip
                new_ops.append(_enc(t, ln - rem_clip))
        else:
            if is_read:
                read_clipped += ln
            if is_ref:
                ref_clipped += ln
        idx += 1
    new_ops += post[idx:]
    return [_enc(5, hard + soft + read_clipped)] + new_ops, ref_clipped


def _clip_end(ops, clip_amount):                       # cigar.rs:760-841
    hard = soft = skip = 0
    for op in reversed(ops):
        if op & 0xF == 5:
            hard += op >> 4; skip += 1
        else:
            break
    end_idx = len(ops) - skip
    for op in reversed(ops[:end_idx]):
        if op & 0xF == 4:
            soft += op >> 4; skip += 1
        else:
            break
    post = list(ops[:len(ops) - skip])
    read_clipped = 0
    new_ops, idx = [], len(post)
    while idx > 0:
        op = post[idx - 1]; t, ln = op & 0xF, op >> 4
        if read_clipped == clip_amount and not new_ops and t == 2:
            idx -= 1
            continue
        if read_clipped >= clip_amount:
            break
        is_read = _consumes_read(t)
        if is_read and ln > clip_amount - read_clipped:
            if t == 1:
                read_clipped += ln
            else:
                rem_clip = clip_amount - read_clipped
                read_clipped += rem_clip
                new_ops.append(_enc(t, ln - rem_clip))
        elif is_read:
            read_clipped += ln
        idx -= 1
    res = post[:idx] + list(reversed(new_ops))
    res.append(_enc(5, hard + soft + read_clipped))
    return res, 0


def clip_cigar_ops(ops, clip_amount, from_start):      # cigar.rs:355-397
    if clip_amount == 0 or not ops:
        return list(ops), 0
    seq = ops if from_start else list(reversed(ops))
    existing = 0
    for op in seq:
        if op & 0xF in (4, 5):
            existing += op >> 4
        else:
            break
    if clip_amount <= existing:
        return _upgrade_clipping(list(ops), clip_amount, from_start)
    extra = clip_amount - existing
    return _clip_start(list(ops), extra) if from_start else _clip_end(list(ops), extra)


def read_pos_at_ref_pos(ops, alignment_start, ref_pos, return_last_if_deleted):   # cigar.rs:412-457
    if ref_pos < alignment_start:
        return None
    ref_off = q_off = 0
    for op in ops:
        t, ln = op & 0xF, op >> 4
        op_ref_start = alignment_start + ref_off
        if consumes_ref(t):
            op_ref_end = op_ref_start + ln - 1
            if op_ref_start <= ref_pos <= op_ref_end:
                if consumes_query(t):
                    return q_off + (ref_pos - op_ref_start) + 1
                if return_last_if_deleted:
                    return q_off if q_off > 0 else 1
                return None
        if consumes_ref(t):
            ref_off += ln
        if consumes_query(t):
            q_off += ln
    return None


@dataclass
class ClippedInfo:                                     # codec_caller.rs ClippedRecordInfo
    raw_idx: int
    clip_amount: int
    clip_from_start: bool
    clipped_seq_len: int
    clipped_cigar: list
    adjusted_pos: int
    flags: int


class CodecCallerOracle:
    """CodecConsensusCaller::consensus_reads_raw, codec_caller.rs:531-814."""

    def __init__(self, prefix, rg, min_reads_per_strand=1, min_duplex_length=1, pre=45, post=40,
                 ss_qual=None, outer_qual=None, outer_len=5, max_dis=None, max_rate=1.0,
                 per_base=False, cell_tag=None, vote_fn=None, builder_fn=None, codec_job_fn=None):
        self.prefix, self.rg = prefix, rg
        self.min_reads, self.min_duplex_length = min_reads_per_strand, min_duplex_length
        self.ss_qual, self.outer_qual, self.outer_len = ss_qual, outer_qual, outer_len
        self.max_dis, self.max_rate = max_dis, max_rate
        self.per_base, self.cell_tag = per_base, cell_tag
        # ss_options :326-339: min_reads 1, min_consensus_base_quality 0, trim false
        self.ss_opt = VanillaOptions(error_rate_pre_umi=pre, error_rate_post_umi=post, min_reads=1,
                                     min_consensus_base_quality=0)
        self.vote, self.builder_call, self.codec_job = vote_fn, builder_fn, codec_job_fn
        self.total_input_reads = self.consensus_reads_generated = self.reads_filtered = 0
        self.duplex_bases = self.duplex_disagreements = 0
        self.rejections: Dict[str, int] = {}
        self.counter = 0

    def _reject(self, n, reason):
        self.rejections[reason] = self.rejections.get(reason, 0) + n
        self.reads_filtered += n

    @staticmethod
    def _clipped_info(r: Rec, idx: int, clip: int) -> ClippedInfo:     # :817-851
        from_start = bool(r.flags & REVERSE)
        cig, ref_consumed = clip_cigar_ops(r.cigar_ops(), clip, from_start)
        adj = (r.pos + 1) + (ref_consumed if from_start else 0)
        return ClippedInfo(idx, clip, from_start, max(r.l_seq - clip, 0), cig, adj, r.flags)

    def _filter(self, infos: List[ClippedInfo]) -> List[ClippedInfo]:  # :867-909
        if len(infos) < 2:
            return infos
        indexed = []
        for i, inf in enumerate(infos):
            c = simplify_cigar(inf.clipped_cigar)
            if inf.flags & REVERSE:
                c = list(reversed(c))
            indexed.append((i, inf.clipped_seq_len, c))
        indexed.sort(key=lambda t: -t[1])
        best = set(select_most_common_alignment_group(indexed))
        rej = len(infos) - len(best)
        if rej:
            self._reject(rej, "MinorityAlignment")
        return [inf for i, inf in enumerate(infos) if i in best]

    @staticmethod
    def check_overlap_phase(r1: ClippedInfo, r2: ClippedInfo, ov_start: int, ov_end: int) -> bool:   # :911-946
        a = read_pos_at_ref_pos(r1.clipped_cigar, r1.adjusted_pos, ov_start, True)
        b = read_pos_at_ref_pos(r2.clipped_cigar, r2.adjusted_pos, ov_start, True)
        c = read_pos_at_ref_pos(r1.clipped_cigar, r1.adjusted_pos, ov_end, True)
        d = read_pos_at_ref_pos(r2.clipped_cigar, r2.adjusted_pos, ov_end, True)
        return None not in (a, b, c, d) and (a - b) == (c - d)

    @staticmethod
    def compute_consensus_length(pos: ClippedInfo, neg: ClippedInfo, ov_end: int) -> Optional[int]:   # :949-968
        pp = read_pos_at_ref_pos(pos.clipped_cigar, pos.adjusted_pos, ov_end, False)
        nn = read_pos_at_ref_pos(neg.clipped_cigar, neg.adjusted_pos, ov_end, False)
        if pp is None or nn is None:
            return None
        return pp + neg.clipped_seq_len - nn

    @staticmethod
    def _source_row(r: Rec, inf: ClippedInfo):          # to_source_read_for_codec_raw :414-469
        bases, quals = r.sequence(), r.quals()
        clip = min(inf.clip_amount, len(bases))
        if clip > 0:
            if inf.clip_from_start:
                bases, quals = bases[clip:], quals[clip:]
            else:
                bases, quals = bases[:len(bases) - clip], quals[:len(quals) - clip]
        if r.flags & REVERSE:
            bases = reverse_complement(bases)
            quals = bytearray(reversed(quals))
        return bytes(bases), bytes(quals)

    def consensus_reads(self, records: List[bytes]) -> Tuple[bytes, int]:
        self.total_input_reads += len(records)
        if not records:
            return b"", 0
        recs = [Rec(b) for b in records]
        umi = recs[0].find_string(b"MI")
        umi = umi.decode("utf-8", "replace") if umi is not None else None
        paired, frag = [], 0
        for i, r in enumerate(recs):                    # phase 1 :545-561
            if not r.flags & PAIRED:
                frag += 1
                continue
            if r.flags & (SECONDARY | SUPPLEMENTARY | UNMAPPED):
                continue
            if not is_fr_pair(r):
                continue
            paired.append(i)
        if frag:
            self._reject(frag, "FragmentRead")
        if not paired:
            return b"", 0
        by_name: Dict[bytes, List[int]] = {}
        order = []
        for i in paired:                                # phase 2 :572-611
            nm = recs[i].name
            if nm not in by_name:
                order.append(nm)
            by_name.setdefault(nm, []).append(i)
        r1s, r2s = [], []
        for nm in order:
            idxs = by_name[nm]
            if len(idxs) != 2:
                continue
            i1, i2 = (idxs[0], idxs[1]) if recs[idxs[0]].flags & FIRST_SEGMENT else (idxs[1], idxs[0])
            r1s.append(self._clipped_info(recs[i1], i1, num_bases_extending_past_mate(recs[i1])))
            r2s.append(self._clipped_info(recs[i2], i2, num_bases_extending_past_mate(recs[i2])))
        if not r1s:
            return b"", 0
        if len(r1s) < self.min_reads:
            self._reject(len(r1s) + len(r2s), "InsufficientReads")
            return b"", 0
        r1s, r2s = self._filter(r1s), self._filter(r2s)   # phase 3
        if not r1s or not r2s:
            return b"", 0
        if len(r1s) < self.min_reads or len(r2s) < self.min_reads:
            self._reject(len(r1s) + len(r2s), "InsufficientReads")
            return b"", 0

        def longest(infos):                             # `.iter().rev().max_by_key(..)`: first max wins
            best = None
            for inf in infos:
                rl = reference_length(inf.clipped_cigar)
                if best is None or rl > best[0]:
                    best = (rl, inf)
            return best[1]
        l1, l2 = longest(r1s), longest(r2s)
        r1_neg = bool(l1.flags & REVERSE)
        lpos, lneg = (l2, l1) if r1_neg else (l1, l2)
        neg_start, pos_start = lneg.adjusted_pos, lpos.adjusted_pos
        pos_ref_len = reference_length(lpos.clipped_cigar)
        pos_end = pos_start + max(pos_ref_len - 1, 0)
        ov_start, ov_end = neg_start, pos_end
        if ov_end - ov_start + 1 < self.min_duplex_length:
            self._reject(len(r1s) + len(r2s), "InsufficientOverlap")
            return b"", 0
        if not self.check_overlap_phase(l1, l2, ov_start, ov_end):
            self._reject(len(r1s) + len(r2s), "IndelErrorBetweenStrands")
            return b"", 0
        r2_neg = bool(l2.flags & REVERSE)
        cons_len = self.compute_consensus_length(lpos, lneg, ov_end)
        if cons_len is None:
            self._reject(len(r1s) + len(r2s), "IndelErrorBetweenStrands")
            return b"", 0
        rows1 = [self._source_row(recs[i.raw_idx], i) for i in r1s]
        rows2 = [self._source_row(recs[i.raw_idx], i) for i in r2s]
        ss1 = self.vote(rows1, self.ss_opt)
        ss2 = self.vote(rows2, self.ss_opt)
        if cons_len < len(ss1[0]) or cons_len < len(ss2[0]):
            self._reject(len(r1s) + len(r2s), "IndelErrorBetweenStrands")
            return b"", 0
        res = self.codec_job(ss1, ss2, r1_neg, r2_neg, cons_len, self)
        self.duplex_bases += res["duplex_bases"] if res["duplex_bases"] > 0 else 0
        self.duplex_disagreements += res["disagreements"] if res["duplex_bases"] > 0 else 0
        if res["status"] != 0:
            return b"", 0                                 # bail!("High duplex disagreement..") -> dropped
        raws = [recs[i.raw_idx] for i in r1s] + [recs[i.raw_idx] for i in r2s]
        rec = self._record(res, umi, raws, recs)
        self.consensus_reads_generated += 1
        return rec, 1

    def _record(self, res, umi, source_raws, all_recs) -> bytes:          # :1226-1368
        self.counter += 1
        name = f"{self.prefix}:{umi}" if umi is not None else f"{self.prefix}:{self.counter}"
        cons, ac, bc = res["consensus"], res["ss_for_ac"], res["ss_for_bc"]
        rec = unmapped_record(name.encode(), UNMAPPED, cons[0], cons[1])
        rec += tag_string(b"RG", self.rg.encode())
        if umi is not None:
            rec += tag_string(b"MI", umi.encode())
        tot = [int(x) + int(y) for x, y in zip(ac[2], bc[2])]
        tmax, tmin = (max(tot) if tot else 0), (min(tot) if tot else 0)
        terr, tbases = int(sum(int(e) for e in cons[3])), sum(tot)
        rec += tag_int(b"cD", tmax) + tag_int(b"cM", tmin)
        rec += tag_float(b"cE", (np.float32(terr) / np.float32(tbases)) if tbases > 0 else np.float32(0))

        def strand(s):
            mx = max((int(d) for d in s[2]), default=0)
            mn = min((int(d) for d in s[2]), default=0)
            te, tb = sum(int(e) for e in s[3]), sum(int(d) for d in s[2])
            return mx, mn, (np.float32(te) / np.float32(tb)) if tb > 0 else np.float32(0)
        for pre, s in ((b"a", ac), (b"b", bc)):
            mx, mn, er = strand(s)
            rec += tag_int(pre + b"D", mx) + tag_int(pre + b"M", mn) + tag_float(pre + b"E", er)
        if self.per_base:
            wrap = lambda v: ((int(v) + 32768) % 65536) - 32768     # `d as i16`
            rec += tag_i16_array(b"ad", [wrap(d) for d in ac[2]]) + tag_i16_array(b"bd", [wrap(d) for d in bc[2]])
            rec += tag_i16_array(b"ae", [wrap(e) for e in ac[3]]) + tag_i16_array(b"be", [wrap(e) for e in bc[3]])
            rec += tag_string(b"ac", ac[0]) + tag_string(b"bc", bc[0])
            rec += tag_phred33(b"aq", ac[1]) + tag_phred33(b"bq", bc[1])
        if self.cell_tag is not None:
            for r in source_raws:
                v = r.find_string(self.cell_tag)
                if v is not None and len(v) > 0:
                    rec += tag_string(self.cell_tag, v)
                    break
        umis = []
        for r in all_recs:
            v = r.find_string(b"RX")
            if v is None:
                continue
            try:
                umis.append(v.decode("utf-8"))
            except UnicodeDecodeError:
                pass
        if umis:
            rx = consensus_umis(umis, lambda pre, post, b, q: self.builder_call(pre, post, b, q)[:2])
            if rx:
                rec += tag_string(b"RX", rx.encode())
        return with_block_size(rec)


def _rc_ss(s):                                         # reverse_complement_ss, codec_caller.rs:507-520
    return (bytes(reverse_complement(s[0])), bytes(reversed(s[1])), list(reversed(s[2])), list(reversed(s[3])))


def _pad_ss(s, new_len, left):                         # pad_consensus, codec_caller.rs:980-1023
    cur = len(s[0])
    if new_len <= cur:
        return s
    n = new_len - cur
    pb, pq, pd, pe = b"n" * n, bytes(n), [0] * n, [0] * n
    if left:
        return (pb + s[0], pq + s[1], pd + list(s[2]), pe + list(s[3]))
    return (s[0] + pb, s[1] + pq, list(s[2]) + pd, list(s[3]) + pe)


def codec_strands(ss1, ss2, r1_neg, r2_neg, cons_len):
    """codec_caller.rs:746-766: oriented+padded single strands and the ac/bc views of them."""
    ss1 = (bytes(ss1[0]), bytes(ss1[1]), list(ss1[2]), list(ss1[3]))
    ss2 = (bytes(ss2[0]), bytes(ss2[1]), list(ss2[2]), list(ss2[3]))
    o1, o2 = (_rc_ss(ss1), ss2) if r1_neg else (ss1, _rc_ss(ss2))
    p1, p2 = _pad_ss(o1, cons_len, r1_neg), _pad_ss(o2, cons_len, r2_neg)
    ac, bc = (_rc_ss(p1), _rc_ss(p2)) if r1_neg else (p1, p2)
    return p1, p2, ac, bc


# =================================================================================================
# Overlapping-bases pre-pass (crates/fgumi-consensus/src/overlapping.rs)
# =================================================================================================
AGREE_CONSENSUS, AGREE_MAX_QUAL, AGREE_PASS_THROUGH = 0, 1, 2          # AgreementStrategy :20-28
DISAGREE_CONSENSUS, DISAGREE_MASK_BOTH, DISAGREE_MASK_LOWER = 0, 1, 2  # DisagreementStrategy :31-39


class _ReadAndRefPosIterator:
    """ReadAndRefPosIterator, overlapping.rs:382-553 (1-based read and reference positions)."""

    def __init__(self, rec: Rec, rec_start, rec_end, mate_start, mate_end):    # :411-449
        self.ops = [(op & 0xF, op >> 4) for op in rec.cigar_ops()]
        min_ref, max_ref = max(rec_start, mate_start), min(rec_end, mate_end)
        self.start_read_pos, self.end_read_pos = 1, rec.l_seq
        self.start_ref_pos, self.end_ref_pos = max(rec_start, min_ref), min(rec_end, max_ref)
        self.cur_read_pos, self.cur_ref_pos = 1, rec_start
        self.element_index = self.in_elem_offset = 0
        self._skip_to_start()

    def _on_target(self):                                                # :452-460
        if self.element_index >= len(self.ops):
            return 0
        k, n = self.ops[self.element_index]
        return n if k in (0, 2, 3, 7, 8) else 0

    def _on_query(self):                                                 # :463-471
        if self.element_index >= len(self.ops):
            return 0
        k, n = self.ops[self.element_index]
        return n if k in (0, 1, 4, 7, 8) else 0

    def _is_alignment(self):                                             # :474-481
        return self.element_index < len(self.ops) and self.ops[self.element_index][0] in (0, 7, 8)

    def _skip_to_start(self):                                            # :484-499
        while self.element_index < len(self.ops):
            ref_end = self.cur_ref_pos + self._on_target() - 1
            read_end = self.cur_read_pos + self._on_query() - 1
            if ref_end >= self.start_ref_pos and read_end >= self.start_read_pos:
                break
            self.cur_ref_pos += self._on_target()
            self.cur_read_pos += self._on_query()
            self.element_index += 1
        self._skip_non_aligned()

    def _skip_non_aligned(self):                                         # :502-521
        self.in_elem_offset = 0
        while self.element_index < len(self.ops) and not self._is_alignment():
            self.cur_ref_pos += self._on_target()
            self.cur_read_pos += self._on_query()
            self.element_index += 1
        if self.element_index < len(self.ops) and (self.cur_ref_pos < self.start_ref_pos or
                                                   self.cur_read_pos < self.start_read_pos):
            off = max(self.start_ref_pos - self.cur_ref_pos, self.start_read_pos - self.cur_read_pos)
            self.in_elem_offset = off
            self.cur_ref_pos += off
            self.cur_read_pos += off

    def next(self):                                                      # :531-559
        if self.element_index < len(self.ops):
            if self.in_elem_offset >= self.ops[self.element_index][1]:
                self.element_index += 1
                self._skip_non_aligned()
        if (self.element_index >= len(self.ops) or self.cur_read_pos > self.end_read_pos or
                self.cur_ref_pos > self.end_ref_pos):
            return None
        pos = (self.cur_read_pos - 1, self.cur_ref_pos)
        self.cur_read_pos += 1
        self.cur_ref_pos += 1
        self.in_elem_offset += 1
        return pos


def _set_base(rec: bytearray, seq_off: int, i: int, base: int):          # sequence.rs:53-61
    code = b"=ACMGRSVTWYHKDBN".find(bytes([base]))
    code = 15 if code < 0 else code
    j = seq_off + i // 2
    rec[j] = ((code << 4) | (rec[j] & 0x0F)) if i % 2 == 0 else ((rec[j] & 0xF0) | code)


class OverlappingOracle:
    """OverlappingBasesConsensusCaller (overlapping.rs:79-337) + apply_overlapping_consensus (:625)."""

    def __init__(self, agreement=AGREE_CONSENSUS, disagreement=DISAGREE_CONSENSUS):
        self.agreement, self.disagreement = agreement, disagreement
        self.overlapping_bases = self.bases_agreeing = self.bases_disagreeing = self.bases_corrected = 0

    def stats(self):
        return (self.overlapping_bases, self.bases_agreeing, self.bases_disagreeing, self.bases_corrected)

    def call(self, r1: bytearray, r2: bytearray) -> bool:                # :236-337
        v1, v2 = Rec(bytes(r1)), Rec(bytes(r2))
        if (v1.flags & UNMAPPED) or (v2.flags & UNMAPPED) or v1.ref_id != v2.ref_id:
            return False

        def span(v):                                                     # cigar.rs:314-335
            if v.pos < 0:
                return None
            rl = reference_length(v.cigar_ops())
            return (v.pos + 1, v.pos + rl) if rl != 0 else None
        s1, s2 = span(v1), span(v2)
        if s1 is None or s2 is None:
            return False
        it1 = _ReadAndRefPosIterator(v1, s1[0], s1[1], s2[0], s2[1])
        it2 = _ReadAndRefPosIterator(v2, s2[0], s2[1], s1[0], s1[1])
        pairs = []                                                       # merge walk :586-617
        a, b = it1.next(), it2.next()
        while a is not None and b is not None:
            if a[1] < b[1]:
                a = it1.next()
            elif a[1] > b[1]:
                b = it2.next()
            else:
                pairs.append((a[0], b[0]))
                a, b = it1.next(), it2.next()
        if not pairs:
            return False
        seq1, seq2 = v1.sequence(), v2.sequence()
        q1, q2 = v1.quals(), v2.quals()
        modified = False
        nocall = (ord("N"), ord("n"), ord("."))
        for o1, o2 in pairs:
            b1, b2 = seq1[o1], seq2[o2]
            if b1 in nocall or b2 in nocall:
                continue
            self.overlapping_bases += 1
            x, y = q1[o1], q2[o2]
            if b1 == b2:
                self.bases_agreeing += 1
                if self.agreement == AGREE_PASS_THROUGH:
                    continue
                nq = min(x + y, 93) if self.agreement == AGREE_CONSENSUS else max(x, y)
                q1[o1] = q2[o2] = nq
                if nq != x or nq != y:
                    self.bases_corrected += 1
                    modified = True
            else:
                self.bases_disagreeing += 1
                modified = True
                if self.disagreement == DISAGREE_CONSENSUS:
                    if x == y:
                        cb, cq = ord("N"), 2
                    elif x > y:
                        cb, cq = b1, max(x - y, 2)
                    else:
                        cb, cq = b2, max(y - x, 2)
                    seq1[o1] = seq2[o2] = cb
                    q1[o1] = q2[o2] = cq
                    self.bases_corrected += 2
                elif self.disagreement == DISAGREE_MASK_BOTH or x == y:
                    seq1[o1] = seq2[o2] = ord("N")
                    q1[o1] = q2[o2] = 2
                    self.bases_corrected += 2
                elif x < y:
                    seq1[o1], q1[o1] = ord("N"), 2
                    self.bases_corrected += 1
                else:
                    seq2[o2], q2[o2] = ord("N"), 2
                    self.bases_corrected += 1
        if modified:
            for rec, v, seq, q in ((r1, v1, seq1, q1), (r2, v2, seq2, q2)):
                so = v.seq_offset()
                for i, base in enumerate(seq):
                    _set_base(rec, so, i, base)
                qo = so + (v.l_seq + 1) // 2
                rec[qo:qo + len(q)] = q
        return True

    def apply(self, records: List[bytearray]):                           # :625-667
        pairs: Dict[bytes, List[Optional[int]]] = {}
        for idx, raw in enumerate(records):
            v = Rec(bytes(raw))
            if v.flags & (SECONDARY | SUPPLEMENTARY):
                continue
            if v.flags & FIRST_SEGMENT:
                pairs.setdefault(v.name, [None, None])[0] = idx
            elif v.flags & LAST_SEGMENT:
                pairs.setdefault(v.name, [None, None])[1] = idx
        for i1, i2 in pairs.values():
            if i1 is not None and i2 is not None:
                self.call(records[i1], records[i2])


# =================================================================================================
# Consensus filter (crates/fgumi-consensus/src/filter.rs + src/lib/commands/filter.rs), simplex reads
# =================================================================================================
def _aux_tags(aux: bytes):
    """Walk BAM aux data -> {tag: (type, value)}; B arrays -> (subtype, [values])."""
    out, p = {}, 0
    fixed = {"A": ("<c", 1), "c": ("<b", 1), "C": ("<B", 1), "s": ("<h", 2), "S": ("<H", 2),
             "i": ("<i", 4), "I": ("<I", 4), "f": ("<f", 4)}
    while p + 3 <= len(aux):
        tag, vt = bytes(aux[p:p + 2]), chr(aux[p + 2])
        p += 3
        if vt in fixed:
            fmt, n = fixed[vt]
            out[tag] = (vt, struct.unpack_from(fmt, aux, p)[0])
            p += n
        elif vt in "ZH":
            e = aux.index(b"\0", p)
            out[tag] = (vt, bytes(aux[p:e]))
            p = e + 1
        elif vt == "B":
            st = chr(aux[p])
            (cnt,) = struct.unpack_from("<I", aux, p + 1)
            fmt, n = fixed[st]
            out[tag] = ("B" + st, list(struct.unpack_from("<%d%s" % (cnt, fmt[1]), aux, p + 5)))
            p += 5 + cnt * n
        else:
            break
    return out


@dataclass
class FilterThresholds:                                  # filter.rs:31-40
    min_reads: int = 1
    max_read_error_rate: float = 1.0
    max_base_error_rate: float = 1.0


FILTER_PASS, FILTER_INSUFFICIENT_READS, FILTER_EXCESSIVE_ERROR_RATE = 0, 1, 2


def filter_read(aux: bytes, th: FilterThresholds) -> int:          # filter.rs:453-471
    tags = _aux_tags(aux)
    cd = tags.get(b"cD")
    if cd is not None and cd[0] in "cCsSiI" and cd[1] < th.min_reads:
        return FILTER_INSUFFICIENT_READS
    ce = tags.get(b"cE")
    if ce is not None and ce[0] == "f" and float(np.float32(ce[1])) > th.max_read_error_rate:
        return FILTER_EXCESSIVE_ERROR_RATE
    return FILTER_PASS


def compute_read_stats(rec: bytes) -> Tuple[int, float]:            # filter.rs:565-590
    r = Rec(bytes(rec))
    seq, q = r.sequence(), r.quals()
    n_count = sum(1 for b in seq if b == ord("N"))
    qs = sum(int(x) for b, x in zip(seq, q) if b != ord("N"))
    non_n = len(seq) - n_count
    return n_count, (qs / non_n if non_n else 0.0)


def _array_u16(v):
    """array_tag_to_vec_u16 / array_tag_element_u16, raw-bam tags.rs:479-506: unsigned 8/16-bit elements
    as they are, signed ones clamped at 0, every other element type reads as 0."""
    if v is None or not v[0].startswith("B"):
        return None
    st = v[0][1]
    if st in "CS":
        return [int(x) for x in v[1]]
    if st in "cs":
        return [max(int(x), 0) for x in v[1]]
    return [0] * len(v[1])


def mask_bases(rec: bytearray, th: FilterThresholds, min_base_quality: Optional[int]) -> int:   # filter.rs:655-696
    r = Rec(bytes(rec))
    tags = _aux_tags(r.aux())
    cd = tags.get(b"cd")
    ce = tags.get(b"ce")
    cdv, cev = _array_u16(cd), _array_u16(ce)
    so = r.seq_offset()
    qo = so + (r.l_seq + 1) // 2
    seq = r.sequence()
    masked = 0
    for i in range(r.l_seq):
        depth = cdv[i] if cdv is not None and i < len(cdv) else 0
        errors = cev[i] if cev is not None and i < len(cev) else 0
        qual = rec[qo + i]
        should = ((min_base_quality is not None and qual < min_base_quality) or depth < th.min_reads or
                  (depth > 0 and (float(errors) / float(depth)) > th.max_base_error_rate))
        if should:
            if seq[i] != ord("N"):
                masked += 1
            _set_base(rec, so, i, ord("N"))                 # mask_base: nibble 15
            rec[qo + i] = 2
    return masked


def check_no_call_and_quality(rec: bytes, min_mean_qual: Optional[float], max_no_call_frac: float) -> bool:
    """commands/filter.rs:909-929"""
    no_calls, mean_q = compute_read_stats(rec)
    if min_mean_qual is not None and mean_q < min_mean_qual:
        return False
    n = Rec(bytes(rec)).l_seq
    if max_no_call_frac >= 1.0:
        return float(no_calls) <= max_no_call_frac
    frac = no_calls / n if n > 0 else 0.0
    return frac <= max_no_call_frac


class SimplexFilterOracle:
    """`fgumi filter` on single-strand consensus records, template mode
    (commands/filter.rs:614-697, 738-905): mask bases, then read-level checks; a template (records
    sharing a name, consecutive) is kept only if all of its primary records pass."""

    def __init__(self, th: FilterThresholds, min_base_quality: Optional[int] = None,
                 min_mean_base_quality: Optional[float] = None, max_no_call_fraction: float = 0.2):
        self.th, self.min_bq = th, min_base_quality
        self.min_mean, self.max_nc = min_mean_base_quality, max_no_call_fraction
        self.total = self.passed = self.bases_masked = 0

    def process_record(self, rec: bytearray) -> bool:
        self.bases_masked += mask_bases(rec, self.th, self.min_bq)
        if filter_read(Rec(bytes(rec)).aux(), self.th) != FILTER_PASS:
            return False
        return check_no_call_and_quality(bytes(rec), self.min_mean, self.max_nc)

    def filter_stream(self, data: bytes) -> Tuple[bytes, int]:
        recs, p = [], 0
        while p < len(data):
            (n,) = struct.unpack_from("<I", data, p)
            recs.append(bytearray(data[p + 4:p + 4 + n]))
            p += 4 + n
        out, kept, i = bytearray(), 0, 0
        while i < len(recs):
            j = i
            name = Rec(bytes(recs[i])).name
            while j < len(recs) and Rec(bytes(recs[j])).name == name:
                j += 1
            passes = []
            for k in range(i, j):
                self.total += 1
                passes.append(self.process_record(recs[k]))
            if all(passes):                                  # all records here are primary
                for k in range(i, j):
                    out += with_block_size(bytes(recs[k]))
                    kept += 1
                    self.passed += 1
            i = j
        return bytes(out), kept


# ---- duplex consensus reads (filter.rs:443-447, 477-557, 621-639, 702-806) ----------------------
def is_duplex_consensus(aux: bytes) -> bool:                        # filter.rs:443-446
    tags = _aux_tags(aux)
    return b"aD" in tags or b"bD" in tags


def _find_int(tags, tag):                                           # bam_fields::find_int_tag: any integer type
    v = tags.get(tag)
    return int(v[1]) if v is not None and v[0] in "cCsSiI" else None


def _find_float(tags, tag):                                         # bam_fields::find_float_tag: 'f' only
    v = tags.get(tag)
    return float(np.float32(v[1])) if v is not None and v[0] == "f" else None


def filter_duplex_read(aux: bytes, cc: FilterThresholds, ab: FilterThresholds, ba: FilterThresholds) -> int:
    """filter.rs:477-557.  `ab` is the stricter tier (checked against the better strand of each
    metric), `ba` the lenient one (checked against the worse strand)."""
    r = filter_read(aux, cc)
    if r != FILTER_PASS:
        return r
    tags = _aux_tags(aux)
    a_d = _find_int(tags, b"aD")
    a_d = a_d if a_d is not None else _find_int(tags, b"aM")
    b_d = _find_int(tags, b"bD")
    b_d = b_d if b_d is not None else _find_int(tags, b"bM")
    a_e, b_e = _find_float(tags, b"aE"), _find_float(tags, b"bE")
    if a_d is not None and b_d is not None:
        worst_d, best_d = (a_d, b_d) if a_d < b_d else (b_d, a_d)
    elif a_d is not None:
        worst_d, best_d = 0, a_d
    elif b_d is not None:
        worst_d, best_d = 0, b_d
    else:
        return FILTER_PASS
    if a_e is not None and b_e is not None:
        best_e, worst_e = (a_e, b_e) if a_e < b_e else (b_e, a_e)
    elif a_e is not None:
        best_e = worst_e = a_e
    elif b_e is not None:
        best_e = worst_e = b_e
    else:
        best_e = worst_e = 0.0
    U64 = (1 << 64) - 1                       # `(depth as usize) < min_reads`: a negative tag value wraps
    if (best_d & U64) < ab.min_reads:
        return FILTER_INSUFFICIENT_READS
    if best_e > ab.max_read_error_rate:
        return FILTER_EXCESSIVE_ERROR_RATE
    if (worst_d & U64) < ba.min_reads:
        return FILTER_INSUFFICIENT_READS
    if worst_e > ba.max_read_error_rate:
        return FILTER_EXCESSIVE_ERROR_RATE
    return FILTER_PASS


def _string_or_u8_array(tags, tag):                                 # filter.rs:621-639
    v = tags.get(tag)
    if v is None:
        return None
    if v[0] == "Z":
        return bytes(v[1])
    if v[0] in ("BC", "Bc"):
        return bytes(x & 0xFF for x in v[1])
    return None


def mask_duplex_bases(rec: bytearray, cc: FilterThresholds, ab: FilterThresholds, ba: FilterThresholds,
                      min_base_quality: Optional[int], require_ss_agreement: bool) -> int:   # filter.rs:702-806
    r = Rec(bytes(rec))
    tags = _aux_tags(r.aux())

    ad, ae, bd, be = (_array_u16(tags.get(t)) for t in (b"ad", b"ae", b"bd", b"be"))
    ac = _string_or_u8_array(tags, b"ac") if require_ss_agreement else None
    bc = _string_or_u8_array(tags, b"bc") if require_ss_agreement else None
    so = r.seq_offset()
    qo = so + (r.l_seq + 1) // 2
    seq = r.sequence()
    get = lambda v, i: v[i] if v is not None and i < len(v) else 0
    masked = 0
    for i in range(r.l_seq):
        if seq[i] == ord("N"):                                      # is_base_n: already masked
            continue
        a_d, b_d, a_e, b_e = get(ad, i), get(bd, i), get(ae, i), get(be, i)
        best_d, worst_d = max(a_d, b_d), min(a_d, b_d)
        a_r = float(a_e) / float(a_d) if a_d > 0 else 0.0
        b_r = float(b_e) / float(b_d) if b_d > 0 else 0.0
        best_r, worst_r = min(a_r, b_r), max(a_r, b_r)
        tot_d = a_d + b_d
        tot_r = float(a_e + b_e) / float(tot_d) if tot_d > 0 else 0.0
        qual = rec[qo + i]
        should = ((min_base_quality is not None and qual < min_base_quality) or
                  tot_d < cc.min_reads or tot_r > cc.max_base_error_rate or
                  best_d < ab.min_reads or best_r > ab.max_base_error_rate or
                  worst_d < ba.min_reads or worst_r > ba.max_base_error_rate)
        ss_dis = False
        if require_ss_agreement and a_d > 0 and b_d > 0:
            ab_b = ac[i] if ac is not None and i < len(ac) else ord("N")
            bb_b = bc[i] if bc is not None and i < len(bc) else ord("N")
            ss_dis = ab_b != bb_b
        if should or ss_dis:
            masked += 1
            _set_base(rec, so, i, ord("N"))
            rec[qo + i] = 2
    return masked


class DuplexFilterOracle(SimplexFilterOracle):
    """`fgumi filter` on duplex consensus records (commands/filter.rs:770-793, 949-968): duplex
    masking with the CC / AB / BA tiers, then the duplex read-level gates and the shared mean-quality
    and no-call checks.  Records without aD/bD tags take the single-strand path with the CC tier
    (`effective_single_strand_thresholds`, filter.rs:217-219)."""

    def __init__(self, cc: FilterThresholds, ab: FilterThresholds, ba: FilterThresholds,
                 min_base_quality: Optional[int] = None, min_mean_base_quality: Optional[float] = None,
                 max_no_call_fraction: float = 0.2, require_ss_agreement: bool = False):
        super().__init__(cc, min_base_quality, min_mean_base_quality, max_no_call_fraction)
        self.ab, self.ba, self.ss_agree = ab, ba, require_ss_agreement

    def process_record(self, rec: bytearray) -> bool:
        if not is_duplex_consensus(Rec(bytes(rec)).aux()):
            return super().process_record(rec)
        self.bases_masked += mask_duplex_bases(rec, self.th, self.ab, self.ba, self.min_bq, self.ss_agree)
        if filter_duplex_read(Rec(bytes(rec)).aux(), self.th, self.ab, self.ba) != FILTER_PASS:
            return False
        return check_no_call_and_quality(bytes(rec), self.min_mean, self.max_nc)


# =================================================================================================
# MI grouping of the input stream -- src/lib/mi_group.rs:386-470 (MiGroupIterator), fgumi-umi lib.rs:355-363
# =================================================================================================
def extract_mi_base(mi: str) -> str:
    return mi[:-2] if mi.endswith("/A") or mi.endswith("/B") else mi


def mi_groups(records: List[bytes], tag: bytes = b"MI", strip_strand_suffix: bool = False,
              cell_tag: Optional[bytes] = None) -> List[Tuple[str, List[int]]]:
    """[(key, indices of the group's records)]; records without the tag are skipped."""
    out: List[Tuple[str, List[int]]] = []
    for i, b in enumerate(records):
        r = Rec(b)
        v = r.find_string(tag)
        if v is None:
            continue
        key = v.decode("utf-8", "replace")
        if strip_strand_suffix:
            key = extract_mi_base(key)
        if cell_tag is not None:
            cv = r.find_string(cell_tag)
            key += "\t" + (cv.decode("utf-8", "replace") if cv is not None else "")
        if out and out[-1][0] == key:
            out[-1][1].append(i)
        else:
            out.append((key, [i]))
    return out
