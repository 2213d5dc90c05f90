"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Restatement (pure Python) of `fgumi filter [--ref]` on raw records without its methylation branches, record bytes in,
kept / rejected record bytes out, in the single-threaded order of the reference.  Masks and gates come from
oracle/record_oracle.py, template order from tests/dedup_oracle.py.  Citations are relative to the fgumi source tree:
  filter.rs          src/lib/commands/filter.rs                    (process_record_raw, template / single-read modes)
  alignment_tags.rs  crates/fgumi-sam/src/alignment_tags.rs        (regenerate_alignment_tags_raw)
  tags.rs            crates/fgumi-raw-bam/src/tags.rs              (update_int_tag, update_string_tag, remove_tag)
  tag_reversal.rs    src/lib/tag_reversal.rs                       (reverse_per_base_tags_raw)
  reference.rs       src/lib/reference.rs                          (the sequential FASTA reader, fetch_slice)
"""
from __future__ import annotations

import os
import struct
import sys
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import record_oracle as R   # noqa: E402
from tests import dedup_oracle as D     # noqa: E402

CODES = b"=ACMGRSVTWYHKDBN"
FIXED = {ord("A"): 1, ord("c"): 1, ord("C"): 1, ord("s"): 2, ord("S"): 2, ord("i"): 4, ord("I"): 4, ord("f"): 4}


class FilterError(ValueError):
    """Where the reference fails the command: the product fails the call; `record` is the input index."""

    def __init__(self, msg: str, record: int):
        super().__init__(msg)
        self.record = record


# ---- the reference ----------------------------------------------------------------------------------------------
def parse_fasta(data: bytes) -> Dict[bytes, bytes]:
    """new_sequential (reference.rs:229-244): name up to the first space / tab after '>', sequence = the following
    lines with their \\n / \\r\\n removed, bytes as they are; a later contig of the same name replaces an earlier."""
    if data[:2] == b"\x1f\x8b":
        raise ValueError("compressed FASTA")
    out, name, seq = {}, None, []
    for ln in data.split(b"\n"):
        if ln.endswith(b"\r"):
            ln = ln[:-1]
        if not ln:
            continue
        if ln.startswith(b">"):
            if name is not None:
                out[name] = b"".join(seq)
            body = ln[1:]
            cut = min([i for i in (body.find(b" "), body.find(b"\t")) if i >= 0], default=len(body))
            name, seq = body[:cut], []
        else:
            if name is None:
                raise ValueError("text before the first '>'")
            seq.append(ln)
    if name is not None:
        out[name] = b"".join(seq)
    return out


def sq_names(header_text: bytes) -> List[bytes]:
    out = []
    for ln in header_text.split(b"\n"):
        if ln.startswith(b"@SQ\t"):
            f = dict(x.split(b":", 1) for x in ln.split(b"\t")[1:] if b":" in x)
            out.append(f.get(b"SN", b"").rstrip(b"\r"))
    return out


# ---- raw tag editing (tags.rs) --------------------------------------------------------------------------------------
def aux_offset(r: bytes) -> int:
    l_rn, nc, ls = r[8], struct.unpack_from("<H", r, 12)[0], struct.unpack_from("<I", r, 16)[0]
    return 32 + l_rn + 4 * nc + (ls + 1) // 2 + ls


def value_size(vt: int, d: bytes) -> Optional[int]:        # tag_value_size (fields.rs:289-310)
    if vt in FIXED:
        return FIXED[vt] if len(d) >= FIXED[vt] else None
    if vt in (ord("Z"), ord("H")):
        e = d.find(b"\0")
        return None if e < 0 else e + 1
    if vt == ord("B"):
        if len(d) < 5 or d[0] not in FIXED:
            return None
        return 5 + struct.unpack_from("<I", d, 1)[0] * FIXED[d[0]]
    return None


def find_tag(r: bytes, tag: bytes) -> Optional[Tuple[int, int, int]]:
    """find_tag_position + find_tag_bounds: (start, end, type) of the first entry, absolute offsets; None when absent
    or its value is cut short."""
    a = aux_offset(r)
    p = a
    while p + 3 <= len(r):
        vt = r[p + 2]
        size = value_size(vt, r[p + 3:])
        if r[p:p + 2] == tag:
            return None if size is None else (p, p + 3 + size, vt)
        if size is None:
            return None
        p += 3 + size
    return None


def append_int(tag: bytes, v: int) -> bytes:              # append_int_tag (tags.rs:533-553)
    if -128 <= v <= 127:
        return tag + b"c" + struct.pack("<b", v)
    if 0 <= v <= 255:
        return tag + b"C" + struct.pack("<B", v)
    if 0 <= v <= 65535:
        return tag + b"S" + struct.pack("<H", v)
    if -32768 <= v < 0:
        return tag + b"s" + struct.pack("<h", v)
    return tag + b"i" + struct.pack("<i", v)


def update_int(r: bytearray, tag: bytes, v: int) -> None:   # update_int_tag (tags.rs:729-750)
    f = find_tag(bytes(r), tag)
    if f is not None:
        s, e, vt = f
        if vt in (ord("i"), ord("I")) and e - s == 7:
            r[s + 3:s + 7] = struct.pack("<i", v)
            return
        del r[s:e]
    r += append_int(tag, v)


def update_string(r: bytearray, tag: bytes, v: bytes) -> None:   # update_string_tag (tags.rs:694-721)
    f = find_tag(bytes(r), tag)
    if f is not None:
        s, e, _ = f
        if e - s - 4 == len(v):
            r[s + 3:s + 3 + len(v)] = v
        else:
            r[s:e] = tag + b"Z" + v + b"\0"
        return
    r += tag + b"Z" + v + b"\0"


def remove_tag(r: bytearray, tag: bytes) -> None:           # remove_tag (tags.rs:670-683)
    f = find_tag(bytes(r), tag)
    if f is not None:
        del r[f[0]:f[1]]


# ---- reverse_per_base_tags_raw (tag_reversal.rs) -------------------------------------------------------------------
COMP = {ord("A"): ord("T"), ord("a"): ord("T"), ord("T"): ord("A"), ord("t"): ord("A"), ord("C"): ord("G"),
        ord("c"): ord("G"), ord("G"): ord("C"), ord("g"): ord("C")}


def reverse_per_base_tags(r: bytearray) -> None:
    if not struct.unpack_from("<H", r, 14)[0] & 0x10:
        return
    for tag in (b"cd", b"ce", b"ad", b"ae", b"bd", b"be", b"aq", b"bq", b"ac", b"bc"):
        f = find_tag(bytes(r), tag)
        if f is None:
            continue
        s, e, vt = f
        if vt == ord("B") and tag not in (b"ac", b"bc"):
            es, cnt = FIXED[r[s + 3]], struct.unpack_from("<I", r, s + 4)[0]
            d = s + 8
            elems = [bytes(r[d + k * es:d + (k + 1) * es]) for k in range(cnt)]
            r[d:d + cnt * es] = b"".join(elems[::-1])
        elif vt == ord("Z"):
            v = bytes(r[s + 3:e - 1])[::-1]
            if tag in (b"ac", b"bc"):
                v = bytes(COMP.get(c, c) for c in v)
            r[s + 3:e - 1] = v


# ---- regenerate_alignment_tags_raw (alignment_tags.rs:254-420) ----------------------------------------------------
def regenerate(r: bytearray, idx: int, sq: Sequence[bytes], genome: Dict[bytes, bytes]) -> None:
    rec = R.Rec(bytes(r))
    if rec.flags & 0x4:
        for t in (b"NM", b"UQ", b"MD"):
            remove_tag(r, t)
        return
    if rec.ref_id < 0:
        return
    if rec.ref_id >= len(sq):
        raise FilterError("Reference sequence ID not found in header", idx)
    if rec.pos < 0:
        raise FilterError("Invalid alignment start position", idx)
    ops = rec.cigar_ops()
    span = sum(op >> 4 for op in ops if (op & 0xF) in (0, 2, 3, 7, 8))
    if span == 0:
        update_int(r, b"NM", 0)
        update_int(r, b"UQ", 0)
        update_string(r, b"MD", b"0")
        return
    name = sq[rec.ref_id]
    if name not in genome:
        raise FilterError("reference sequence not found", idx)
    contig = genome[name]
    if rec.pos + span > len(contig):
        raise FilterError("region exceeds sequence length", idx)
    ref = contig[rec.pos:rec.pos + span]
    seq, qual = rec.sequence(), rec.quals()
    nm = uq = run = ro = sp = 0
    md = bytearray()
    for op in ops:
        t, n = op & 0xF, op >> 4
        if t in (0, 7, 8):
            if sp + n > rec.l_seq:
                raise FilterError("CIGAR consumes more bases than sequence length", idx)
            for k in range(n):
                sb, rb = seq[sp], ref[ro + k]
                if sb == ord("N") or bytes([sb]).lower() != bytes([rb]).lower():
                    nm += 1
                    uq += qual[sp]
                    md += str(run).encode() + bytes([rb])
                    run = 0
                else:
                    run += 1
                sp += 1
            ro += n
        elif t == 1:
            if sp + n > rec.l_seq:
                raise FilterError("CIGAR consumes more bases than sequence length", idx)
            nm += n
            sp += n
        elif t == 2:
            nm += n
            md += str(run).encode() + b"^" + ref[ro:ro + n]
            run = 0
            ro += n
        elif t == 4:
            if sp + n > rec.l_seq:
                raise FilterError("CIGAR consumes more bases than sequence length", idx)
            sp += n
        elif t == 3:
            ro += n
    md += str(run).encode()
    update_int(r, b"NM", nm)
    update_int(r, b"UQ", min(uq, 2 ** 31 - 1))
    update_string(r, b"MD", bytes(md))


# ---- the command ------------------------------------------------------------------------------------------------
@dataclass
class Config:
    min_reads: Sequence[int] = (1,)
    max_read_error_rate: Sequence[float] = (0.025,)
    max_base_error_rate: Sequence[float] = (0.1,)
    min_base_quality: Optional[int] = None
    min_mean_base_quality: Optional[float] = None
    max_no_call_fraction: float = 0.2
    require_ss_agreement: bool = False
    filter_by_template: bool = True
    reverse_per_base_tags: bool = False

    def tiers(self):   # FilterConfig::new (filter.rs:237-330): missing values from the last one given
        three = lambda v: (list(v) + [list(v)[-1]] * 3)[:3]
        mr, re, be = three(self.min_reads), three(self.max_read_error_rate), three(self.max_base_error_rate)
        return [R.FilterThresholds(mr[k], re[k], be[k]) for k in range(3)]


def process_record(r: bytearray, idx: int, cfg: Config, sq, genome) -> Tuple[int, bool]:
    """process_record_raw (filter.rs:738-905) without methylation: (bases masked, pass)."""
    if len(r) < 32:
        raise FilterError("record shorter than 32 bytes", idx)
    if aux_offset(bytes(r)) > len(r) or 32 + r[8] > len(r):
        raise FilterError("truncated record", idx)
    flags = struct.unpack_from("<H", r, 14)[0]
    if genome is None and not flags & 0x4:
        raise FilterError("--ref is required when filtering mapped reads", idx)
    if cfg.reverse_per_base_tags:
        reverse_per_base_tags(r)
    cc, ab, ba = cfg.tiers()
    duplex = R.is_duplex_consensus(bytes(r[aux_offset(bytes(r)):]))
    if duplex:
        masked = R.mask_duplex_bases(r, cc, ab, ba, cfg.min_base_quality, cfg.require_ss_agreement)
    else:
        masked = R.mask_bases(r, cc, cfg.min_base_quality)
    if genome is not None:
        regenerate(r, idx, sq, genome)
    aux = R.Rec(bytes(r)).aux()
    st = R.filter_duplex_read(aux, cc, ab, ba) if duplex else R.filter_read(aux, cc)
    ok = st == R.FILTER_PASS and R.check_no_call_and_quality(bytes(r), cfg.min_mean_base_quality,
                                                            cfg.max_no_call_fraction)
    return masked, ok


def block(r: bytes) -> bytes:
    return struct.pack("<I", len(r)) + bytes(r)


def filter_records(records: Sequence[bytes], header_text: bytes, cfg: Config,
                   genome: Optional[Dict[bytes, bytes]]) -> Tuple[bytes, bytes, Dict[str, int]]:
    """(kept stream, rejects stream, {total, passed, failed, bases_masked}); FilterError for the first bad record in
    input order (every record is checked, so the first of several errors is found whatever the processing order)."""
    sq = sq_names(header_text)
    recs = [bytearray(r) for r in records]
    results, first_err = {}, None
    for i, r in enumerate(recs):   # per-record work in input order: the first failing record wins
        try:
            results[i] = process_record(r, i, cfg, sq, genome)
        except FilterError as e:
            first_err = e
            break
    if cfg.filter_by_template:
        lim = first_err.record if first_err else len(records)
        try:
            names = [R.Rec(bytes(records[i])).name for i in range(lim)]
            i = 0
            order_groups = []
            while i < lim:
                j = i + 1
                while j < lim and names[j] == names[i]:
                    j += 1
                order_groups.append(template_order(records, i, j))
                i = j
        except FilterError as e:
            first_err = e if first_err is None or e.record < first_err.record else first_err
    if first_err is not None:
        raise first_err
    kept, rej = bytearray(), bytearray()
    passed = masked = 0
    for i in range(len(recs)):
        masked += results[i][0]
    if not cfg.filter_by_template:
        for i, r in enumerate(recs):
            if results[i][1]:
                kept += block(r)
                passed += 1
            else:
                rej += block(r)
    else:
        for grp in order_groups:   # template_passes (fgumi-consensus filter.rs:371-395)
            prim = [k for k in grp if not struct.unpack_from("<H", recs[k], 14)[0] & 0x900]
            tpass = bool(prim) and all(results[k][1] for k in prim)
            for k in grp:
                primary = not struct.unpack_from("<H", recs[k], 14)[0] & 0x900
                ok = tpass if primary else tpass and results[k][1]
                if ok:
                    kept += block(recs[k])
                    passed += 1
                else:
                    rej += block(recs[k])
    n = len(records)
    return bytes(kept), bytes(rej), {"total": n, "passed": passed, "failed": n - passed, "bases_masked": masked}


def template_order(records: Sequence[bytes], b: int, e: int) -> List[int]:
    """Template::from_records order of records [b, e) as input indexes (dedup_oracle.build_templates)."""
    sub = [bytearray(records[k]) for k in range(b, e)]   # distinct objects, so that identity maps them back
    idx = {id(r): k for k, r in enumerate(sub, b)}
    try:
        t = D.build_templates(sub)
    except D.DedupError as err:
        # the second primary R1 / R2 of the run
        seen = set()
        for k in range(b, e):
            f = struct.unpack_from("<H", records[k], 14)[0]
            if f & 0x900:
                continue
            r1 = not f & 0x1 or f & 0x40
            if r1 in seen:
                raise FilterError(str(err), k)
            seen.add(r1)
        raise
    return [idx[id(r)] for r in t[0].records]
