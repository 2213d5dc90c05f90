"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Restatement (pure Python) of `fgumi sort` in coordinate and template-coordinate order: the two key functions, the
library lookup, the output header and `--verify`, line by line.  Citations are relative to the fgumi 0.2.0 source
tree:
  inline_buffer.rs  src/lib/sort/inline_buffer.rs         (PackedCoordinateKey, TemplateKey, core_cmp)
  raw.rs            src/lib/sort/raw.rs                   (LibraryLookup, extract_template_key_inline)
  mod.rs            src/lib/sort/mod.rs                   (create_output_header)
  sort.rs           src/lib/commands/sort.rs              (verify_sort_order, the cell tag)
  tags.rs           crates/fgumi-raw-bam/src/tags.rs      (parse_mi_bytes, extract_template_aux_tags)
  fields.rs         crates/fgumi-raw-bam/src/fields.rs    (tag_value_size, aux_data_slice)
  cigar.rs          crates/fgumi-raw-bam/src/cigar.rs     (unclipped_5prime_raw, mate_unclipped_5prime)

The one deviation: the reference hashes read names and cell barcodes with ahash (raw.rs:212-220, 274-290), whose
values depend on the CPU features of the build; here both are `fnv1a64`.  Every path of the reference sorts stably, so
the order is Python's stable `sorted` by the key.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Optional, Sequence, Tuple

M64 = (1 << 64) - 1
I32_MAX = 2 ** 31 - 1
PAIRED, UNMAPPED, MATE_UNMAPPED, REVERSE, MATE_REVERSE, LAST = 0x1, 0x4, 0x8, 0x10, 0x20, 0x80


def fnv1a64(data: bytes) -> int:
    """THE DEVIATION: 64-bit FNV-1a in place of the reference's seeded ahash, for read names and cell barcodes."""
    h = 0xcbf29ce484222325
    for c in data:
        h = ((h ^ c) * 0x100000001b3) & M64
    return h


def _i32(x: int) -> int:   # Rust i32 arithmetic wraps in a release build
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >= 1 << 31 else x


def _fields(r: bytes):
    tid, pos = struct.unpack_from("<ii", r, 0)
    flag = struct.unpack_from("<H", r, 14)[0]
    mate_tid, mate_pos = struct.unpack_from("<ii", r, 20)
    return tid, pos, flag, mate_tid, mate_pos


# ---- coordinate -------------------------------------------------------------------------------------------------
def coordinate_key(r: bytes) -> int:
    """extract_coordinate_key_inline (inline_buffer.rs:423-436) + PackedCoordinateKey::new (:66-78)."""
    tid, pos, flag, _, _ = _fields(r)
    if tid < 0:
        return M64                                               # PackedCoordinateKey::unmapped (:83-85)
    return ((tid << 34) | ((((pos & M64) + 1) & M64) << 1) | (1 if flag & REVERSE else 0)) & M64


# ---- aux scan ---------------------------------------------------------------------------------------------------
_FIXED = {ord(c): n for c, n in (("A", 1), ("c", 1), ("C", 1), ("s", 2), ("S", 2), ("i", 4), ("I", 4), ("f", 4))}


def tag_value_size(t: int, data: bytes) -> Optional[int]:
    """fields.rs:289-310 (TAG_FIXED_SIZES :269-280: fixed sizes whether or not the value fits)."""
    if t in _FIXED:
        return _FIXED[t]
    if t in (ord("Z"), ord("H")):
        z = data.find(b"\0")
        return None if z < 0 else z + 1
    if t == ord("B"):
        if len(data) < 5 or data[0] not in _FIXED:
            return None
        return 5 + struct.unpack_from("<I", data, 1)[0] * _FIXED[data[0]]
    return None


def aux_data(r: bytes) -> bytes:
    """aux_data_slice (fields.rs:449-483): empty when the offset runs past the record."""
    n_cig = struct.unpack_from("<H", r, 12)[0]
    l_seq = struct.unpack_from("<I", r, 16)[0]
    off = 32 + r[8] + 4 * n_cig + (l_seq + 1) // 2 + l_seq
    return r[off:] if off <= len(r) else b""


def parse_mi_bytes(s: bytes) -> Optional[Tuple[int, bool]]:
    """tags.rs:184-212."""
    if not s:
        return None
    if len(s) >= 2 and s[-2] == ord("/"):
        num, is_a = s[:-2], s[-1] != ord("B")
    else:
        num, is_a = s, True
    if not num:
        return None
    v = 0
    for c in num:
        if not 0x30 <= c <= 0x39:
            return None
        v = min(v * 10, M64)                                     # saturating_mul(10)
        v = min(v + (c - 0x30), M64)                             # saturating_add
    return v, is_a


def _utf8(b: bytes) -> bool:
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def _int_value(a: bytes, p: int, t: int) -> Optional[int]:
    """extract_int_value (tags.rs:127-151)."""
    fmt = {ord("c"): "<b", ord("C"): "<B", ord("s"): "<h", ord("S"): "<H", ord("i"): "<i", ord("I"): "<I"}.get(t)
    if fmt is None or p + 3 + struct.calcsize(fmt) > len(a):
        return None
    return struct.unpack_from(fmt, a, p + 3)[0]


def template_aux_tags(r: bytes, cell_tag: Optional[bytes]):
    """extract_template_aux_tags (tags.rs:299-377): (mi, is_a), rg, cell, mc -- one pass that ends early once every
    wanted tag has been met, a later entry replacing an earlier one until then; MC only if it is UTF-8."""
    a = aux_data(r)
    mi, rg, cell, mc = (0, True), None, None, None
    target = 0xF if cell_tag is not None else 0b1011
    found = 0
    p = 0
    while p + 3 <= len(a):
        t, vt = a[p:p + 2], a[p + 2]
        if t == b"MI":
            if vt == ord("Z"):
                end = a.find(b"\0", p + 3)
                if end < 0:
                    break
                mi = parse_mi_bytes(a[p + 3:end]) or (0, True)
                p = end + 1
            else:
                v = _int_value(a, p, vt)
                if v is not None and v >= 0:
                    mi = (v, True)
                size = tag_value_size(vt, a[p + 3:])
                if size is None:
                    break
                p += 3 + size
            found |= 1
            if found & target == target:
                return mi, rg, cell, mc
            continue
        if vt == ord("Z"):
            end = a.find(b"\0", p + 3)
            if end < 0:
                break
            value = a[p + 3:end]
            if t == b"RG":
                rg = value
                found |= 2
            if cell_tag is not None and t == cell_tag:
                cell = value
                found |= 4
            if t == b"MC":
                mc = value if _utf8(value) else None
                found |= 8
            if found & target == target:
                return mi, rg, cell, mc
            p = end + 1
            continue
        size = tag_value_size(vt, a[p + 3:])
        if size is None:
            break
        p += 3 + size
    return mi, rg, cell, mc


# ---- positions --------------------------------------------------------------------------------------------------
def unclipped_5prime_raw(r: bytes, pos: int, is_reverse: bool) -> int:
    """cigar.rs:237-255, 470-508: 0-based like pos; pos unchanged without a CIGAR or when it runs past the record."""
    n = struct.unpack_from("<H", r, 12)[0]
    if n == 0:
        return pos
    start = 32 + r[8]
    if start + 4 * n > len(r):
        return pos
    ops = struct.unpack_from("<%dI" % n, r, start)
    if not is_reverse:
        clipped = 0
        for op in ops:
            if op & 0xF in (4, 5):
                clipped += op >> 4
            else:
                break
        return _i32(pos - clipped)
    ref_len = trailing = 0
    saw = False
    for op in ops:
        if op & 0xF in (0, 2, 3, 7, 8):
            ref_len += op >> 4
            trailing = 0
            saw = True
        elif op & 0xF in (4, 5) and saw:
            trailing += op >> 4
    return _i32(pos + ref_len + trailing - 1)


def _parse_num(s: bytes) -> int:   # str::parse::<i32>().unwrap_or(0) on a run of digits
    return int(s) if s and int(s) <= I32_MAX else 0


def mate_unclipped_5prime(mate_pos: int, mate_reverse: bool, mc: bytes) -> int:
    """cigar.rs:263-269 over unclipped_other_start / _end (:294-306) and the MC parsers (:514-573); 0-based."""
    start = 0
    if not mate_reverse:
        clipped = 0
        for i, c in enumerate(mc):
            if 0x30 <= c <= 0x39:
                continue
            if c in b"SH":
                clipped += _parse_num(mc[start:i])
                start = i + 1
            else:
                break
        return _i32(mate_pos - clipped)
    ref_len = trailing = 0
    saw = False
    for i, c in enumerate(mc):
        if 0x30 <= c <= 0x39:
            continue
        num = _parse_num(mc[start:i])
        start = i + 1
        if c in b"MDN=X":
            ref_len += num
            trailing = 0
            saw = True
        elif c in b"SH" and saw:
            trailing += num
    return _i32(mate_pos + ref_len + trailing - 1)


# ---- library lookup ---------------------------------------------------------------------------------------------
def library_lookup(header_text: bytes) -> Dict[bytes, int]:
    """LibraryLookup::from_header (raw.rs:237-283): RG ID -> ordinal of its LB among the distinct LB values sorted
    bytewise, from 1; an RG without LB takes the ordinal of "" (0 unless some LB is empty)."""
    rgs = []
    for line in header_text.split(b"\n"):
        line = line.rstrip(b"\r")
        if not line.startswith(b"@RG\t"):
            continue
        rid, lb = None, None
        for f in line.split(b"\t")[1:]:
            if f.startswith(b"ID:"):
                rid = f[3:]
            elif f.startswith(b"LB:"):
                lb = f[3:]
        if rid is not None:
            rgs.append((rid, lb))
    libraries = sorted({lb for _, lb in rgs if lb is not None})
    lib_to_ordinal = {b"": 0}
    for i, lb in enumerate(libraries):
        lib_to_ordinal[lb] = i + 1
    return {rid: lib_to_ordinal.get(lb if lb is not None else b"", 0) for rid, lb in rgs}


# ---- template-coordinate ----------------------------------------------------------------------------------------
def template_key_new(tid1, pos1, neg1, tid2, pos2, neg2, cb_hash, library, mi, name_hash, is_upper) -> Tuple[int, ...]:
    """TemplateKey::new (inline_buffer.rs:478-520), truncations included."""
    def tid(t):
        return 0xFFFF if t == I32_MAX else max(t, 0) & 0xFFFF

    def pos(p):
        return (p & 0xFFFFFFFF) ^ 0x80000000

    p1 = (tid(tid1) << 48) | (tid(tid2) << 32) | pos(pos1)
    p2 = (pos(pos2) << 32) | ((not neg1) << 1) | (not neg2)
    p3 = ((library & 0xFFFF) << 48) | ((mi[0] & 0xFFFFFFFFFFFF) << 1) | (not mi[1])
    p4 = ((name_hash << 1) & M64) | is_upper
    return p1, p2, cb_hash, p3, p4


def template_key_unmapped(name_hash: int, cb_hash: int, is_read2: bool) -> Tuple[int, ...]:
    """TemplateKey::unmapped (inline_buffer.rs:524-532)."""
    return M64, M64, cb_hash, 0, ((name_hash << 1) & M64) | is_read2


def template_key(r: bytes, libs: Dict[bytes, int], cell_tag: Optional[bytes] = b"CB") -> Tuple[int, ...]:
    """extract_template_key_inline (raw.rs:2917-3013)."""
    mi, rg, cell, mc = template_aux_tags(r, cell_tag)
    library = libs.get(rg, 0) if rg is not None else 0           # ordinal_from_rg (raw.rs:307-312)
    cb_hash = fnv1a64(cell) if cell is not None else 0
    tid, pos, flag, mate_tid, mate_pos = _fields(r)
    is_unmapped, mate_unmapped = bool(flag & UNMAPPED), bool(flag & MATE_UNMAPPED)
    is_reverse, mate_reverse, is_paired = bool(flag & REVERSE), bool(flag & MATE_REVERSE), bool(flag & PAIRED)
    name_len = max(r[8] - 1, 0)
    name = r[32:32 + name_len] if name_len > 0 and 32 + name_len <= len(r) else b""
    name_hash = fnv1a64(name)
    if is_unmapped:
        if is_paired and not mate_unmapped:
            mate_unclipped = mate_pos if mc is None else mate_unclipped_5prime(mate_pos, mate_reverse, mc)
            return template_key_new(mate_tid, mate_unclipped, mate_reverse, I32_MAX, I32_MAX, False, cb_hash, library,
                                    mi, name_hash, True)
        return template_key_unmapped(name_hash, cb_hash, bool(flag & LAST))
    this_pos = unclipped_5prime_raw(r, pos, is_reverse)
    if is_paired and not mate_unmapped:
        mate_unclipped = mate_pos if mc is None else mate_unclipped_5prime(mate_pos, mate_reverse, mc)
        is_upper = (tid, this_pos) > (mate_tid, mate_unclipped) or \
            ((tid, this_pos) == (mate_tid, mate_unclipped) and is_reverse)
        if is_upper:
            return template_key_new(mate_tid, mate_unclipped, mate_reverse, tid, this_pos, is_reverse, cb_hash, library,
                                    mi, name_hash, True)
        return template_key_new(tid, this_pos, is_reverse, mate_tid, mate_unclipped, mate_reverse, cb_hash, library, mi,
                                name_hash, False)
    return template_key_new(tid, this_pos, is_reverse, I32_MAX, I32_MAX, False, cb_hash, library, mi, name_hash, False)


def core_key(k: Tuple[int, ...]) -> Tuple[int, ...]:
    """TemplateKey::core_cmp (inline_buffer.rs:604-618): everything but name_hash_upper."""
    return k[:4]


# ---- the command ------------------------------------------------------------------------------------------------
def keys(records: Sequence[bytes], header_text: bytes, order: str, cell_tag: Optional[bytes] = b"CB"):
    """The key of each record as the 5-word tuple the product reports (coordinate: the one word, then zeros)."""
    if order == "coordinate":
        return [(coordinate_key(r), 0, 0, 0, 0) for r in records]
    libs = library_lookup(header_text)
    return [template_key(r, libs, cell_tag) for r in records]


def sort_records(records: Sequence[bytes], header_text: bytes, order: str,
                 cell_tag: Optional[bytes] = b"CB") -> List[bytes]:
    """A stable sort by the key."""
    k = keys(records, header_text, order, cell_tag)
    return [records[i] for i in sorted(range(len(records)), key=lambda i: k[i])]


def sorted_stream(records: Sequence[bytes], header_text: bytes, order: str, cell_tag: Optional[bytes] = b"CB") -> bytes:
    return b"".join(struct.pack("<I", len(r)) + r for r in sort_records(records, header_text, order, cell_tag))


def verify(records: Sequence[bytes], header_text: bytes, order: str,
           cell_tag: Optional[bytes] = b"CB") -> Tuple[int, Optional[int]]:
    """verify_sort_order (sort.rs:376-408) with the comparisons of :700-720: the records whose key is below the
    previous one's (template-coordinate: core_cmp), and the index of the first of them."""
    k = keys(records, header_text, order, cell_tag)
    cmp = (lambda x: x[:1]) if order == "coordinate" else core_key
    violations, first = 0, None
    for i in range(1, len(k)):
        if cmp(k[i]) < cmp(k[i - 1]):
            violations += 1
            if first is None:
                first = i
    return violations, first


def output_header(header_text: bytes, order: str) -> Dict[str, str]:
    """create_output_header (mod.rs:72-129): the @HD fields of the output -- the input's, SO / GO / SS replaced."""
    hd = next((ln for ln in header_text.decode().split("\n") if ln.startswith("@HD")), None)
    fields = {}
    if hd is not None:
        for f in hd.split("\t")[1:]:
            k, _, v = f.partition(":")
            fields[k] = v
    for t in ("SO", "GO", "SS"):
        fields.pop(t, None)
    if order == "coordinate":
        fields["SO"] = "coordinate"
    else:
        fields.update(SO="unsorted", GO="query", SS="template-coordinate")
    return fields
