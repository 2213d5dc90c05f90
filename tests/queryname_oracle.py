"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Restatement (pure Python) of `fgumi sort --order queryname` and `--order queryname::natural`: the name and flag
extraction, the two comparators, the output header and `--verify`, line by line.  It sits beside oracle/sort_oracle.py
(coordinate and template-coordinate), which it leaves unchanged.  Citations are relative to the fgumi 0.2.0 source
tree:
  keys.rs      src/lib/sort/keys.rs                   (queryname_flag_order, extract_raw_name_and_flags,
                                                       RawQuerynameKey, RawQuerynameLexKey)
  raw_sort.rs  crates/fgumi-raw-bam/src/sort.rs       (natural_compare_nul)
  mod.rs       src/lib/sort/mod.rs                    (create_output_header)
  sort.rs      src/lib/commands/sort.rs               (the order strings, --verify)

The reference sorts each in-memory chunk with an unstable sort (raw.rs:2193), so records with equal keys have no
defined order there; here, as for the other orders, the order is Python's stable `sorted` by the comparator.
"""
from __future__ import annotations

import functools
import struct
from typing import Dict, List, Optional, Sequence, Tuple

ORDERS = ("queryname", "queryname::natural")   # sort.rs:71-76 (the ::lex aliases are the first)


def queryname_flag_order(flags: int) -> int:
    """keys.rs:361-363."""
    return ((flags & 0xc0) << 8) | ((flags & 0x100) << 3) | ((flags & 0x800) >> 3)


def name_and_flags(r: bytes) -> Tuple[bytes, int]:
    """extract_raw_name_and_flags (keys.rs:450-456): bam[32 .. 32 + l_read_name - 1] if that fits the record, else
    empty (l_read_name 0 or 1 too); the flag order."""
    name_len = max(r[8] - 1, 0)
    name = r[32:32 + name_len] if name_len > 0 and 32 + name_len <= len(r) else b""
    return name, queryname_flag_order(struct.unpack_from("<H", r, 14)[0])


def _sign(x: int) -> int:
    return (x > 0) - (x < 0)


def natural_compare_nul(a: bytes, b: bytes) -> int:
    """raw_sort.rs:181-238 on NUL-terminated strings: both are cut at their first NUL (RawQuerynameKey::new appends
    one, keys.rs:515-520), and reading at the end gives the terminating 0.  -1, 0 or 1."""
    a = a.split(b"\0", 1)[0] + b"\0"
    b = b.split(b"\0", 1)[0] + b"\0"

    def dig(c):
        return 0x30 <= c <= 0x39

    pa = pb = 0
    while a[pa] != 0 and b[pb] != 0:
        if not dig(a[pa]) or not dig(b[pb]):
            if a[pa] != b[pb]:
                return _sign(a[pa] - b[pb])
            pa += 1
            pb += 1
        else:
            while a[pa] == 0x30:                               # skip leading zeros
                pa += 1
            while b[pb] == 0x30:
                pb += 1
            while dig(a[pa]) and a[pa] == b[pb]:               # skip matching significant digits
                pa += 1
                pb += 1
            a_digit, b_digit = dig(a[pa]), dig(b[pb])
            diff = a[pa] - b[pb]
            if a_digit and b_digit:
                pa += 1
                pb += 1
            while dig(a[pa]) and dig(b[pb]):
                pa += 1
                pb += 1
            if dig(a[pa]):
                return 1
            if dig(b[pb]):
                return -1
            if diff != 0:
                return _sign(diff)
    if a[pa] != 0:
        return 1
    if b[pb] != 0:
        return -1
    return 0


def lexicographic_compare(a: bytes, b: bytes) -> int:
    """RawQuerynameLexKey::cmp's name part (keys.rs:624-628): a byte compare, embedded NULs included."""
    return _sign((a > b) - (a < b))


def name_compare(a: bytes, b: bytes, order: str) -> int:
    return natural_compare_nul(a, b) if order == "queryname::natural" else lexicographic_compare(a, b)


def compare(ra: bytes, rb: bytes, order: str) -> int:
    """The full key of two records: the name, then the flag order (RawQuerynameKey::cmp, keys.rs:541-549;
    RawQuerynameLexKey::cmp, :624-628)."""
    (na, fa), (nb, fb) = name_and_flags(ra), name_and_flags(rb)
    return name_compare(na, nb, order) or _sign(fa - fb)


def sort_records(records: Sequence[bytes], order: str) -> List[bytes]:
    """A stable sort by the key."""
    return sorted(records, key=functools.cmp_to_key(lambda x, y: compare(x, y, order)))


def sorted_stream(records: Sequence[bytes], order: str) -> bytes:
    return b"".join(struct.pack("<I", len(r)) + r for r in sort_records(records, order))


def verify(records: Sequence[bytes], order: str) -> Tuple[int, Optional[int]]:
    """verify_sort_order (sort.rs:376-408) with the comparisons of :692-707: the records whose full key is below the
    previous record's, and the index of the first of them."""
    violations, first = 0, None
    for i in range(1, len(records)):
        if compare(records[i], records[i - 1], order) < 0:
            violations += 1
            if first is None:
                first = i
    return violations, first


def output_header(header_text: bytes, order: str) -> Dict[str, str]:
    """create_output_header (mod.rs:95-118) with header_ss_tag (keys.rs:202-209): the input's @HD fields with SO, GO
    and SS removed, then SO:queryname and SS:lexicographic or SS:natural."""
    hd = next((ln for ln in header_text.decode().split("\n") if ln.startswith("@HD")), None)
    fields = {}
    if hd is not None:
        for f in hd.split("\t")[1:]:
            k, _, v = f.partition(":")
            fields[k] = v
    for t in ("SO", "GO", "SS"):
        fields.pop(t, None)
    fields["SO"] = "queryname"
    fields["SS"] = "natural" if order == "queryname::natural" else "lexicographic"
    return fields
