"""`fgumi sort` on raw BAM records: coordinate, template-coordinate and queryname order (lexicographic and natural),
keyed, radix-sorted and gathered on the device (fgb_sort_records), with the same keys and `--verify` on the host
(fgb_host_sort_keys, fgb_host_sort_name_key, fgb_host_sort_verify).

    s = RecordSorter(device=0, order="template-coordinate")
    stream = s.sort(header_text, bodies, rec_off)     # bytearray: [u32 block_size][record]..., stable by the key
    s.last_timing()                                   # upload / key kernel / sort / gather / download / merge, ms
    violations, first = verify(header_text, *bamio.split_stream(stream))   # 0, None
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional, Tuple

import numpy as np

from . import lib as _l

ORDERS = {"coordinate": _l.FGB_SORT_COORDINATE, "template-coordinate": _l.FGB_SORT_TEMPLATE_COORDINATE,
          "queryname": _l.FGB_SORT_QUERYNAME, "queryname::natural": _l.FGB_SORT_QUERYNAME_NATURAL}
NAME_KEY_WORDS = 65                                  # queryname: at most 64 name words and the last word
TIMING_NAMES = ("upload_ms", "key_kernel_ms", "sort_ms", "gather_ms", "download_ms", "merge_ms")


def options(order: str = "template-coordinate", cell_tag: Optional[bytes] = b"CB", device_bytes: int = 0,
            n_threads: Optional[int] = None) -> _l.FgbSortOptions:
    """fgb_sort_options; cell_tag None = no cell barcode in the template-coordinate key (the other orders ignore
    it)."""
    if order not in ORDERS:
        raise ValueError(f"unknown sort order {order!r} ({', '.join(ORDERS)})")
    if cell_tag is not None and len(cell_tag) != 2:
        raise ValueError("cell_tag must be two characters")
    threads = min(os.cpu_count() or 1, 16) if n_threads is None else n_threads
    return _l.FgbSortOptions(ORDERS[order], threads, cell_tag or b"", (C.c_uint8 * 6)(), device_bytes)


def _arrays(bodies, rec_off) -> Tuple[np.ndarray, np.ndarray]:
    bodies = np.ascontiguousarray(bodies, np.uint8)
    if bodies.size == 0:
        bodies = np.zeros(1, np.uint8)
    return bodies, np.ascontiguousarray(rec_off, np.uint64)


def _layout_error(st: int, bad: int, where: str):
    if st == _l.FGB_ERR_LAYOUT:
        raise _l.FgbError(st, where, f"record {bad} is shorter than its 32-byte fixed part")
    raise _l.FgbError(st, where)


def sort_keys(header_text: bytes, bodies, rec_off, order: str = "template-coordinate",
              cell_tag: Optional[bytes] = b"CB", n_threads: Optional[int] = None) -> np.ndarray:
    """The sort keys of every record as uint64[n, 5] (coordinate: column 0), from the code the key kernel runs.
    Coordinate and template-coordinate only: queryname keys are name_key's."""
    lib = _l.load()
    b, off = _arrays(bodies, rec_off)
    n = len(off) - 1
    keys = np.zeros((max(n, 1), 5), np.uint64)
    bad = C.c_uint64()
    o = options(order, cell_tag, 0, n_threads)
    st = lib.fgb_host_sort_keys(C.byref(o), header_text, len(header_text), b.ctypes.data, off.ctypes.data, n,
                                keys.ctypes.data, C.byref(bad))
    if st != _l.FGB_OK:
        _layout_error(st, bad.value, "fgb_host_sort_keys")
    return keys[:n]


def name_key(record: bytes, order: str = "queryname") -> Tuple[int, ...]:
    """The queryname key words of one record (no block_size prefix) from the code the key kernel runs: its name words,
    zero-padded to 64 as they would be in a run with longer names, then the last word (len(E) << 16 | flag order).
    Tuples of any two records compare as the device sorts them."""
    if order not in ("queryname", "queryname::natural"):
        raise ValueError(f"name_key takes a queryname order, not {order!r}")
    rec = np.frombuffer(bytes(record) or b"\0", np.uint8)
    words = np.zeros(NAME_KEY_WORDS, np.uint64)
    n = C.c_uint32()
    o = options(order, None, 0, 1)
    st = _l.load().fgb_host_sort_name_key(C.byref(o), rec.ctypes.data, len(record), words.ctypes.data,
                                          NAME_KEY_WORDS, C.byref(n))
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_host_sort_name_key")
    k = n.value - 1
    return tuple(int(w) for w in words[:k]) + (0,) * (NAME_KEY_WORDS - 1 - k) + (int(words[k]),)


def verify(header_text: bytes, bodies, rec_off, order: str = "template-coordinate",
           cell_tag: Optional[bytes] = b"CB", n_threads: Optional[int] = None) -> Tuple[int, Optional[int]]:
    """`fgumi sort --verify`: (records whose key is below the previous record's, index of the first or None)."""
    lib = _l.load()
    b, off = _arrays(bodies, rec_off)
    v, first, bad = C.c_uint64(), C.c_uint64(), C.c_uint64()
    o = options(order, cell_tag, 0, n_threads)
    st = lib.fgb_host_sort_verify(C.byref(o), header_text, len(header_text), b.ctypes.data, off.ctypes.data,
                                  len(off) - 1, C.byref(v), C.byref(first), C.byref(bad))
    if st != _l.FGB_OK:
        _layout_error(st, bad.value, "fgb_host_sort_verify")
    return v.value, (None if first.value == 2 ** 64 - 1 else first.value)


class RecordSorter:
    """fgb_sort_records on one GPU.  device_bytes bounds one sorted run (0: from the free device memory per call);
    a larger input is sorted in several runs and merged on the host."""

    def __init__(self, device: int = 0, order: str = "template-coordinate", cell_tag: Optional[bytes] = b"CB",
                 device_bytes: int = 0, n_threads: Optional[int] = None):
        from .engine import Engine
        self.opt = options(order, cell_tag, device_bytes, n_threads)
        self.order = order
        self._eng = Engine(device)
        self._lib = self._eng._lib

    def close(self):
        self._eng.close()

    def sort(self, header_text: bytes, bodies, rec_off) -> bytearray:
        """The records as [u32 block_size][record]..., stably sorted by their keys: a bytearray the library writes
        in place (no second copy of a stream of several GB)."""
        b, off = _arrays(bodies, rec_off)
        n = len(off) - 1
        out = bytearray(int(off[-1]) - int(off[0]) + 4 * n)
        buf = (C.c_uint8 * max(len(out), 1)).from_buffer(out) if out else (C.c_uint8 * 1)()
        out_len, bad = C.c_uint64(), C.c_uint64()
        st = self._lib.fgb_sort_records(self._eng._h, C.byref(self.opt), header_text, len(header_text), b.ctypes.data,
                                        off.ctypes.data, n, buf, len(out), C.byref(out_len), C.byref(bad))
        del buf
        if st == _l.FGB_ERR_LAYOUT:
            _layout_error(st, bad.value, "fgb_sort_records")
        self._eng._check(st, "fgb_sort_records")
        return out

    def last_timing(self) -> Dict[str, float]:
        ms = (C.c_double * 6)()
        self._eng._check(self._lib.fgb_sort_last_timing(self._eng._h, ms), "fgb_sort_last_timing")
        return dict(zip(TIMING_NAMES, list(ms)))
