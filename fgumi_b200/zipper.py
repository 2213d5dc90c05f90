"""`fgumi zipper` on raw BAM records (fgb_zipper_records): mapped records get their mate information, the unmapped
reads' tags and QC flag, normalised AS / XS and, on secondary and supplementary records, the tc tag; unmapped-only
templates pass through or are excluded.  The output comes back as a [u32 block_size][record] stream."""
from __future__ import annotations

import ctypes as C
import time
from typing import Dict, Iterable, Optional, Tuple

import numpy as np

from . import lib as _l
from .sort import _arrays

TIMING_NAMES = ("upload_ms", "sizes_ms", "scan_ms", "write_ms", "download_ms", "host_ms")
# TagSets (fgumi-umi lib.rs:200-210): the reference's lists exactly
CONSENSUS_REVERSE = ("ad", "ae", "bd", "be", "cd")
CONSENSUS_REVCOMP = ("aD", "bD", "cD")


def expand_tags(remove: Iterable[str], reverse: Iterable[str], revcomp: Iterable[str]):
    """TagInfo::new (fgumi-umi lib.rs:246-267): the name Consensus expands in the reverse and revcomp lists; names
    that are not two bytes match no tag and are dropped.  Sorted, duplicates removed."""
    rev, rc = set(), set()
    for t in reverse:
        rev.update(CONSENSUS_REVERSE if t == "Consensus" else [t])
    for t in revcomp:
        rc.update(CONSENSUS_REVCOMP if t == "Consensus" else [t])
    two = lambda s: sorted(t for t in s if len(t.encode()) == 2)
    return two(set(remove)), two(rev), two(rc)


def _names(tags) -> C.Array:
    buf = (C.c_char * max(2 * len(tags), 2))()
    for i, t in enumerate(tags):
        buf[2 * i:2 * i + 2] = t.encode()
    return buf


class Zipper:
    """fgb_zipper_records on one GPU with `--tags-to-remove / --tags-to-reverse / --tags-to-revcomp`,
    `--exclude-missing-reads` and `--skip-pa-tags`.  zip() takes whole QNAME runs of both streams."""

    def __init__(self, device: int = 0, tags_to_remove=(), tags_to_reverse=(), tags_to_revcomp=(),
                 exclude_missing_reads: bool = False, skip_pa_tags: bool = False, n_threads: int = 1,
                 device_bytes: int = 0):
        from .engine import Engine
        self.remove, self.reverse, self.revcomp = expand_tags(tags_to_remove, tags_to_reverse, tags_to_revcomp)
        self._bufs = [_names(self.remove), _names(self.reverse), _names(self.revcomp)]
        o = _l.FgbZipperOptions()
        o.exclude_missing_reads = 1 if exclude_missing_reads else 0
        o.skip_pa_tags = 1 if skip_pa_tags else 0
        o.n_threads = n_threads
        o.device_bytes = device_bytes
        o.n_remove, o.n_reverse, o.n_revcomp = len(self.remove), len(self.reverse), len(self.revcomp)
        o.tags_to_remove, o.tags_to_reverse, o.tags_to_revcomp = [C.addressof(b) for b in self._bufs]
        self.opt = o
        self._eng = Engine(device)
        self._lib = self._eng._lib
        self.bad_record: Optional[int] = None
        self.last_copy_s = 0.0

    def close(self):
        self._eng.close()

    def zip(self, u_bodies, u_off, m_bodies, m_off, last_call: bool = True) -> Tuple[bytes, int, Dict[str, int]]:
        """(output stream, mapped records consumed, {merged, unmapped_only, excluded, records_out}).  A failing call
        raises FgbError and sets self.bad_record (unmapped records first, then the mapped ones)."""
        ub, uo = _arrays(u_bodies, u_off)
        mb, mo = _arrays(m_bodies, m_off)
        out, n, used, bad = C.c_void_p(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        stats = (C.c_uint64 * 4)()
        st = self._lib.fgb_zipper_records(self._eng._h, C.byref(self.opt), ub.ctypes.data, uo.ctypes.data, len(uo) - 1,
                                          mb.ctypes.data, mo.ctypes.data, len(mo) - 1, int(last_call), C.byref(out),
                                          C.byref(n), C.byref(used), stats, C.byref(bad))
        self.bad_record = None if bad.value == 2 ** 64 - 1 else bad.value
        self._eng._check(st, "fgb_zipper_records")
        t0 = time.perf_counter()
        data = C.string_at(out.value, n.value) if n.value else b""
        self.last_copy_s = time.perf_counter() - t0   # the stream copied out of the library into Python bytes
        return data, used.value, dict(zip(_l.ZIPPER_STAT_NAMES, list(stats)))

    def last_timing(self) -> Dict[str, float]:
        ms = (C.c_double * 6)()
        self._eng._check(self._lib.fgb_zipper_last_timing(self._eng._h, ms), "fgb_zipper_last_timing")
        return dict(zip(TIMING_NAMES, list(ms)))


def host_zip(opt, u_bodies, u_off, m_bodies, m_off, last_call: bool = True):
    """fgb_host_zipper_records with the options of a Zipper-like `opt` (FgbZipperOptions): (status, stream, consumed,
    stats, bad_record).  The host twin of the device call, for tests."""
    lib = _l.load()
    ub, uo = _arrays(u_bodies, u_off)
    mb, mo = _arrays(m_bodies, m_off)
    out, n, used, bad = C.c_void_p(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    stats = (C.c_uint64 * 4)()
    st = lib.fgb_host_zipper_records(C.byref(opt), ub.ctypes.data, uo.ctypes.data, len(uo) - 1, mb.ctypes.data,
                                     mo.ctypes.data, len(mo) - 1, int(last_call), C.byref(out), C.byref(n),
                                     C.byref(used), stats, C.byref(bad))
    data = C.string_at(out.value, n.value) if st == 0 and n.value else b""
    if out.value:
        lib.fgb_host_free_buffer(out)
    return st, data, used.value, list(stats), (None if bad.value == 2 ** 64 - 1 else bad.value)


def options(tags_to_remove=(), tags_to_reverse=(), tags_to_revcomp=(), exclude_missing_reads=False,
            skip_pa_tags=False, n_threads=1):
    """An FgbZipperOptions without a device (for host_zip); keeps its name buffers alive on the object."""
    remove, reverse, revcomp = expand_tags(tags_to_remove, tags_to_reverse, tags_to_revcomp)
    o = _l.FgbZipperOptions()
    o._bufs = [_names(remove), _names(reverse), _names(revcomp)]
    o.exclude_missing_reads, o.skip_pa_tags, o.n_threads = int(exclude_missing_reads), int(skip_pa_tags), n_threads
    o.n_remove, o.n_reverse, o.n_revcomp = len(remove), len(reverse), len(revcomp)
    o.tags_to_remove, o.tags_to_reverse, o.tags_to_revcomp = [C.addressof(b) for b in o._bufs]
    return o
