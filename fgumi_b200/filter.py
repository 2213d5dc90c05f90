"""`fgumi filter --ref` on raw BAM records (fgb_filter_records): masking, NM / UQ / MD regenerated against a reference
resident on the GPU, and the read- or template-level decision; kept and rejected records come back as
[u32 block_size][record] streams.  Methylation options and compressed FASTA are not offered."""
from __future__ import annotations

import ctypes as C
import os
import time
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import lib as _l
from .caller import DuplexConsensusFilter
from .sort import _arrays

TIMING_NAMES = ("upload_ms", "pass1_ms", "decide_scan_ms", "pass2_ms", "download_ms", "host_ms")


class Reference:
    """An uncompressed FASTA file parsed on the host and uploaded once to `device` (fgb_reference_create), where it
    stays until close().  The file is handed to the library through np.memmap."""

    def __init__(self, path: str, device: int = 0):
        self._lib = _l.load()
        self._h = C.c_void_p()
        size = os.path.getsize(path)
        data = np.memmap(path, dtype=np.uint8, mode="r") if size else np.zeros(1, np.uint8)
        st = self._lib.fgb_reference_create(device, data.ctypes.data, size, C.byref(self._h))
        del data
        if st != _l.FGB_OK:
            self._h = C.c_void_p()
            raise _l.FgbError(st, "fgb_reference_create", path)
        self.device = device

    def contigs(self) -> List[Tuple[str, int]]:
        out = []
        name, length = C.c_char_p(), C.c_uint64()
        for i in range(self._lib.fgb_reference_contigs(self._h)):
            self._lib.fgb_reference_contig(self._h, i, C.byref(name), C.byref(length))
            out.append((name.value.decode("utf-8", "replace"), length.value))
        return out

    def close(self):
        if self._h:
            self._lib.fgb_reference_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


class RecordFilter:
    """fgb_filter_records on one GPU.  The thresholds are DuplexConsensusFilter's (one to three values per option for
    the [duplex, AB, BA] tiers; simplex reads use the first); filter_by_template=False is `--filter-by-template false`.
    A call holds whole templates: filter() takes a whole input, and the caller cuts batches at QNAME changes."""

    def __init__(self, device: int = 0, min_reads=(1,), max_read_error_rate=(0.025,), max_base_error_rate=(0.1,),
                 min_base_quality=None, min_mean_base_quality=None, max_no_call_fraction: float = 0.2,
                 require_single_strand_agreement: bool = False, filter_by_template: bool = True,
                 reverse_per_base_tags: bool = False, track_rejects: bool = False, n_threads: int = 1,
                 device_bytes: int = 0):
        from .engine import Engine
        self.thresholds = DuplexConsensusFilter(min_reads, max_read_error_rate, max_base_error_rate, min_base_quality,
                                                min_mean_base_quality, max_no_call_fraction,
                                                require_single_strand_agreement)
        o = _l.FgbRecordFilterOptions()
        self.thresholds.fill(o.filter)
        o.filter_by_template = 1 if filter_by_template else 0
        o.reverse_per_base_tags = 1 if reverse_per_base_tags else 0
        o.track_rejects = 1 if track_rejects else 0
        o.n_threads = n_threads
        o.device_bytes = device_bytes
        self.opt = o
        self._eng = Engine(device)
        self._lib = self._eng._lib
        self.bad_record: Optional[int] = None
        self.last_copy_s = 0.0

    def close(self):
        self._eng.close()

    def filter(self, header_text: bytes, bodies, rec_off, reference: Optional[Reference] = None
               ) -> Tuple[bytes, bytes, Dict[str, int]]:
        """(kept stream, rejects stream, {total, passed, failed, bases_masked}).  A failing call raises FgbError and
        sets self.bad_record to the first bad record."""
        b, off = _arrays(bodies, rec_off)
        n = len(off) - 1
        kp, kl, rp, rl, bad = C.c_void_p(), C.c_uint64(), C.c_void_p(), C.c_uint64(), C.c_uint64()
        stats = (C.c_uint64 * 4)()
        st = self._lib.fgb_filter_records(self._eng._h, C.byref(self.opt), reference._h if reference else None,
                                          header_text, len(header_text), b.ctypes.data, off.ctypes.data, n,
                                          C.byref(kp), C.byref(kl), C.byref(rp), C.byref(rl), stats, C.byref(bad))
        self.bad_record = None if bad.value == 2 ** 64 - 1 else bad.value
        self._eng._check(st, "fgb_filter_records")
        t0 = time.perf_counter()
        kept = C.string_at(kp.value, kl.value) if kl.value else b""
        rejects = C.string_at(rp.value, rl.value) if rl.value else b""
        self.last_copy_s = time.perf_counter() - t0   # the streams copied out of the library into Python bytes
        return kept, rejects, dict(zip(_l.FILTER_STAT_NAMES, list(stats)))

    def last_timing(self) -> Dict[str, float]:
        ms = (C.c_double * 6)()
        self._eng._check(self._lib.fgb_filter_last_timing(self._eng._h, ms), "fgb_filter_last_timing")
        return dict(zip(TIMING_NAMES, list(ms)))


def filter_stats_text(stats: Dict[str, int]) -> str:
    """write_filter_stats (commands/filter.rs:713-731): four lines, pass_rate to 4 decimals."""
    total, passed = stats["total"], stats["passed"]
    rate = passed / total if total > 0 else 0.0
    return (f"total_reads\t{total}\npassed_reads\t{passed}\nfailed_reads\t{stats['failed']}\n"
            f"pass_rate\t{rate:.4f}\n")
