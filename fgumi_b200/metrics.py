"""`fgumi duplex-metrics` and `fgumi simplex-metrics` from raw BAM records (fgb_metrics_*): the QC tables of a
UMI-grouped stream -- family-size histograms, yield at 5 %..100 % downsampling and UMI counts.  The template pass and
the family counting run on the device; the UMI consensus and the tables on host threads.

    m = MetricsCollector(header_text, duplex=True, intervals=None, device=0)
    m.add_records(bodies, rec_off)      # whole QNAME runs per call, as many calls as wanted
    tables = m.finish()                  # {"family_sizes": text, "duplex_family_sizes": ..., ...}
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np

from . import lib as _l

TABLES = ("family_sizes", "duplex_family_sizes", "yield_metrics", "umi_counts", "duplex_umi_counts")
TEMPLATE_FIELDS = tuple(f for f, _ in _l.FgbMetricsTemplate._fields_ if f != "reserved")


class MetricsError(ValueError):
    """A failing add_records / finish: `bad_record` is the first bad record's index over every call."""

    def __init__(self, msg: str, status: int, bad_record: Optional[int]):
        super().__init__(msg)
        self.status = status
        self.bad_record = bad_record


def _options(duplex: bool, min_ab_reads: int, min_ba_reads: int, min_reads: int, duplex_umi_counts: bool,
             n_threads: int, device_bytes: int) -> _l.FgbMetricsOptions:
    o = _l.FgbMetricsOptions()
    o.mode = 1 if duplex else 0
    o.n_threads = n_threads
    o.min_ab_reads = min_ab_reads
    o.min_ba_reads = min_ba_reads
    o.min_reads = min_reads
    o.duplex_umi_counts = 1 if duplex_umi_counts else 0
    o.device_bytes = device_bytes
    return o


class MetricsCollector:
    """One collector per input stream.  device=FGB_DEVICE_NONE (-1) makes a planning-only collector that refuses
    add_records and finish."""

    def __init__(self, header_text: bytes, duplex: bool = True, intervals: Optional[bytes] = None, device: int = 0,
                 min_ab_reads: int = 1, min_ba_reads: int = 1, min_reads: int = 1, duplex_umi_counts: bool = False,
                 n_threads: int = 1, device_bytes: int = 0):
        self._lib = _l.load()
        self.duplex = duplex
        self.opt = _options(duplex, min_ab_reads, min_ba_reads, min_reads, duplex_umi_counts, n_threads, device_bytes)
        h = C.c_void_p()
        st = self._lib.fgb_metrics_create(device, C.byref(self.opt), header_text, len(header_text), intervals,
                                          len(intervals) if intervals is not None else 0, C.byref(h))
        if st != _l.FGB_OK:
            raise _l.FgbError(st, "fgb_metrics_create")
        self._h = h

    def close(self) -> None:
        if self._h:
            self._lib.fgb_metrics_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:   # pragma: no cover
            pass

    def _error(self) -> str:
        n = self._lib.fgb_metrics_last_error(self._h, None, 0)
        buf = C.create_string_buffer(n + 1)
        self._lib.fgb_metrics_last_error(self._h, buf, n + 1)
        return buf.value.decode(errors="replace")

    def _raise(self, st: int, bad: C.c_uint64, where: str):
        b = None if bad.value == 2 ** 64 - 1 else bad.value
        raise MetricsError(f"{where}: {self._error()}", st, b)

    def add_records(self, bodies: np.ndarray, rec_off: np.ndarray) -> None:
        bodies = np.ascontiguousarray(bodies, np.uint8)
        rec_off = np.ascontiguousarray(rec_off, np.uint64)
        bad = C.c_uint64()
        st = self._lib.fgb_metrics_add_records(self._h, bodies.ctypes.data, rec_off.ctypes.data, len(rec_off) - 1,
                                               C.byref(bad))
        if st != _l.FGB_OK:
            self._raise(st, bad, "fgb_metrics_add_records")

    def finish(self) -> Dict[str, str]:
        """The tables this mode writes, by name (TABLES), as TSV text."""
        bad = C.c_uint64()
        st = self._lib.fgb_metrics_finish(self._h, C.byref(bad))
        if st != _l.FGB_OK:
            self._raise(st, bad, "fgb_metrics_finish")
        out = {}
        for i, name in enumerate(TABLES):
            p, n = C.c_char_p(), C.c_uint64()
            if self._lib.fgb_metrics_table(self._h, i, C.byref(p), C.byref(n)) == _l.FGB_OK:
                out[name] = C.string_at(p, n.value).decode()
        return out

    def stats(self) -> Dict[str, int]:
        s = (C.c_uint64 * 8)()
        self._lib.fgb_metrics_stats(self._h, s)
        return dict(zip(_l.METRICS_STAT_NAMES, s))

    def last_timing(self) -> Dict[str, float]:
        t = (C.c_double * 4)()
        self._lib.fgb_metrics_last_timing(self._h, t)
        return dict(zip(("template_pass_ms", "family_pass_ms", "umi_consensus_ms", "host_ms"), t))


def host_templates(header_text: bytes, bodies: np.ndarray, rec_off: np.ndarray,
                   intervals: Optional[bytes] = None) -> list:
    """fgb_host_metrics_templates: one dict per QNAME run (TEMPLATE_FIELDS).  A malformed record or a template with
    two primary R1s / R2s raises MetricsError naming the record."""
    lib = _l.load()
    bodies = np.ascontiguousarray(bodies, np.uint8)
    rec_off = np.ascontiguousarray(rec_off, np.uint64)
    n = len(rec_off) - 1
    out = (_l.FgbMetricsTemplate * max(n, 1))()
    nt, bad = C.c_uint64(), C.c_uint64()
    st = lib.fgb_host_metrics_templates(header_text, len(header_text), intervals,
                                        len(intervals) if intervals is not None else 0, bodies.ctypes.data,
                                        rec_off.ctypes.data, n, out, n, C.byref(nt), C.byref(bad))
    if st != _l.FGB_OK:
        raise MetricsError("fgb_host_metrics_templates", st, None if bad.value == 2 ** 64 - 1 else bad.value)
    return [{f: getattr(out[i], f) for f in TEMPLATE_FIELDS} for i in range(nt.value)]


def name_fraction(name: bytes) -> Tuple[int, float, int]:
    """(Murmur3 hash, hash fraction, bucket) of a read name, as the collector computes them."""
    lib = _l.load()
    h, f, b = C.c_int32(), C.c_double(), C.c_uint32()
    st = lib.fgb_host_metrics_name_fraction(name, len(name), C.byref(h), C.byref(f), C.byref(b))
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_host_metrics_name_fraction")
    return h.value, f.value, b.value


def bucket(hash32: int) -> int:
    return _l.load().fgb_host_metrics_bucket(hash32)


def parse_intervals(text: bytes) -> list:
    """(name, start, end) 0-based half-open; ValueError for an unparsable line."""
    lib = _l.load()
    n = C.c_uint64()
    if lib.fgb_host_metrics_intervals(text, len(text), None, None, None, None, 0, C.byref(n)) != _l.FGB_OK:
        raise ValueError("unparsable interval text")
    k = n.value
    off, ln = np.zeros(max(k, 1), np.uint64), np.zeros(max(k, 1), np.uint64)
    s, e = np.zeros(max(k, 1), np.int64), np.zeros(max(k, 1), np.int64)
    lib.fgb_host_metrics_intervals(text, len(text), off.ctypes.data, ln.ctypes.data, s.ctypes.data, e.ctypes.data, k,
                                   C.byref(n))
    return [(text[int(off[i]):int(off[i] + ln[i])].decode(), int(s[i]), int(e[i])) for i in range(k)]


def format_float(v: float) -> str:
    buf = C.create_string_buffer(64)
    _l.load().fgb_host_metrics_format_float(v, buf, 64)
    return buf.value.decode()
