"""`fgumi dedup` from raw BAM records: position grouping that keeps secondary and supplementary records
(fgb_host_dedup_group_by_position) and the record-level deduper (fgb_deduper_*), whose UMI graph runs on the device
through fgb_umi_assign and whose template scores run on the device beside it (fgb_record_quality_scores).

    keep, groups = group_by_position(bodies, rec_off, header_text)   # every record is kept
    d = Deduper(device=0, strategy="adjacency", edits=1)
    d.add_groups(bodies, rec_off, groups)
    stream = d.flush()          # [u32 block_size][record]... with MI tags and 0x400 on the duplicates
    d.metrics()                 # DedupMetricsOutput (dedup.rs:122-150)
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np

from . import lib as _l
from .group import _AssignQueue, _group_by_position
from .umi import options as _umi_options

METRIC_NAMES = ("total_templates", "unique_templates", "duplicate_templates", "duplicate_rate", "total_reads",
                "unique_reads", "duplicate_reads", "secondary_reads", "supplementary_reads", "missing_tc_tag")


def group_by_position(bodies: np.ndarray, rec_off: np.ndarray, header_text: bytes,
                      cell_tag: Optional[bytes] = b"CB") -> Tuple[np.ndarray, np.ndarray]:
    """(keep mask, all ones; group table over the records).  A paired mapped primary record with a mapped mate and no
    MC tag raises ValueError naming the record."""
    return _group_by_position("fgb_host_dedup_group_by_position", bodies, rec_off, header_text, cell_tag)


def dedup_metrics(stats: Dict[str, int]) -> dict:
    """DedupMetricsOutput (dedup.rs:122-150): the counters and duplicate_rate = duplicate / total templates."""
    m = {k: stats[k] for k in METRIC_NAMES if k != "duplicate_rate"}
    m["duplicate_rate"] = stats["duplicate_templates"] / stats["total_templates"] if stats["total_templates"] else 0.0
    return {k: m[k] for k in METRIC_NAMES}


def record_quality_scores(engine, bodies: np.ndarray, rec_off: np.ndarray) -> np.ndarray:
    """fgb_record_quality_scores on an engine.Engine (or a bare fgb_handle*): per record the sum of its quality bytes
    capped at 15 (dedup.rs:230-249), computed on the device."""
    lib = _l.load()
    handle = getattr(engine, "_h", engine)
    n = len(rec_off) - 1
    out = np.zeros(max(n, 1), np.uint32)
    bodies = np.ascontiguousarray(bodies, np.uint8) if len(bodies) else np.zeros(1, np.uint8)
    rec_off = np.ascontiguousarray(rec_off, np.uint64)
    st = lib.fgb_record_quality_scores(handle, bodies.ctypes.data, rec_off.ctypes.data, n, out.ctypes.data)
    if st != _l.FGB_OK:
        buf = C.create_string_buffer(1024)
        lib.fgb_last_error(handle, buf, len(buf))
        raise _l.FgbError(st, "fgb_record_quality_scores", buf.value.decode(errors="replace"))
    return out[:n]


class Deduper(_AssignQueue):
    """fgb_deduper_* on one GPU; device=None gives a planning-only deduper (pending / flush_with_ids)."""
    _prefix, _stat_names, _n_stats = "fgb_deduper", _l.DEDUP_STAT_NAMES, _l.FGB_DEDUP_NSTATS
    _timing_names = ("prepare_ms", "device_phase_ms", "kernels_ms", "resolve_ms", "score_phase_ms", "score_kernel_ms",
                    "emit_ms")

    def __init__(self, device: Optional[int] = 0, strategy: str = "adjacency", edits: int = 1,
                 min_umi_length: Optional[int] = None, min_map_q: int = 0, include_non_pf: bool = False,
                 no_umi: bool = False, remove_duplicates: bool = False, umi_tag: bytes = b"RX",
                 assign_tag: bytes = b"MI", first_mi: int = 0, n_threads: int = 1):
        self._lib = _l.load()
        u = _umi_options(strategy, 0 if strategy == "identity" else edits, "mapped", min_umi_length, n_threads)
        self.opt = _l.FgbDedupOptions(u, min_map_q, int(include_non_pf), int(no_umi), int(remove_duplicates),
                                      umi_tag, assign_tag, first_mi)
        h = C.c_void_p()
        st = self._lib.fgb_deduper_create(_l.FGB_DEVICE_NONE if device is None else device, C.byref(self.opt),
                                          C.byref(h))
        if st != _l.FGB_OK:
            raise _l.FgbError(st, "fgb_deduper_create")
        self._h = h

    def flush_with_ids(self, kinds, ids, group_mi_count, scores) -> bytes:
        """Completes the flush from an assignment and template scores computed elsewhere, each indexed like the
        flattened pending() batch."""
        def flat(x, dt):
            return np.ascontiguousarray(np.asarray(x, dt).reshape(-1)) if len(x) else np.zeros(1, dt)
        kinds, ids, cnt_in, sc = (flat(kinds, np.uint8), flat(ids, np.uint64), flat(group_mi_count, np.uint64),
                                  flat(scores, np.uint32))
        data, n, cnt = C.c_void_p(), C.c_uint64(), C.c_uint64()
        self._call("flush_with_ids", ids.ctypes.data, kinds.ctypes.data, cnt_in.ctypes.data, sc.ctypes.data,
                   C.byref(data), C.byref(n), C.byref(cnt))
        return self._take(data, n)

    def histogram(self) -> Dict[int, int]:
        """Family sizes over every flush so far (unassigned templates skipped)."""
        n = C.c_uint64()
        self._call("histogram", None, None, 0, C.byref(n))
        sizes = np.zeros(max(n.value, 1), np.uint64)
        counts = np.zeros(max(n.value, 1), np.uint64)
        self._call("histogram", sizes.ctypes.data, counts.ctypes.data, n.value, C.byref(n))
        return {int(s): int(c) for s, c in zip(sizes[:n.value], counts[:n.value])}

    def last_timing(self) -> Dict[str, float]:
        """ms of the last flush: the assignment's host key tables, device phase, edge kernels (CUDA events) and host
        rules; the score phase as the host saw it and its kernel (CUDA events); then selection, flags and emit."""
        return super().last_timing()

    def metrics(self) -> dict:
        return dedup_metrics(self.stats())
