"""`fgumi group` from raw BAM records: position grouping (fgb_host_group_by_position) and the record-level grouper
(fgb_grouper_*), whose UMI graph runs on the device through fgb_umi_assign.

    keep, groups = group_by_position(bodies, rec_off, header_text)
    bodies, rec_off = compact(bodies, rec_off, keep)
    g = ReadGrouper(device=0, strategy="adjacency", edits=1)
    g.add_groups(bodies, rec_off, groups)
    stream = g.flush()          # [u32 block_size][record]... with MI tags, in input order
    g.metrics()                 # UmiGroupingMetrics (group.rs:670-716)
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np

from . import lib as _l
from .umi import options as _umi_options


def _group_by_position(fn: str, bodies: np.ndarray, rec_off: np.ndarray, header_text: bytes,
                       cell_tag: Optional[bytes]) -> Tuple[np.ndarray, np.ndarray]:
    """Position grouping through the C function `fn` (fgb_host_group_by_position or its dedup form)."""
    lib = _l.load()
    n = len(rec_off) - 1
    keep = np.zeros(max(n, 1), np.uint8)
    gb = np.zeros(n + 2, np.uint64)
    ng, bad = C.c_uint64(), C.c_uint64()
    bodies = np.ascontiguousarray(bodies, np.uint8)
    rec_off = np.ascontiguousarray(rec_off, np.uint64)
    st = getattr(lib, fn)(bodies.ctypes.data, rec_off.ctypes.data, n, header_text, len(header_text), cell_tag,
                          keep.ctypes.data, gb.ctypes.data, C.byref(ng), C.byref(bad))
    if st == _l.FGB_ERR_INVALID_ARG and bad.value < n:
        i = bad.value
        rec = bodies[int(rec_off[i]):int(rec_off[i + 1])].tobytes()
        raise ValueError(f"record {i} ({rec[32:32 + rec[8] - 1].decode(errors='replace')}): paired-end reads need "
                         "MC tags for position grouping")
    if st != _l.FGB_OK:
        raise _l.FgbError(st, fn)
    return keep[:n], gb[:ng.value + 1]


def group_by_position(bodies: np.ndarray, rec_off: np.ndarray, header_text: bytes,
                      cell_tag: Optional[bytes] = b"CB") -> Tuple[np.ndarray, np.ndarray]:
    """(keep mask, group table over the kept records).  A paired mapped record with a mapped mate and no MC tag
    raises ValueError naming the record."""
    return _group_by_position("fgb_host_group_by_position", bodies, rec_off, header_text, cell_tag)


def compact(bodies: np.ndarray, rec_off: np.ndarray, keep: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """The kept records back to back, with their offset table: one slice copy per run of consecutive kept records."""
    k = keep.astype(bool)
    if k.all():
        return bodies, rec_off
    edges = np.flatnonzero(np.diff(np.concatenate([[0], k.view(np.int8), [0]])))   # run starts and ends, alternating
    runs = edges.reshape(-1, 2)
    parts = [bodies[int(rec_off[a]):int(rec_off[b])] for a, b in runs]
    lens = (rec_off[1:] - rec_off[:-1])[k]
    off = np.zeros(len(lens) + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    return (np.concatenate(parts) if parts else np.zeros(0, np.uint8)), off


def grouping_metrics(stats: Dict[str, int], family_sizes: Dict[int, int]) -> dict:
    """UmiGroupingMetrics (build_grouping_metrics, group.rs:670-716); the median is the first size whose cumulative
    count reaches total / 2 in integer division."""
    m = {k: stats[k] for k in ("total_records", "accepted_records", "discarded_non_pf", "discarded_poor_alignment",
                               "discarded_ns_in_umi", "discarded_umi_too_short")}
    total = sum(family_sizes.values())
    m.update(total_families=total, unique_molecule_ids=total, avg_reads_per_molecule=0.0,
             median_reads_per_molecule=0, min_reads_per_molecule=0, max_reads_per_molecule=0)
    if total:
        m["avg_reads_per_molecule"] = m["accepted_records"] / total
    if family_sizes:
        sizes = sorted(family_sizes.items())
        cum = 0
        for s, c in sizes:
            cum += c
            if cum >= total // 2:
                m["median_reads_per_molecule"] = s
                break
        m["min_reads_per_molecule"], m["max_reads_per_molecule"] = sizes[0][0], sizes[-1][0]
    return m


class _AssignQueue:
    """What ReadGrouper and Deduper share: the C handle `<_prefix>_*` of a queue of position groups around
    fgb_umi_assign, its `_n_stats` counters named by `_stat_names` and its flush timings named by `_timing_names`."""
    _prefix: str
    _stat_names: Tuple[str, ...]
    _n_stats: int
    _timing_names: Tuple[str, ...]
    _h = None

    def close(self):
        if self._h:
            getattr(self._lib, self._prefix + "_destroy")(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st: int, where: str):
        if st != _l.FGB_OK:
            buf = C.create_string_buffer(1024)
            getattr(self._lib, self._prefix + "_last_error")(self._h, buf, len(buf))
            raise _l.FgbError(st, where, buf.value.decode(errors="replace"))

    def _call(self, fn: str, *args):
        """`<_prefix>_<fn>(handle, *args)`, checked."""
        name = f"{self._prefix}_{fn}"
        self._check(getattr(self._lib, name)(self._h, *args), name)

    def add_groups(self, bodies: np.ndarray, rec_off: np.ndarray, groups: np.ndarray):
        bodies = np.ascontiguousarray(bodies, np.uint8)
        rec_off = np.ascontiguousarray(rec_off, np.uint64)
        groups = np.ascontiguousarray(groups, np.uint64)
        self._call("add_groups", bodies.ctypes.data, rec_off.ctypes.data, groups.ctypes.data, len(groups) - 1)

    def pending(self):
        """The queued UMI batch as fgb_umi_assign would receive it: groups -> calls -> UMIs (bytes)."""
        um, uo, co, go = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        nu, nc, ng = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._call("pending", C.byref(um), C.byref(uo), C.byref(nu), C.byref(co), C.byref(nc), C.byref(go),
                   C.byref(ng))

        def arr(p, n):
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint64)), (n,)).copy()
        uoff, coff, goff = arr(uo, nu.value + 1), arr(co, nc.value + 1), arr(go, ng.value + 1)
        blob = C.string_at(um.value, int(uoff[-1])) if uoff[-1] else b""
        umis = [blob[int(uoff[i]):int(uoff[i + 1])] for i in range(nu.value)]
        calls = [umis[int(coff[c]):int(coff[c + 1])] for c in range(nc.value)]
        return [calls[int(goff[g]):int(goff[g + 1])] for g in range(ng.value)]

    def _take(self, data, n) -> bytes:
        return C.string_at(data.value, n.value) if n.value else b""

    def flush(self) -> bytes:
        data, n, cnt = C.c_void_p(), C.c_uint64(), C.c_uint64()
        self._call("flush", C.byref(data), C.byref(n), C.byref(cnt))
        return self._take(data, n)

    def stats(self) -> Dict[str, int]:
        s = (C.c_uint64 * self._n_stats)()
        self._call("stats", s)
        return dict(zip(self._stat_names, list(s)))

    def last_timing(self) -> Dict[str, float]:
        ms = (C.c_double * len(self._timing_names))()
        self._call("last_timing", ms)
        return dict(zip(self._timing_names, list(ms)))


class ReadGrouper(_AssignQueue):
    """fgb_grouper_* on one GPU; device=None gives a planning-only grouper (pending / flush_with_ids)."""
    _prefix, _stat_names, _n_stats = "fgb_grouper", _l.GROUP_STAT_NAMES, _l.FGB_GROUP_NSTATS
    _timing_names = ("prepare_ms", "device_phase_ms", "kernels_ms", "resolve_ms", "emit_ms")

    def __init__(self, device: Optional[int] = 0, strategy: str = "adjacency", edits: int = 1,
                 allow_unmapped: bool = False, min_umi_length: Optional[int] = None, min_map_q: int = 1,
                 include_non_pf: bool = False, no_umi: bool = False, umi_tag: bytes = b"RX",
                 assign_tag: bytes = b"MI", first_mi: int = 0, n_threads: int = 1):
        self._lib = _l.load()
        u = _umi_options(strategy, 0 if strategy == "identity" else edits,
                         "unmapped" if allow_unmapped else "mapped", min_umi_length, n_threads)
        self.opt = _l.FgbGroupOptions(u, min_map_q, int(include_non_pf), int(no_umi), 0, umi_tag, assign_tag,
                                      first_mi)
        h = C.c_void_p()
        st = self._lib.fgb_grouper_create(_l.FGB_DEVICE_NONE if device is None else device, C.byref(self.opt),
                                          C.byref(h))
        if st != _l.FGB_OK:
            raise _l.FgbError(st, "fgb_grouper_create")
        self._h = h

    def flush_with_ids(self, kinds, ids, group_mi_count) -> bytes:
        kinds = np.ascontiguousarray(np.asarray(kinds, np.uint8).reshape(-1)) if len(kinds) else np.zeros(1, np.uint8)
        ids = np.ascontiguousarray(np.asarray(ids, np.uint64).reshape(-1)) if len(ids) else np.zeros(1, np.uint64)
        cnt_in = (np.ascontiguousarray(np.asarray(group_mi_count, np.uint64)) if len(group_mi_count)
                  else np.zeros(1, np.uint64))
        data, n, cnt = C.c_void_p(), C.c_uint64(), C.c_uint64()
        self._call("flush_with_ids", ids.ctypes.data, kinds.ctypes.data, cnt_in.ctypes.data, C.byref(data),
                   C.byref(n), C.byref(cnt))
        return self._take(data, n)

    def histogram(self, which: str = "family") -> Dict[int, int]:
        """Family sizes ("family") or position-group sizes ("position") over every flush so far."""
        w = _l.FGB_GROUP_HIST_FAMILY if which == "family" else _l.FGB_GROUP_HIST_POSITION
        n = C.c_uint64()
        self._call("histogram", w, None, None, 0, C.byref(n))
        sizes = np.zeros(max(n.value, 1), np.uint64)
        counts = np.zeros(max(n.value, 1), np.uint64)
        self._call("histogram", w, sizes.ctypes.data, counts.ctypes.data, n.value, C.byref(n))
        return {int(s): int(c) for s, c in zip(sizes[:n.value], counts[:n.value])}

    def last_timing(self) -> Dict[str, float]:
        """ms of the last flush: the assignment's host key tables, device phase, edge kernels (CUDA events) and host
        rules, then the sort, tags and output stream."""
        return super().last_timing()

    def metrics(self) -> dict:
        return grouping_metrics(self.stats(), self.histogram("family"))
