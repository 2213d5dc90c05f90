"""Molecule IDs from UMIs on the device: the four `fgumi group` strategies behind fgb_umi_assign.

    a = UmiAssigner(device=0, strategy="adjacency", edits=1)               # mapped rules (the default)
    res = a.assign([[["ACGTACGT", "ACGTACGA"]], [["TTTTGGGG"]]])           # groups -> calls -> UMIs
    res.mi_strings(base=0)                                                 # ["0", "0", "1"]

A call is one UmiAssigner::assign of the reference; a position group's orientation sub-groups are separate calls
of one group.  UMIs are what umi_for_read made of the read's tag (`umi_for_read` below).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence, Union

import numpy as np

from . import lib as _l

STRATEGIES = {"identity": _l.FGB_UMI_IDENTITY, "edit": _l.FGB_UMI_EDIT, "adjacency": _l.FGB_UMI_ADJACENCY,
              "paired": _l.FGB_UMI_PAIRED}
RULES = {"mapped": _l.FGB_UMI_RULES_MAPPED, "unmapped": _l.FGB_UMI_RULES_UNMAPPED}
KEY_DTYPE = np.dtype([("bits", "<u8"), ("str_off", "<u8"), ("str_len", "<u4"), ("count", "<u4"), ("first", "<u4"),
                      ("dash", "<u4"), ("len", "u1"), ("flags", "u1"), ("reserved", "u1", 6)])
assert KEY_DTYPE.itemsize == C.sizeof(_l.FgbUmiKey)

Umi = Union[str, bytes]


def _b(u: Umi) -> bytes:
    return u.encode() if isinstance(u, str) else bytes(u)


def options(strategy: str, edits: int, rules: str = "mapped", min_umi_length: Optional[int] = None,
            n_threads: int = 1) -> _l.FgbUmiOptions:
    return _l.FgbUmiOptions(STRATEGIES[strategy], edits, RULES[rules], min_umi_length or 0, n_threads, 0)


def pack_umis(umis: Sequence[Umi]):
    """UMIs -> (blob, off[n + 1])."""
    bs = [_b(u) for u in umis]
    off = np.zeros(len(bs) + 1, np.uint64)
    if bs:
        off[1:] = np.cumsum([len(b) for b in bs])
    blob = np.frombuffer(b"".join(bs) or b"\0", np.uint8).copy()
    return blob, off


def pack_groups(groups):
    """groups -> calls -> UMIs to the flat arrays fgb_umi_assign takes: (blob, umi_off, call_off, group_off)."""
    calls = [c for g in groups for c in g]
    blob, umi_off = pack_umis([u for c in calls for u in c])
    call_off = np.zeros(len(calls) + 1, np.uint64)
    call_off[1:] = np.cumsum([len(c) for c in calls])
    group_off = np.zeros(len(groups) + 1, np.uint64)
    group_off[1:] = np.cumsum([len(g) for g in groups])
    return blob, umi_off, call_off, group_off


@dataclass
class UmiAssignment:
    kinds: np.ndarray          # u8 per UMI: FGB_MOL_NONE / SINGLE / A / B
    ids: np.ndarray            # u64 per UMI, local to its group
    mi_counts: np.ndarray      # u64 per group: max(id) + 1
    group_of_umi: np.ndarray   # group index per UMI

    def mi_strings(self, base: int = 0):
        """MI values (lib.rs:79-98): N, N/A or N/B with N = id + base + the earlier groups' counts; "" for None."""
        gbase = base + np.concatenate([[0], np.cumsum(self.mi_counts, dtype=np.uint64)[:-1]]).astype(np.uint64)
        out = []
        for k, i, g in zip(self.kinds.tolist(), self.ids.tolist(), self.group_of_umi.tolist()):
            if k == _l.FGB_MOL_NONE:
                out.append("")
            else:
                n = str(i + int(gbase[g]))
                out.append(n + ("/A" if k == _l.FGB_MOL_A else "/B" if k == _l.FGB_MOL_B else ""))
        return out


class UmiAssigner:
    """fgb_umi_assign on one GPU.  rules="unmapped" gives `group --allow-unmapped`'s assigners."""

    def __init__(self, device: int = 0, strategy: str = "adjacency", edits: int = 1, rules: str = "mapped",
                 min_umi_length: Optional[int] = None, n_threads: int = 1):
        from .engine import Engine
        self.engine = Engine(device)
        self.opt = options(strategy, edits, rules, min_umi_length, n_threads)

    def close(self):
        self.engine.close()

    def assign_packed(self, blob, umi_off, call_off, group_off) -> UmiAssignment:
        lib = _l.load()
        n, nc, ng = len(umi_off) - 1, len(call_off) - 1, len(group_off) - 1
        ids = np.zeros(max(n, 1), np.uint64)
        kinds = np.zeros(max(n, 1), np.uint8)
        counts = np.zeros(max(ng, 1), np.uint64)
        umi_off = np.ascontiguousarray(umi_off, np.uint64)
        call_off = np.ascontiguousarray(call_off, np.uint64)
        group_off = np.ascontiguousarray(group_off, np.uint64)
        st = lib.fgb_umi_assign(self.engine._h, C.byref(self.opt), blob.ctypes.data, umi_off.ctypes.data, n,
                                call_off.ctypes.data, nc, group_off.ctypes.data, ng, ids.ctypes.data,
                                kinds.ctypes.data, counts.ctypes.data)
        self.engine._check(st, "fgb_umi_assign")
        calls_per_group = np.diff(group_off.astype(np.int64))
        umis_per_call = np.diff(call_off.astype(np.int64))
        group_of_call = np.repeat(np.arange(ng), calls_per_group)
        return UmiAssignment(kinds[:n], ids[:n], counts[:ng], np.repeat(group_of_call, umis_per_call))

    def edges(self, umis: Sequence[Umi]):
        """The capture lists the device finds for ONE call (fgb_umi_edges): a list of ascending key-index lists, keys
        in the order of the call's key table."""
        lib = _l.load()
        blob, off = pack_umis(umis)
        n = len(umis)
        eo = np.zeros(n + 1, np.uint64)
        nk, ne = C.c_uint64(), C.c_uint64()
        args = (self.engine._h, C.byref(self.opt), blob.ctypes.data, off.ctypes.data, n, C.byref(nk), eo.ctypes.data)
        self.engine._check(lib.fgb_umi_edges(*args, None, 0, C.byref(ne)), "fgb_umi_edges")
        e = np.zeros(max(ne.value, 1), np.uint32)
        self.engine._check(lib.fgb_umi_edges(*args, e.ctypes.data, ne.value, C.byref(ne)), "fgb_umi_edges")
        return [e[int(eo[k]):int(eo[k + 1])].tolist() for k in range(nk.value)]

    def last_timing(self):
        """ms of the last assign: host key tables, device phase (host clock), edge kernels (CUDA events), host rules."""
        ms = (C.c_double * 4)()
        self.engine._check(_l.load().fgb_umi_last_timing(self.engine._h, ms), "fgb_umi_last_timing")
        return dict(zip(("prepare_ms", "device_phase_ms", "kernels_ms", "resolve_ms"), list(ms)))

    def assign(self, groups) -> UmiAssignment:
        """groups: a list of position groups, each a list of calls, each a list of UMIs (str or bytes)."""
        return self.assign_packed(*pack_groups(groups))


def umi_for_read(umi: Umi, is_r1_earlier: bool, strategy: str, edits: int, rules: str = "mapped") -> bytes:
    """umi_for_read (group.rs:300-350) through the library."""
    lib = _l.load()
    u = _b(umi)
    o = options(strategy, edits, rules)
    out = C.create_string_buffer(len(u) + 2 * edits + 8)
    n = C.c_size_t()
    st = lib.fgb_host_umi_for_read(C.byref(o), u, len(u), int(is_r1_earlier), out, len(out), C.byref(n))
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_host_umi_for_read")
    return out.raw[:n.value]
