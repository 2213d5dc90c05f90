"""Host-side mirror of the consensus boundary over the C-ABI (include/fgumi_b200.h).

`Engine` owns one `fgb_handle` (one per GPU, like one caller per worker in the reference,
simplex.rs:574).  `PackedBatch` is the SoA batch the ABI consumes: base/qual byte columns with
per-read descriptors, per-unit descriptors and the tile table.  PyTorch is used only to hold
device memory and streams; every computation happens in libfgumi_b200.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import lib as _l

UNIT_DTYPE = np.dtype([("out_off", "<u8"), ("read_begin", "<u4"), ("cons_len", "<u4")])
TILE_DTYPE = np.dtype([("byte_begin", "<u8"), ("byte_len", "<u4"), ("unit_begin", "<u4"),
                       ("n_units", "<u4"), ("read_begin", "<u4"), ("n_reads", "<u4"),
                       ("flags", "<u4")])
DUPLEX_JOB_DTYPE = np.dtype([("unit_a", "<u4"), ("unit_b", "<u4"), ("out_off", "<u8")])
CODEC_JOB_DTYPE = np.dtype([("unit_a", "<u4"), ("unit_b", "<u4"), ("out_off", "<u8"),
                            ("len", "<u4"), ("pad_a_left", "<u4"), ("pad_b_left", "<u4"),
                            ("rc_a", "u1"), ("rc_b", "u1"), ("rc_out", "u1"), ("reserved0", "u1")])
assert UNIT_DTYPE.itemsize == 16 and TILE_DTYPE.itemsize == 32
assert DUPLEX_JOB_DTYPE.itemsize == 16 and CODEC_JOB_DTYPE.itemsize == 32


def _round_up(x, m):
    return (x + m - 1) // m * m


@dataclass
class VanillaUmiConsensusOptions:
    """vanilla_caller.rs:284-341 (defaults :322-341); CLI defaults are common.rs:225-249."""
    error_rate_pre_umi: int = 45
    error_rate_post_umi: int = 40
    min_input_base_quality: int = 10
    min_reads: int = 2
    max_reads: Optional[int] = None
    produce_per_base_tags: bool = True
    trim: bool = False
    min_consensus_base_quality: int = 40


@dataclass
class PackedBatch:
    """Host (numpy) form of fgb_batch."""
    bases: np.ndarray       # uint8, length padded to a multiple of 16
    quals: np.ndarray       # uint8, same length
    reads: np.ndarray       # uint64 descriptors (off << 16 | len), length padded to even
    units: np.ndarray       # UNIT_DTYPE, U+1 entries (sentinel last)
    n_units: int
    n_reads: int
    n_bytes: int
    n_out: int
    tiles: Optional[np.ndarray] = None   # TILE_DTYPE

    def unit_slices(self) -> List[slice]:
        u = self.units
        return [slice(int(u["out_off"][i]), int(u["out_off"][i]) + int(u["cons_len"][i]))
                for i in range(self.n_units)]


def consensus_length(lengths: Sequence[int], min_reads: int) -> int:
    """min_reads-th longest read, vanilla_caller.rs:1269-1277."""
    s = sorted(lengths, reverse=True)
    return s[min_reads - 1]


def pack_source_reads(units: Sequence[Sequence[Tuple[bytes, bytes]]], min_reads: int) -> PackedBatch:
    """Pack already-prepared SourceRead rows (bases, quals) per unit.  Small-scale packer used by
    tests; rows are padded to FGB_READ_ALIGN, outputs to FGB_OUT_ALIGN."""
    n_units = len(units)
    n_reads = sum(len(u) for u in units)
    reads = np.zeros(_round_up(n_reads, 2) + 2, dtype=np.uint64)
    uarr = np.zeros(n_units + 1, dtype=UNIT_DTYPE)
    chunks_b, chunks_q = [], []
    off = 0
    r = 0
    out = 0
    for i, unit in enumerate(units):
        uarr[i]["read_begin"] = r
        uarr[i]["out_off"] = out
        lens = []
        for (b, q) in unit:
            if len(b) != len(q):
                raise ValueError("bases/quals length mismatch")
            ln = len(b)
            if ln > _l.FGB_MAX_READ_LEN:     # the descriptor's low 16 bits; a longer row would spill into its offset
                raise ValueError(f"a row of {ln} bases is longer than FGB_MAX_READ_LEN ({_l.FGB_MAX_READ_LEN})")
            lens.append(ln)
            reads[r] = (off << 16) | ln
            pad = _round_up(ln, _l.FGB_READ_ALIGN) - ln
            chunks_b.append(np.frombuffer(bytes(b) + b"\0" * pad, dtype=np.uint8))
            chunks_q.append(np.frombuffer(bytes(q) + b"\0" * pad, dtype=np.uint8))
            off += ln + pad
            r += 1
        cl = consensus_length(lens, min_reads) if len(lens) >= max(1, min_reads) else 0
        uarr[i]["cons_len"] = cl
        out += _round_up(cl, _l.FGB_OUT_ALIGN)
    uarr[n_units]["read_begin"] = r
    uarr[n_units]["out_off"] = out
    n_bytes = off
    tot = _round_up(max(n_bytes, 1), 16)
    bases = np.zeros(tot, dtype=np.uint8)
    quals = np.zeros(tot, dtype=np.uint8)
    if chunks_b:
        bases[:n_bytes] = np.concatenate(chunks_b)
        quals[:n_bytes] = np.concatenate(chunks_q)
    return PackedBatch(bases, quals, reads, uarr, n_units, n_reads, n_bytes, out)


def pack_uniform(bases: np.ndarray, quals: np.ndarray, min_reads: int = 1) -> PackedBatch:
    """Pack a dense [U, D, L] uint8 pileup (fixed depth D, fixed length L) — vectorised."""
    U, D, L = bases.shape
    Lp = _round_up(L, _l.FGB_READ_ALIGN)
    bp = np.zeros((U, D, Lp), dtype=np.uint8)
    qp = np.zeros((U, D, Lp), dtype=np.uint8)
    bp[:, :, :L] = bases
    qp[:, :, :L] = quals
    n_reads = U * D
    n_bytes = n_reads * Lp
    tot = _round_up(max(n_bytes, 1), 16)
    fb = np.zeros(tot, dtype=np.uint8)
    fq = np.zeros(tot, dtype=np.uint8)
    fb[:n_bytes] = bp.reshape(-1)
    fq[:n_bytes] = qp.reshape(-1)
    reads = np.zeros(_round_up(n_reads, 2) + 2, dtype=np.uint64)
    reads[:n_reads] = (np.arange(n_reads, dtype=np.uint64) * np.uint64(Lp) << np.uint64(16)) | np.uint64(L)
    Lo = _round_up(L, _l.FGB_OUT_ALIGN)
    uarr = np.zeros(U + 1, dtype=UNIT_DTYPE)
    uarr["read_begin"] = np.arange(U + 1, dtype=np.uint32) * D
    uarr["out_off"] = np.arange(U + 1, dtype=np.uint64) * Lo
    uarr["cons_len"][:U] = L if D >= min_reads else 0
    return PackedBatch(fb, fq, reads, uarr, U, n_reads, n_bytes, U * Lo)


RAW_READ_DTYPE = np.dtype([("src_off", "<u8"), ("raw_len", "<u4"), ("flags", "<u4")])
assert RAW_READ_DTYPE.itemsize == 16
_NIBBLE = np.full(256, 15, dtype=np.uint8)
for _i, _c in enumerate(b"=ACMGRSVTWYHKDBN"):
    _NIBBLE[_c] = _i
    _NIBBLE[ord(chr(_c).lower())] = _i


@dataclass
class RawColumns:
    """fgb_raw_columns: the records' 4-bit sequence + raw qualities, and one fgb_raw_read per row."""
    seq4: np.ndarray
    quals_raw: np.ndarray
    raw_reads: np.ndarray
    n_raw: int
    min_input_base_quality: int

    def struct(self) -> "_l.FgbRawColumns":
        return _l.FgbRawColumns(self.n_raw, self.seq4.ctypes.data, self.quals_raw.ctypes.data,
                                self.raw_reads.ctypes.data, self.min_input_base_quality)


def pack_raw_reads(units, min_reads: int, min_input_base_quality: int):
    """units: [[(seq ASCII bytes, raw quals bytes, reverse: bool, row_len: int), ...], ...] where
    (seq, quals) is the KEPT raw span of the record and row_len the SourceRead length the host
    computed (vanilla_caller.rs:899-927).  Returns (layout PackedBatch without columns, RawColumns)."""
    lens = [[r[3] for r in u] for u in units]
    layout = pack_source_reads([[(b"\0" * n, b"\0" * n) for n in ul] for ul in lens], min_reads)
    layout.bases = None
    layout.quals = None
    R = layout.n_reads
    rr = np.zeros(R + 1, dtype=RAW_READ_DTYPE)
    seqs, quals = [], []
    off = 0
    k = 0
    for u in units:
        for seq, q, rev, _ in u:
            n = len(seq)
            assert len(q) == n
            rr[k] = (off, n, 1 if rev else 0)
            pad = (-n) % 8                       # spans start on even (here 8-aligned) indices
            seqs.append(np.frombuffer(seq, np.uint8)); quals.append(np.frombuffer(q, np.uint8))
            if pad:
                seqs.append(np.zeros(pad, np.uint8)); quals.append(np.zeros(pad, np.uint8))
            off += n + pad
            k += 1
    allseq = np.concatenate(seqs) if seqs else np.zeros(0, np.uint8)
    allq = np.concatenate(quals) if quals else np.zeros(0, np.uint8)
    nib = _NIBBLE[allseq]
    if nib.size % 2:
        nib = np.concatenate([nib, np.zeros(1, np.uint8)])
    seq4 = ((nib[0::2] << 4) | nib[1::2]).astype(np.uint8)
    seq4 = np.concatenate([seq4, np.zeros(32, np.uint8)])
    allq = np.concatenate([allq, np.zeros(32, np.uint8)])
    return layout, RawColumns(seq4, allq, rr, off, min_input_base_quality)


def pack8_encode(bases: np.ndarray, quals: np.ndarray) -> Optional[np.ndarray]:
    """fgb_pack8_encode over a (bases, quals) column pair; None when the batch is not encodable
    (IUPAC / lower-case bases, N with a quality other than 2, quality above 61)."""
    lib = _l.load()
    n = int(bases.size)
    out = np.empty(n, dtype=np.uint8)
    st = lib.fgb_pack8_encode(bases.ctypes.data, quals.ctypes.data, n, out.ctypes.data)
    if st == _l.FGB_ERR_NOT_ENCODABLE:
        return None
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_pack8_encode")
    return out


def plan_tiles(batch: PackedBatch) -> np.ndarray:
    """fgb_plan_tiles: greedy segmentation of the batch into shared-memory tiles."""
    lib = _l.load()
    n = C.c_uint64(0)
    up = batch.units.ctypes.data_as(C.c_void_p)
    rp = batch.reads.ctypes.data_as(C.c_void_p)
    st = lib.fgb_plan_tiles(up, batch.n_units, rp, batch.n_reads, None, 0, C.byref(n))
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_plan_tiles")
    tiles = np.zeros(max(int(n.value), 1), dtype=TILE_DTYPE)
    st = lib.fgb_plan_tiles(up, batch.n_units, rp, batch.n_reads, tiles.ctypes.data_as(C.c_void_p),
                            int(n.value), C.byref(n))
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_plan_tiles")
    batch.tiles = tiles[: int(n.value)]
    return batch.tiles


TILE_JOBS_DTYPE = np.dtype([("begin", "<u4"), ("count", "<u2"), ("max_items", "<u2")])


def plan_tiles_jobs(batch: PackedBatch, jobs: np.ndarray):
    """fgb_plan_tiles_jobs: tiles (class-sorted) that keep a duplex job's two units together, plus the per-tile job
    lists the vote kernels' duplex epilogue runs.  Returns (tiles, class_tiles, tile_jobs, job_index, n_attached);
    `batch.tiles` is left alone (the returned tiles are in class order, not unit order)."""
    lib = _l.load()
    jobs = np.ascontiguousarray(jobs)
    n = C.c_uint64(0)
    na = C.c_uint64(0)
    up = batch.units.ctypes.data_as(C.c_void_p)
    rp = batch.reads.ctypes.data_as(C.c_void_p)
    jp = jobs.ctypes.data_as(C.c_void_p)
    st = lib.fgb_plan_tiles_jobs(up, batch.n_units, rp, batch.n_reads, jp, len(jobs), None, 0, C.byref(n),
                                 None, None, None, None)
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_plan_tiles_jobs")
    nt = int(n.value)
    tiles = np.zeros(max(nt, 1), dtype=TILE_DTYPE)
    tile_jobs = np.zeros(max(nt, 1), dtype=TILE_JOBS_DTYPE)
    job_index = np.zeros(max(len(jobs), 1), dtype=np.uint32)
    counts = (C.c_uint64 * 3)()
    st = lib.fgb_plan_tiles_jobs(up, batch.n_units, rp, batch.n_reads, jp, len(jobs),
                                 tiles.ctypes.data_as(C.c_void_p), nt, C.byref(n), counts,
                                 tile_jobs.ctypes.data_as(C.c_void_p), job_index.ctypes.data_as(C.c_void_p),
                                 C.byref(na))
    if st != _l.FGB_OK:
        raise _l.FgbError(st, "fgb_plan_tiles_jobs")
    return tiles[:nt], (int(counts[0]), int(counts[1]), int(counts[2])), tile_jobs[:nt], job_index, int(na.value)


def sort_tiles_by_class(tiles: np.ndarray):
    """fgb_sort_tiles_by_class on a COPY of the tile table: (sorted tiles, run lengths per class).  For
    device-resident batches (fgb_vote_device); the host-buffer calls sort their chunks themselves."""
    lib = _l.load()
    out = np.ascontiguousarray(tiles).copy()
    counts = (C.c_uint64 * 3)()
    st = lib.fgb_sort_tiles_by_class(out.ctypes.data_as(C.c_void_p), len(out), counts)
    if st != 0:
        raise _l.FgbError(st, "fgb_sort_tiles_by_class")
    return out, (int(counts[0]), int(counts[1]), int(counts[2]))


@dataclass
class HostColumns:
    base: np.ndarray
    qual: np.ndarray
    depth: np.ndarray
    errors: np.ndarray

    @staticmethod
    def alloc(n_out: int) -> "HostColumns":
        n = max(n_out, 1)
        return HostColumns(np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint16),
                           np.zeros(n, np.uint16))


class DeviceBatch:
    """fgb_batch whose arrays are torch CUDA tensors (device-resident form)."""

    def __init__(self, batch: PackedBatch, device):
        import torch
        if batch.tiles is None:
            plan_tiles(batch)
        self.host = batch
        self.device = device
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(device)
        self.bases = t(batch.bases)
        self.quals = t(batch.quals)
        self.reads = t(batch.reads)
        self.units = t(batch.units)
        sorted_tiles, self.class_tiles = sort_tiles_by_class(batch.tiles)   # the host copy keeps the unit order
        self.tiles = t(sorted_tiles) if len(batch.tiles) else torch.zeros(32, dtype=torch.uint8, device=device)
        self.n_tiles = len(batch.tiles)

    def struct(self) -> _l.FgbBatch:
        b = self.host
        return _l.FgbBatch(b.n_units, b.n_reads, b.n_bytes, b.n_out, self.n_tiles,
                           self.bases.data_ptr(), self.quals.data_ptr(), self.reads.data_ptr(),
                           self.units.data_ptr(), self.tiles.data_ptr(), (C.c_uint64 * 3)(*self.class_tiles))


class DeviceColumns:
    def __init__(self, n_out: int, device):
        import torch
        n = max(n_out, 4)
        self.n_out = n_out
        self.base = torch.zeros(n, dtype=torch.uint8, device=device)
        self.qual = torch.zeros(n, dtype=torch.uint8, device=device)
        self.depth = torch.zeros(n, dtype=torch.int16, device=device)
        self.errors = torch.zeros(n, dtype=torch.int16, device=device)

    def struct(self) -> _l.FgbColumns:
        return _l.FgbColumns(self.base.data_ptr(), self.qual.data_ptr(), self.depth.data_ptr(),
                             self.errors.data_ptr())

    def to_host(self) -> HostColumns:
        n = self.n_out
        return HostColumns(self.base[:n].cpu().numpy(), self.qual[:n].cpu().numpy(),
                           self.depth[:n].cpu().numpy().view(np.uint16),
                           self.errors[:n].cpu().numpy().view(np.uint16))


class Engine:
    """One GPU's consensus engine (fgb_handle)."""

    def __init__(self, device: int = 0, error_rate_pre_umi: int = 45, error_rate_post_umi: int = 40,
                 min_reads: int = 1, min_consensus_base_quality: int = 2):
        self._lib = _l.load()
        self._h = C.c_void_p()
        p = _l.FgbParams(error_rate_pre_umi, error_rate_post_umi, min_consensus_base_quality, 0,
                         min_reads)
        st = self._lib.fgb_create(device, C.byref(p), C.byref(self._h))
        if st != _l.FGB_OK:
            self._h = C.c_void_p()
            raise _l.FgbError(st, "fgb_create")
        self.device = device
        self.min_reads = min_reads

    @classmethod
    def from_options(cls, opt: VanillaUmiConsensusOptions, device: int = 0) -> "Engine":
        return cls(device, opt.error_rate_pre_umi, opt.error_rate_post_umi, opt.min_reads,
                   opt.min_consensus_base_quality)

    def close(self):
        if self._h:
            self._lib.fgb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st: int, where: str):
        if st != _l.FGB_OK:
            buf = C.create_string_buffer(512)
            self._lib.fgb_last_error(self._h, buf, 512)
            raise _l.FgbError(st, where, buf.value.decode(errors="replace"))

    def tables(self):
        correct = np.zeros(94, np.float64)
        err_alt = np.zeros(94, np.float64)
        ln_pre = C.c_double()
        sq = np.zeros(94, np.uint8)
        self._check(self._lib.fgb_get_tables(self._h, correct.ctypes.data, err_alt.ctypes.data,
                                             C.addressof(ln_pre), sq.ctypes.data), "fgb_get_tables")
        return correct, err_alt, ln_pre.value, sq

    # ---- device-resident vote -----------------------------------------------------------------
    def vote_device(self, db: DeviceBatch, out: DeviceColumns, stream: Optional[int] = None):
        b = db.struct()
        c = out.struct()
        self._check(self._lib.fgb_vote_device(self._h, C.byref(b), C.byref(c),
                                              C.c_void_p(stream or 0)), "fgb_vote_device")

    # ---- host-buffer vote (what a ConsensusCaller implementation calls) -------------------------
    def submit(self, batch: PackedBatch, out: HostColumns):
        if batch.tiles is None:
            plan_tiles(batch)
        self._keep = (batch, out)
        b = _l.FgbBatch(batch.n_units, batch.n_reads, batch.n_bytes, batch.n_out, len(batch.tiles),
                        batch.bases.ctypes.data, batch.quals.ctypes.data, batch.reads.ctypes.data,
                        batch.units.ctypes.data, batch.tiles.ctypes.data)
        c = _l.FgbColumns(out.base.ctypes.data, out.qual.ctypes.data, out.depth.ctypes.data,
                          out.errors.ctypes.data)
        self._check(self._lib.fgb_submit(self._h, C.byref(b), C.byref(c)), "fgb_submit")

    def submit_pack8(self, batch: PackedBatch, packed: np.ndarray, out: HostColumns):
        """fgb_submit_pack8: `packed` is the one-byte-per-observation column of `batch`
        (see pack8_encode); half the host->device bytes of submit()."""
        if batch.tiles is None:
            plan_tiles(batch)
        self._keep = (batch, packed, out)
        b = _l.FgbBatch(batch.n_units, batch.n_reads, batch.n_bytes, batch.n_out, len(batch.tiles),
                        packed.ctypes.data, None, batch.reads.ctypes.data,
                        batch.units.ctypes.data, batch.tiles.ctypes.data)
        c = _l.FgbColumns(out.base.ctypes.data, out.qual.ctypes.data, out.depth.ctypes.data,
                          out.errors.ctypes.data)
        self._check(self._lib.fgb_submit_pack8(self._h, C.byref(b), C.byref(c)), "fgb_submit_pack8")

    def submit_bam4(self, layout: PackedBatch, raw: "RawColumns", out: HostColumns):
        """fgb_submit_bam4: rows are built on the device from the 4-bit sequence + raw qualities."""
        if layout.tiles is None:
            plan_tiles(layout)
        self._keep = (layout, raw, out)
        b = _l.FgbBatch(layout.n_units, layout.n_reads, layout.n_bytes, layout.n_out, len(layout.tiles),
                        None, None, layout.reads.ctypes.data, layout.units.ctypes.data,
                        layout.tiles.ctypes.data)
        c = _l.FgbColumns(out.base.ctypes.data, out.qual.ctypes.data, out.depth.ctypes.data,
                          out.errors.ctypes.data)
        r = raw.struct()
        self._check(self._lib.fgb_submit_bam4(self._h, C.byref(b), C.byref(r), C.byref(c)),
                    "fgb_submit_bam4")

    def submit_ex(self, batch: PackedBatch, out: HostColumns, packed: Optional[np.ndarray] = None,
                  raw: Optional["RawColumns"] = None, narrow: bool = False):
        """fgb_submit_ex: input format chosen by what is passed (packed -> PACK8, raw -> BAM4, else the
        two byte columns); narrow=True makes out.depth / out.errors uint8 columns."""
        if batch.tiles is None:
            plan_tiles(batch)
        self._keep = (batch, packed, raw, out)
        fmt = _l.FGB_IN_PACK8 if packed is not None else _l.FGB_IN_BAM4 if raw is not None else _l.FGB_IN_BYTES
        bases = packed.ctypes.data if packed is not None else (batch.bases.ctypes.data if fmt == _l.FGB_IN_BYTES else None)
        quals = batch.quals.ctypes.data if fmt == _l.FGB_IN_BYTES else None
        b = _l.FgbBatch(batch.n_units, batch.n_reads, batch.n_bytes, batch.n_out, len(batch.tiles),
                        bases, quals, batch.reads.ctypes.data, batch.units.ctypes.data,
                        batch.tiles.ctypes.data)
        if narrow:
            assert out.depth.dtype == np.uint8 and out.errors.dtype == np.uint8
        c = _l.FgbColumns(out.base.ctypes.data, out.qual.ctypes.data, out.depth.ctypes.data,
                          out.errors.ctypes.data)
        rs = raw.struct() if raw is not None else None
        o = _l.FgbSubmitOptions(fmt, _l.FGB_OUT_U8 if narrow else _l.FGB_OUT_U16,
                                C.cast(C.pointer(rs), C.c_void_p) if rs is not None else None)
        self._keep = self._keep + (rs,)
        self._check(self._lib.fgb_submit_ex(self._h, C.byref(b), C.byref(c), C.byref(o)), "fgb_submit_ex")

    def wait(self):
        self._check(self._lib.fgb_wait(self._h), "fgb_wait")
        self._keep = None

    def vote(self, batch: PackedBatch) -> HostColumns:
        out = HostColumns.alloc(batch.n_out)
        self.submit(batch, out)
        self.wait()
        return out

    # ---- strand combine -----------------------------------------------------------------------
    def duplex_combine_device(self, db: DeviceBatch, ss: DeviceColumns, jobs, n_jobs: int,
                              out_base, out_qual, out_errors, out_status, stream: Optional[int] = None):
        b = db.struct()
        c = ss.struct()
        o = _l.FgbDuplexOut(out_base.data_ptr(), out_qual.data_ptr(), out_errors.data_ptr(),
                            out_status.data_ptr() if out_status is not None else None)
        self._check(self._lib.fgb_duplex_combine_device(self._h, C.byref(b), C.byref(c),
                                                        C.c_void_p(jobs.data_ptr()), n_jobs,
                                                        C.byref(o), C.c_void_p(stream or 0)),
                    "fgb_duplex_combine_device")

    def vote_duplex_device(self, db, ss: DeviceColumns, jobs, n_jobs: int, tile_jobs, job_index,
                           out_base, out_qual, out_errors, out_status=None, stream: Optional[int] = None):
        """fgb_vote_duplex_device: the vote with the duplex combine in its epilogue.  `db` carries the tiles (and
        class_tiles) of plan_tiles_jobs; tile_jobs / job_index are device tensors of its tables."""
        b = db.struct()
        c = ss.struct()
        o = _l.FgbDuplexOut(out_base.data_ptr(), out_qual.data_ptr(), out_errors.data_ptr(),
                            out_status.data_ptr() if out_status is not None else None)
        self._check(self._lib.fgb_vote_duplex_device(self._h, C.byref(b), C.byref(c),
                                                     C.c_void_p(jobs.data_ptr()), n_jobs,
                                                     C.c_void_p(tile_jobs.data_ptr()),
                                                     C.c_void_p(job_index.data_ptr()),
                                                     C.byref(o), C.c_void_p(stream or 0)),
                    "fgb_vote_duplex_device")

    def codec_combine_device(self, db: DeviceBatch, ss: DeviceColumns, jobs, n_jobs: int,
                             params: _l.FgbCodecParams, out: DeviceColumns, status, disagreements=None,
                             duplex_bases=None, stream: Optional[int] = None):
        b = db.struct()
        c = ss.struct()
        o = _l.FgbCodecOut(out.struct(), status.data_ptr(),
                           disagreements.data_ptr() if disagreements is not None else None,
                           duplex_bases.data_ptr() if duplex_bases is not None else None)
        self._check(self._lib.fgb_codec_combine_device(self._h, C.byref(b), C.byref(c),
                                                       C.c_void_p(jobs.data_ptr()), n_jobs,
                                                       C.byref(params), C.byref(o),
                                                       C.c_void_p(stream or 0)),
                    "fgb_codec_combine_device")

    # ---- statistics ---------------------------------------------------------------------------
    def stats(self) -> dict:
        arr = (C.c_uint64 * _l.FGB_NCOUNTERS)()
        self._check(self._lib.fgb_stats(self._h, arr), "fgb_stats")
        return dict(zip(_l.COUNTER_NAMES, [int(x) for x in arr]))

    def stats_device_ptr(self) -> int:
        p = C.c_void_p()
        self._check(self._lib.fgb_stats_device_ptr(self._h, C.byref(p)), "fgb_stats_device_ptr")
        return int(p.value)

    def stats_reset(self):
        self._check(self._lib.fgb_stats_reset(self._h), "fgb_stats_reset")

    def launch_count(self) -> int:
        return int(self._lib.fgb_launch_count(self._h))
