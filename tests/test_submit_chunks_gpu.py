"""The host-buffer submit across many chunks, on the H100: every input format (two byte columns, PACK8, BAM4) and
output format (u16, u8), 1 MB and 3 MB chunks over one to four slot streams, pageable and page-locked host buffers,
the filter epilogue, slot buffers that grow in the middle of a submit, the documented layout errors of a later chunk,
the one-piece rule of combine jobs, and the benchmark's shape under the default chunk rule.

Every chunked run is compared with the CPU oracle at every position a unit owns, and with a one-chunk run of the same
batch (columns and engine counters); FGB_SUBMIT_TRACE's chunk count must equal the cuts tests/submit_chunks.py
predicts.  FGB_SUBMIT_CHUNK_MB / FGB_SUBMIT_SLOTS / FGB_SUBMIT_TRACE are read when an engine is created."""
import ctypes as C
import re

import numpy as np
import pytest

from tests import oracle_lib as O
from tests import submit_chunks as SC

pytestmark = pytest.mark.gpu

MB = SC.MB
MIN_READS = 2
TAIL = 64                      # sentinel elements behind every output column
SENT8, SENT16 = 0xA5, 0xA5A5


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as graft
    graft.build()
    import fgumi_b200
    return fgumi_b200


class Case:
    """One batch in one input format, its oracle columns and (filled lazily) its one-chunk run."""

    def __init__(self, fmt, batch, rows_batch=None, packed=None, raw=None, min_reads=MIN_READS):
        self.fmt, self.batch, self.packed, self.raw, self.min_reads = fmt, batch, packed, raw, min_reads
        self.oracle = O.simplex_batch(rows_batch, 45, 40, min_reads, 2, 8)[:4] if rows_batch is not None else None
        self.owned = owned_mask(batch)
        self.one = None


def owned_mask(batch) -> np.ndarray:
    cl = batch.units["cons_len"][: batch.n_units].astype(np.int64)
    oo = batch.units["out_off"][: batch.n_units].astype(np.int64)
    idx = np.repeat(oo - np.concatenate([[0], np.cumsum(cl)[:-1]]), cl) + np.arange(int(cl.sum()))
    m = np.zeros(batch.n_out, bool)
    m[idx] = True
    return m


@pytest.fixture(scope="module")
def cases(fg):
    out = {}
    b93 = fg.pack_source_reads(SC.mixed_units(12, qmax=93), MIN_READS)
    fg.plan_tiles(b93)
    out["bytes"] = Case(fg.lib.FGB_IN_BYTES, b93, b93)
    b61 = fg.pack_source_reads(SC.mixed_units(11), MIN_READS)
    fg.plan_tiles(b61)
    out["pack8"] = Case(fg.lib.FGB_IN_PACK8, b61, b61, packed=fg.pack8_encode(b61.bases, b61.quals))
    layout, raw, spans = SC.bam4_batch(fg, 5, MB)
    rows = fg.pack_source_reads(SC.expected_rows(spans, raw.min_input_base_quality), MIN_READS)
    assert np.array_equal(rows.units, layout.units)
    out["bam4"] = Case(fg.lib.FGB_IN_BAM4, layout, rows, raw=raw)
    out["bam4"].spans = spans
    return out


# ---- host buffers -------------------------------------------------------------------------------------------------
class Host:
    """numpy arrays in pageable memory, or in page-locked memory from fgb_host_alloc (freed by close())."""

    def __init__(self, fg, pinned: bool):
        self.lib, self.pinned, self.ptrs = fg.lib.load(), pinned, []

    def array(self, n, dtype, fill=0):
        dtype = np.dtype(dtype)
        if not self.pinned:
            return np.full(n, fill, dtype)
        p = C.c_void_p()
        assert self.lib.fgb_host_alloc(C.byref(p), max(n, 1) * dtype.itemsize) == 0
        self.ptrs.append(p.value)
        assert self.lib.fgb_host_is_pinned(p) == 1
        a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(n, 1) * dtype.itemsize,))
        a = a.view(dtype)[:n]
        a[:] = fill
        return a

    def copy(self, x):
        if x is None:
            return None
        a = self.array(x.size, x.dtype)
        a[:] = x
        return a

    def close(self):
        for p in self.ptrs:
            self.lib.fgb_host_free(p)
        self.ptrs = []


def out_columns(host, n_out, narrow):
    n = n_out + TAIL
    w, s = (np.uint8, SENT8) if narrow else (np.uint16, SENT16)
    return [host.array(n, np.uint8, SENT8), host.array(n, np.uint8, SENT8), host.array(n, w, s), host.array(n, w, s)]


def submit_ex(fg, eng, case, host, narrow, filt=None, status=None, masked=None, raw=None):
    """fgb_submit_ex of `case` from buffers in `host`; returns (outputs, inputs) -- the inputs to be checked after the
    wait.  `raw` replaces the case's raw columns (BAM4)."""
    lib = eng._lib
    b = case.batch
    fmt = case.fmt
    ins = dict(reads=host.copy(b.reads), units=host.copy(b.units), tiles=host.copy(b.tiles))
    if fmt == fg.lib.FGB_IN_BYTES:
        ins["bases"], ins["quals"] = host.copy(b.bases), host.copy(b.quals)
    elif fmt == fg.lib.FGB_IN_PACK8:
        ins["bases"], ins["quals"] = host.copy(case.packed), None
    else:
        ins["bases"] = ins["quals"] = None
        raw = raw if raw is not None else case.raw
        ins["seq4"], ins["qraw"], ins["rr"] = host.copy(raw.seq4), host.copy(raw.quals_raw), host.copy(raw.raw_reads)
    ptr = lambda a: a.ctypes.data if a is not None else None
    bs = fg.lib.FgbBatch(b.n_units, b.n_reads, b.n_bytes, b.n_out, len(b.tiles), ptr(ins["bases"]), ptr(ins["quals"]),
                         ptr(ins["reads"]), ptr(ins["units"]), ptr(ins["tiles"]))
    out = out_columns(host, b.n_out, narrow)
    cs = fg.lib.FgbColumns(*[o.ctypes.data for o in out])
    o = fg.lib.FgbSubmitOptions()
    o.input_format = fmt
    o.output_format = fg.lib.FGB_OUT_U8 if narrow else fg.lib.FGB_OUT_U16
    keep = [bs, cs, o]
    if fmt == fg.lib.FGB_IN_BAM4:
        rs = fg.lib.FgbRawColumns(raw.n_raw, ptr(ins["seq4"]), ptr(ins["qraw"]), ptr(ins["rr"]), raw.min_input_base_quality)
        o.raw = C.cast(C.pointer(rs), C.c_void_p)
        keep.append(rs)
    if filt is not None:
        o.filter = C.cast(C.pointer(filt), C.c_void_p)
        o.unit_status, o.unit_masked = status.ctypes.data, masked.ctypes.data
    saved = {k: v.copy() for k, v in ins.items() if v is not None}
    eng._keep = (keep, ins, out)
    eng._check(lib.fgb_submit_ex(eng._h, C.byref(bs), C.byref(cs), C.byref(o)), "fgb_submit_ex")
    return out, ins, saved


def engine(fg, monkeypatch, chunk_mb, slots, min_reads=MIN_READS):
    if chunk_mb:
        monkeypatch.setenv("FGB_SUBMIT_CHUNK_MB", str(chunk_mb))
    else:
        monkeypatch.delenv("FGB_SUBMIT_CHUNK_MB", raising=False)
    monkeypatch.setenv("FGB_SUBMIT_SLOTS", str(slots))
    monkeypatch.setenv("FGB_SUBMIT_TRACE", "1")
    return fg.Engine(0, 45, 40, min_reads, 2)


def n_chunks(trace: str) -> int:
    return len(set(re.findall(r"^\s+chunk (\d+)\s", trace, re.M)))


def run(fg, case, monkeypatch, capfd, chunk_mb, slots, narrow, pinned, **kw):
    """One fresh engine, one submit + wait; returns (columns as u16 where widened, stats, chunks traced)."""
    eng = engine(fg, monkeypatch, chunk_mb, slots, case.min_reads)
    host = Host(fg, pinned)
    try:
        capfd.readouterr()
        out, ins, saved = submit_ex(fg, eng, case, host, narrow, **kw)
        eng.wait()
        trace = capfd.readouterr().err
        n = case.batch.n_out
        for k, v in saved.items():                        # the inputs are never written
            assert np.array_equal(ins[k], v), k
        for col in out:                                   # the tails behind n_out come back untouched
            assert (col[n:] == (SENT8 if col.dtype == np.uint8 else SENT16)).all()
        cols = [out[0][:n].copy(), out[1][:n].copy(), out[2][:n].astype(np.uint16), out[3][:n].astype(np.uint16)]
        return cols, eng.stats(), n_chunks(trace)
    finally:
        host.close()
        eng.close()


def assert_owned_equal(got, want, owned, what):
    for k, name in enumerate(("base", "qual", "depth", "errors")):
        g, w = got[k][owned], want[k][owned].astype(got[k].dtype)
        bad = np.flatnonzero(g != w)
        assert bad.size == 0, f"{what}: {bad.size} {name} positions differ, first at owned index {bad[:5]}"


def one_chunk(fg, case, monkeypatch, capfd):
    if case.one is None:
        cols, st, n = run(fg, case, monkeypatch, capfd, None, 2, False, False)
        assert n == 1 == len(SC.cuts(case.batch, SC.default_chunk_bytes(case.batch.n_bytes)))
        assert_owned_equal(cols, case.oracle, case.owned, "one chunk vs oracle")
        case.one = (cols, st)
    return case.one


# ---- the format matrix --------------------------------------------------------------------------------------------
# the full product at 1 MB for one and three slots (page-locked buffers with three), spot cases at 3 MB and at 1 MB
# with two and four slots
MATRIX = ([(f, narrow, 1, slots, slots == 3) for f in ("bytes", "pack8", "bam4") for narrow in (False, True)
           for slots in (1, 3)] +
          [("bytes", False, 3, 2, False), ("pack8", True, 3, 4, True), ("bam4", True, 3, 2, True),
           ("bam4", False, 3, 4, False), ("pack8", False, 1, 2, False), ("bytes", True, 1, 4, True),
           ("bam4", True, 1, 4, False)])


@pytest.mark.parametrize("fmt,narrow,chunk_mb,slots,pinned", MATRIX)
def test_chunked_submit_matches_oracle_and_one_chunk(fg, cases, fmt, narrow, chunk_mb, slots, pinned, monkeypatch,
                                                      capfd):
    case = cases[fmt]
    one_cols, one_stats = one_chunk(fg, case, monkeypatch, capfd)
    cols, st, n = run(fg, case, monkeypatch, capfd, chunk_mb, slots, narrow, pinned)
    want_chunks = len(SC.cuts(case.batch, chunk_mb * MB))
    assert n == want_chunks and n > 1
    assert_owned_equal(cols, case.oracle, case.owned, "chunked vs oracle")
    assert_owned_equal(cols, one_cols, case.owned, "chunked vs one chunk")
    assert st == one_stats


def test_bam4_min_quality_branches_across_chunks(fg, cases, monkeypatch, capfd):
    """min_input_base_quality 0 (no mask) and 200 (the words kernel's branch above 127) over the same spans."""
    case = cases["bam4"]
    for min_q in (0, 200):
        raw = SC.with_min_q(case.raw, min_q)
        rows = fg.pack_source_reads(SC.expected_rows(case.spans, min_q), MIN_READS)
        want = O.simplex_batch(rows, 45, 40, MIN_READS, 2, 8)[:4]
        eng = engine(fg, monkeypatch, 1, 2)
        host = Host(fg, False)
        out, _, _ = submit_ex(fg, eng, case, host, False, raw=raw)
        eng.wait()
        cols = [c[: case.batch.n_out] for c in out]
        assert_owned_equal(cols, want, case.owned, f"bam4 min_q {min_q}")
        eng.close()


# ---- the filter epilogue ------------------------------------------------------------------------------------------
def filter_params(fg):
    p = SC.FILTER
    return fg.lib.FgbFilterParams(p["min_reads"], p["min_base_quality"], p["max_read_error_rate"],
                                  p["max_base_error_rate"], p["min_mean_base_quality"], p["max_no_call_fraction"],
                                  p["per_base_tags"])


@pytest.mark.parametrize("fmt", ["bytes", "pack8"])
def test_filter_epilogue_across_chunks(fg, cases, fmt, monkeypatch, capfd):
    """unit_status / unit_masked land at each chunk's units: equal to fgb_vote_device + fgb_filter_simplex_device on
    the whole batch, every status value among them."""
    import torch
    case = cases[fmt]
    b = case.batch
    fp = filter_params(fg)
    eng = engine(fg, monkeypatch, None, 2, MIN_READS)
    db = fg.DeviceBatch(b, "cuda:0")
    dc = fg.DeviceColumns(b.n_out, "cuda:0")
    s = torch.cuda.current_stream().cuda_stream
    eng.vote_device(db, dc, s)
    d_status = torch.full((b.n_units,), 77, dtype=torch.uint8, device="cuda:0")
    d_masked = torch.zeros(b.n_units, dtype=torch.int32, device="cuda:0")
    bs, cs = db.struct(), dc.struct()
    assert eng._lib.fgb_filter_simplex_device(eng._h, C.byref(bs), C.byref(cs), C.byref(fp),
                                              C.c_void_p(d_status.data_ptr()), C.c_void_p(d_masked.data_ptr()),
                                              C.c_void_p(s)) == 0
    torch.cuda.synchronize()
    want = dc.to_host()
    want_status, want_masked = d_status.cpu().numpy(), d_masked.cpu().numpy().view(np.uint32)
    eng.close()
    assert set(want_status.tolist()) == {0, 1, 2, 3, 4, 255}
    for slots, pinned in ((1, False), (3, True)):
        eng = engine(fg, monkeypatch, 1, slots, MIN_READS)
        host = Host(fg, pinned)
        status = host.array(b.n_units + TAIL, np.uint8, SENT8)
        masked = host.array(b.n_units + TAIL, np.uint32, 0xA5A5A5A5)
        capfd.readouterr()
        out, _, _ = submit_ex(fg, eng, case, host, False, filt=fp, status=status, masked=masked)
        eng.wait()
        assert n_chunks(capfd.readouterr().err) == len(SC.cuts(b, MB)) > 1
        assert np.array_equal(status[: b.n_units], want_status)
        assert np.array_equal(masked[: b.n_units], want_masked)
        assert (status[b.n_units:] == SENT8).all() and (masked[b.n_units:] == 0xA5A5A5A5).all()
        cols = [c[: b.n_out] for c in out]
        assert_owned_equal(cols, (want.base, want.qual, want.depth, want.errors), case.owned, f"filtered, {slots} slots")
        st = eng.stats()
        assert st["filter_records"] == int((want_status != 255).sum())
        assert st["filter_passed"] == int((want_status == 0).sum())
        assert st["filter_bases_masked"] == int(want_masked.sum())
        host.close()
        eng.close()


# ---- one engine, batches of changing size and format ----------------------------------------------------------------
def test_slot_buffers_grow_and_are_reused(fg, cases, monkeypatch, capfd):
    """small -> large -> small -> large -> small on one handle, alternating formats: slot buffers grow in the middle
    of a submit (a later chunk larger than every earlier one of its slot) and the tile staging vector is reused."""
    small = {}
    for k, n_units in (("pack8", 300), ("bytes", 400)):
        units = SC.mixed_units(40 + n_units, n_regular=n_units, big=None)
        b = fg.pack_source_reads(units, MIN_READS)
        fg.plan_tiles(b)
        packed = fg.pack8_encode(b.bases, b.quals) if k == "pack8" else None
        small[k] = Case(cases[k].fmt, b, b, packed=packed)
        assert len(SC.cuts(b, MB)) == 1
    seq = [small["pack8"], cases["bam4"], small["bytes"], cases["pack8"], small["pack8"], cases["bytes"], cases["bam4"]]
    eng = engine(fg, monkeypatch, 1, 2)
    host = Host(fg, False)
    try:
        for i, case in enumerate(seq):
            out, _, _ = submit_ex(fg, eng, case, host, i % 2 == 1)
            eng.wait()
            cols = [c[: case.batch.n_out].astype(np.uint16) if c.dtype == np.uint8 and j >= 2 else c[: case.batch.n_out]
                    for j, c in enumerate(out)]
            assert_owned_equal(cols, case.oracle, case.owned, f"step {i}")
    finally:
        host.close()
        eng.close()


# ---- documented status paths --------------------------------------------------------------------------------------
def test_bam4_layout_errors_in_a_later_chunk(fg, cases, monkeypatch, capfd):
    """A span that leaves its chunk's resident range fails fgb_wait; a span past n_raw fails the submit call itself.
    After either, the next submit on the handle is exact."""
    case = cases["bam4"]
    cs = SC.cuts(case.batch, MB, raw_reads=case.raw.raw_reads)
    eng = engine(fg, monkeypatch, 1, 2)
    host = Host(fg, False)
    try:
        # (1) a read in the middle of chunk 3 whose span runs past the chunk's resident range (but not past n_raw)
        c = cs[3]
        r = (c["rf"] + c["r1"]) // 2
        rr = case.raw.raw_reads.copy()
        rr["raw_len"][r] = c["raw_hi"] - int(rr["src_off"][r]) + 2
        assert int(rr["src_off"][r]) + int(rr["raw_len"][r]) <= case.raw.n_raw
        bad = type(case.raw)(case.raw.seq4, case.raw.quals_raw, rr, case.raw.n_raw, case.raw.min_input_base_quality)
        submit_ex(fg, eng, case, host, False, raw=bad)
        with pytest.raises(fg.lib.FgbError) as ei:
            eng.wait()
        assert ei.value.status == fg.lib.FGB_ERR_LAYOUT
        out, _, _ = submit_ex(fg, eng, case, host, True)
        eng.wait()
        assert_owned_equal([x[: case.batch.n_out].astype(np.uint16) if j >= 2 else x[: case.batch.n_out]
                            for j, x in enumerate(out)], case.oracle, case.owned, "after a bad span")
        # (2) the last read of chunk 2 runs past n_raw: the host's check refuses the submit
        c = cs[2]
        rr = case.raw.raw_reads.copy()
        r = c["r1"] - 1
        rr["raw_len"][r] = case.raw.n_raw - int(rr["src_off"][r]) + 2
        bad = type(case.raw)(case.raw.seq4, case.raw.quals_raw, rr, case.raw.n_raw, case.raw.min_input_base_quality)
        with pytest.raises(fg.lib.FgbError) as ei:
            submit_ex(fg, eng, case, host, False, raw=bad)
        assert ei.value.status == fg.lib.FGB_ERR_LAYOUT
        out, _, _ = submit_ex(fg, eng, case, host, False)
        eng.wait()
        assert_owned_equal([x[: case.batch.n_out] for x in out], case.oracle, case.owned, "after a refused submit")
    finally:
        host.close()
        eng.close()


# ---- the one-piece rule -------------------------------------------------------------------------------------------
def _combine_submit(fg, eng, batch, opt_setup):
    out = fg.HostColumns.alloc(batch.n_out)
    bs = fg.lib.FgbBatch(batch.n_units, batch.n_reads, batch.n_bytes, batch.n_out, len(batch.tiles),
                         batch.bases.ctypes.data, batch.quals.ctypes.data, batch.reads.ctypes.data,
                         batch.units.ctypes.data, batch.tiles.ctypes.data)
    cs = fg.lib.FgbColumns(out.base.ctypes.data, out.qual.ctypes.data, out.depth.ctypes.data, out.errors.ctypes.data)
    o = fg.lib.FgbSubmitOptions()
    o.input_format, o.output_format = fg.lib.FGB_IN_BYTES, fg.lib.FGB_OUT_U16
    keep = opt_setup(o)
    eng._check(eng._lib.fgb_submit_ex(eng._h, C.byref(bs), C.byref(cs), C.byref(o)), "fgb_submit_ex")
    eng.wait()
    del keep
    return out


def test_duplex_jobs_run_as_one_piece(fg, monkeypatch, capfd):
    from tests.test_combine_parity import _duplex_molecules
    L = O.load()
    rng = np.random.default_rng(61)
    units, pairs = _duplex_molecules(rng, 700, depth_hi=8, len_lo=100, len_hi=300)
    batch = fg.pack_source_reads(units, 1)
    fg.plan_tiles(batch)
    assert batch.n_bytes > 2 * MB and len(SC.cuts(batch, MB)) > 1
    cons_len, out_off = batch.units["cons_len"], batch.units["out_off"]
    jobs = np.zeros(len(pairs), dtype=fg.DUPLEX_JOB_DTYPE)
    off = 0
    for j, (ua, ub) in enumerate(pairs):
        jobs[j] = (ua, ub, off)
        off += (max(int(cons_len[ua]), int(cons_len[ub])) + 7) // 8 * 8
    n_out = max(off, 8)
    db, dq = np.zeros(n_out, np.uint8), np.zeros(n_out, np.uint8)
    de, ds = np.zeros(n_out, np.uint16), np.full(len(pairs), 77, np.uint8)
    dout = fg.lib.FgbDuplexOut(db.ctypes.data, dq.ctypes.data, de.ctypes.data, ds.ctypes.data)

    def setup(o):
        o.duplex_jobs, o.n_duplex_jobs, o.n_duplex_out = jobs.ctypes.data, len(pairs), n_out
        o.duplex_out = C.cast(C.pointer(dout), C.c_void_p)
        return dout
    eng = engine(fg, monkeypatch, 1, 2, 1)
    capfd.readouterr()
    ss = _combine_submit(fg, eng, batch, setup)
    assert n_chunks(capfd.readouterr().err) == 1 == len(SC.cuts(batch, MB, one_piece=True))
    eng.close()
    ob, oq, od, oe, _ = O.simplex_batch(batch, 45, 40, 1, 2, 8)
    assert_owned_equal([ss.base, ss.qual, ss.depth, ss.errors], (ob, oq, od, oe), owned_mask(batch), "duplex SS")
    seen = set()
    for j, (ua, ub) in enumerate(pairs):
        la, lb = int(cons_len[ua]), int(cons_len[ub])
        oa, obo = int(out_off[ua]), int(out_off[ub])
        rows = units[ua] + units[ub]
        keep = [np.frombuffer(r[0], np.uint8).copy() for r in rows]
        ptrs = (C.c_void_p * len(rows))(*[k.ctypes.data for k in keep])
        lens = (C.c_size_t * len(rows))(*[len(r[0]) for r in rows])
        cap = max(la, lb, 1)
        rb, rq, re_ = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8), np.zeros(cap, np.uint16)
        olen = C.c_size_t()
        st = L.orc_duplex_job(ob[oa:].ctypes.data, oq[oa:].ctypes.data, od[oa:].ctypes.data, oe[oa:].ctypes.data, la,
                              ob[obo:].ctypes.data, oq[obo:].ctypes.data, od[obo:].ctypes.data, oe[obo:].ctypes.data,
                              lb, ptrs, lens, len(rows), rb.ctypes.data, rq.ctypes.data, re_.ctypes.data,
                              C.addressof(olen))
        seen.add(st)
        assert ds[j] == st, j
        o, n = int(jobs[j]["out_off"]), olen.value
        assert np.array_equal(db[o:o + n], rb[:n]) and np.array_equal(dq[o:o + n], rq[:n]), j
        assert np.array_equal(de[o:o + n], re_[:n]), j
    assert seen == {0, 1, 2, 3}


def _codec_molecules(rng, n_mol):
    """R1 / R2 single-strand families of one molecule: four in five read the two strands of one template (the
    consensus length is the template's, so the strands line up), every fifth pairs unrelated templates; one in seven
    carries 15 % substitutions.  Returns (units, [(r1_negative, consensus length)])."""
    comp = np.arange(256, dtype=np.uint8)
    for a, b in zip(b"ACGT", b"TGCA"):
        comp[a] = b

    def strand(tmpl, depth, err):
        rows = []
        for _ in range(depth):
            b = tmpl.copy()
            m = rng.random(b.size) < err
            b[m] = SC.ACGT[rng.integers(0, 4, size=int(m.sum()))]
            q = rng.integers(5, 42, size=b.size).astype(np.uint8)
            n = rng.random(b.size) < 0.03
            b[n], q[n] = ord("N"), 2
            rows.append((b.tobytes(), q.tobytes()))
        return rows
    units, meta = [], []
    for m in range(n_mol):
        k, L = int(rng.integers(1, 7)), int(rng.integers(100, 300))
        err = 0.15 if m % 7 == 4 else 0.01
        tmpl = SC.ACGT[rng.integers(0, 4, size=L)]
        other = comp[tmpl[::-1]] if m % 5 != 2 else SC.ACGT[rng.integers(0, 4, size=L)]
        units += [strand(tmpl, k, err), strand(other, k, err)]
        meta.append((bool(rng.integers(0, 2)), L + (int(rng.integers(0, 30)) if m % 5 == 2 else 0)))
    return units, meta


def test_codec_jobs_run_as_one_piece(fg, monkeypatch, capfd):
    L = O.load()
    n_mol = 1500
    units, meta = _codec_molecules(np.random.default_rng(62), n_mol)
    batch = fg.pack_source_reads(units, 1)
    fg.plan_tiles(batch)
    assert batch.n_bytes > 2 * MB and len(SC.cuts(batch, MB)) > 1
    cons_len, out_off = batch.units["cons_len"], batch.units["out_off"]
    jobs = np.zeros(n_mol, dtype=fg.CODEC_JOB_DTYPE)
    off = 0
    for m, (r1_neg, clen) in enumerate(meta):
        la, lb = int(cons_len[2 * m]), int(cons_len[2 * m + 1])
        jobs[m]["unit_a"], jobs[m]["unit_b"], jobs[m]["out_off"], jobs[m]["len"] = 2 * m, 2 * m + 1, off, clen
        jobs[m]["rc_a"], jobs[m]["rc_b"], jobs[m]["rc_out"] = r1_neg, not r1_neg, r1_neg
        jobs[m]["pad_a_left"] = clen - la if r1_neg else 0
        jobs[m]["pad_b_left"] = clen - lb if not r1_neg else 0
        off += (clen + 7) // 8 * 8
    ss_q, outer_q, outer_len, max_dis, max_rate = 10, 5, 7, 40, 0.1
    cp = fg.lib.FgbCodecParams(ss_q, outer_q, outer_len, max_dis, max_rate)
    cb, cq = np.zeros(off, np.uint8), np.zeros(off, np.uint8)
    cd, ce = np.zeros(off, np.uint16), np.zeros(off, np.uint16)
    cst, cdis, cdup = np.full(n_mol, 255, np.uint8), np.zeros(n_mol, np.uint32), np.zeros(n_mol, np.uint32)
    cout = fg.lib.FgbCodecOut(fg.lib.FgbColumns(cb.ctypes.data, cq.ctypes.data, cd.ctypes.data, ce.ctypes.data),
                              cst.ctypes.data, cdis.ctypes.data, cdup.ctypes.data)

    def setup(o):
        o.codec_jobs, o.n_codec_jobs, o.n_codec_out = jobs.ctypes.data, n_mol, off
        o.codec_params = C.cast(C.pointer(cp), C.c_void_p)
        o.codec_out = C.cast(C.pointer(cout), C.c_void_p)
        return cp, cout
    eng = engine(fg, monkeypatch, 1, 3, 1)
    capfd.readouterr()
    _combine_submit(fg, eng, batch, setup)
    assert n_chunks(capfd.readouterr().err) == 1
    eng.close()
    ob, oq, od, oe, _ = O.simplex_batch(batch, 45, 40, 1, 2, 8)
    statuses = set()
    for m, (r1_neg, clen) in enumerate(meta):
        ua, ub = 2 * m, 2 * m + 1
        la, lb = int(cons_len[ua]), int(cons_len[ub])
        oa, obo = int(out_off[ua]), int(out_off[ub])
        rb, rq = np.zeros(clen, np.uint8), np.zeros(clen, np.uint8)
        rd, re_ = np.zeros(clen, np.uint16), np.zeros(clen, np.uint16)
        nb, nd = C.c_uint64(), C.c_uint64()
        rs = L.orc_codec_job(ob[oa:].ctypes.data, oq[oa:].ctypes.data, od[oa:].ctypes.data, oe[oa:].ctypes.data, la,
                             ob[obo:].ctypes.data, oq[obo:].ctypes.data, od[obo:].ctypes.data, oe[obo:].ctypes.data,
                             lb, int(r1_neg), int(not r1_neg), clen, ss_q, outer_q, outer_len, max_dis, max_rate,
                             rb.ctypes.data, rq.ctypes.data, rd.ctypes.data, re_.ctypes.data, C.addressof(nb),
                             C.addressof(nd))
        o = int(jobs[m]["out_off"])
        assert cst[m] == rs and cdis[m] == nd.value and cdup[m] == nb.value, m
        assert np.array_equal(cb[o:o + clen], rb) and np.array_equal(cq[o:o + clen], rq), m
        assert np.array_equal(cd[o:o + clen], rd) and np.array_equal(ce[o:o + clen], re_), m
        statuses.add(rs)
    assert statuses == {0, 1, 2}


# ---- the benchmark's shape ----------------------------------------------------------------------------------------
def test_bench_shape_default_chunks(fg, monkeypatch, capfd):
    """200 k depth-8 150 bp units from page-locked buffers under the default chunk rule (~30 MB chunks): PACK8 -> U8
    and BAM4 equal fgb_vote_device of the same batch everywhere, and the oracle on every unit of the tiles on either
    side of each chunk boundary plus a random sample."""
    import torch
    batch = SC.bench_batch()
    cs = SC.cuts(batch, SC.default_chunk_bytes(batch.n_bytes))
    assert len(cs) >= 8
    eng = engine(fg, monkeypatch, None, 2, 1)
    db = fg.DeviceBatch(batch, "cuda:0")
    dc = fg.DeviceColumns(batch.n_out, "cuda:0")
    eng.vote_device(db, dc, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = dc.to_host()
    del db, dc
    eng.close()
    owned = owned_mask(batch)
    sample = SC.boundary_units(batch, cs)
    sample = sorted(set(sample) | set(np.random.default_rng(3).choice(batch.n_units, 2000, replace=False).tolist()))
    sub = fg.pack_source_reads([SC.unit_rows(batch, u) for u in sample], 1)
    sb, sq, sd, se, _ = O.simplex_batch(sub, 45, 40, 1, 2, 8)
    for k, u in enumerate(sample):
        o, n, so = int(batch.units["out_off"][u]), int(batch.units["cons_len"][u]), int(sub.units["out_off"][k])
        for got, want in ((ref.base, sb), (ref.qual, sq), (ref.depth, sd), (ref.errors, se)):
            assert np.array_equal(got[o:o + n], want[so:so + n]), u
    nb = batch.n_bytes
    Lp = 152
    nib = SC._nibbles(batch.bases[:nb])
    seq4 = np.concatenate([(nib[0::2] << 4) | nib[1::2], np.zeros(32, np.uint8)])
    rr = np.zeros(batch.n_reads + 1, dtype=fg.RAW_READ_DTYPE)
    rr["src_off"][: batch.n_reads] = np.arange(batch.n_reads, dtype=np.uint64) * np.uint64(Lp)
    rr["raw_len"][: batch.n_reads] = 150
    raw = fg.RawColumns(seq4, batch.quals, rr, nb, 10)
    want = (ref.base, ref.qual, ref.depth, ref.errors)
    pack8 = Case(fg.lib.FGB_IN_PACK8, batch, packed=fg.pack8_encode(batch.bases, batch.quals), min_reads=1)
    bam4 = Case(fg.lib.FGB_IN_BAM4, batch, raw=raw, min_reads=1)
    for case, narrow in ((pack8, True), (bam4, False)):
        cols, st, n = run(fg, case, monkeypatch, capfd, None, 2, narrow, True)
        assert n == len(cs)
        assert_owned_equal(cols, want, owned, "bench shape")
        assert st["units"] == batch.n_units and st["positions"] == int(owned.sum())
