"""The one-warp fallback kernels of the filter (K4) and strand combines (K2 duplex, K3 CODEC), and the vote's pointer
checks.

The device entry points pick a kernel from how the caller's column pointers are aligned: 8-byte aligned byte columns
and 16-byte aligned u16 columns take the word kernels, anything else the fallback kernels (`filter_simplex_kernel`,
`duplex_combine_kernel`, `codec_combine_kernel`).  Buffers from an allocator are always aligned, so these tests pass
views into larger buffers: byte columns start 1..7 bytes and u16 columns 1..7 elements past an aligned address.
Each kernel is compared with a plain reference (the record oracle, the C++ oracle's duplex / CODEC combine), with
the word kernel on the same data and through the engine counters of both runs; bytes outside the rows a unit or job
owns must keep their fill.  The vote kernels cannot run on such pointers at all: fgb_vote_device and
fgb_vote_duplex_device refuse them with FGB_ERR_LAYOUT before anything is enqueued."""
import copy
import ctypes as C
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import record_oracle as R                      # noqa: E402
from tests import oracle_lib as O                           # noqa: E402
from tests.bam_builder import make_record                   # noqa: E402
from tests.test_combine_parity import (_UnitsOnly, _codec_job_mix, _codec_job_reference,   # noqa: E402
                                       _duplex_molecules, _family)

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
UNIT = np.dtype([("out_off", "<u8"), ("read_begin", "<u4"), ("cons_len", "<u4")])
FILL8, FILL16 = 0x55, 0x5555
NO_RECORD = 255


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as graft
    graft.build()
    import fgumi_b200
    return fgumi_b200


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _ptr_misaligned(t, align):
    return t.data_ptr() % align != 0


class _Cols:
    """Consensus columns of `n` elements as views into larger buffers filled with 0x55 / 0x5555: the byte columns start
    `sh8` bytes and the u16 columns `sh16` elements past an aligned allocation (0, 0 = the aligned form)."""

    def __init__(self, fg, n, sh8, sh16, depth=True):
        import torch
        self._fg, self.n, self.sh8, self.sh16 = fg, n, sh8, sh16
        self.raw8 = [torch.full((n + 16,), FILL8, dtype=torch.uint8, device=DEV) for _ in range(2)]
        self.raw16 = [torch.full((n + 16,), FILL16, dtype=torch.int16, device=DEV) for _ in range(2 if depth else 1)]
        self.base, self.qual = (r[sh8:sh8 + n] for r in self.raw8)
        v16 = [r[sh16:sh16 + n] for r in self.raw16]
        self.depth, self.errors = (v16[0], v16[1]) if depth else (None, v16[0])

    def load(self, base, qual, depth=None, errors=None):
        """Copies host arrays (or device tensors) of length n into the views."""
        import torch
        t = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(
            np.ascontiguousarray(a).view(np.int16 if a.dtype == np.uint16 else a.dtype))
        self.base.copy_(t(base)); self.qual.copy_(t(qual))
        if depth is not None:
            self.depth.copy_(t(depth))
        if errors is not None:
            self.errors.copy_(t(errors))

    def misaligned(self):
        ok8 = [not _ptr_misaligned(x, 8) for x in (self.base, self.qual)]
        ok16 = [not _ptr_misaligned(x, 16) for x in (self.depth, self.errors) if x is not None]
        return not all(ok8 + ok16)

    def struct(self):
        d = self.depth.data_ptr() if self.depth is not None else None
        return self._fg.lib.FgbColumns(self.base.data_ptr(), self.qual.data_ptr(), d, self.errors.data_ptr())

    def host_raw(self):
        """Whole buffers on the host: ([base, qual], [depth, errors]) with u16 views."""
        return ([r.cpu().numpy() for r in self.raw8], [r.cpu().numpy().view(np.uint16) for r in self.raw16])

    def host(self):
        b8, b16 = self.host_raw()
        v8 = [x[self.sh8:self.sh8 + self.n] for x in b8]
        v16 = [x[self.sh16:self.sh16 + self.n] for x in b16]
        return v8, v16

    def assert_fill_outside(self, owned):
        """Every element outside `owned` (bool[n], in view coordinates) still holds the fill."""
        b8, b16 = self.host_raw()
        for raw, sh, fill in [(x, self.sh8, FILL8) for x in b8] + [(x, self.sh16, FILL16) for x in b16]:
            keep = np.ones(len(raw), bool)
            keep[sh:sh + self.n] = ~owned
            bad = np.flatnonzero(raw[keep] != fill)
            assert bad.size == 0, ("written outside the owned rows", np.flatnonzero(keep)[bad[:8]] - sh)


# ============================ K4: the filter, both kernel forms ============================================
# Settings: (min_reads, min_base_quality, max_read_error_rate, max_base_error_rate, min_mean_base_quality,
# max_no_call_fraction, per_base_tags).  min_reads 70 000 is above every depth; -1 turns a gate off.
FILTER_GRID = [
    (2, 20, 0.1, 0.1, 30.0, 0.2, 1),
    (1, -1, 1 / 3, 0.25, 35.0, 1.0, 1),
    (0, 0, 0.7, 1 / 3, -1.0, 3.0, 1),
    (1, 10, 0.0, 0.0, 20.0, 0.25, 1),
    (70000, 255, 1.0, 0.1, 25.0, 0.5, 1),
    (1, 5, 0.1, 0.25, 30.0, 0.1, 0),
    (0, -1, 0.7, 0.25, -1.0, 1.0, 0),
]
_ACGT = np.frombuffer(b"ACGT", np.uint8)
_N = ord("N")


def _vote_like(rng, b, q, d, e):
    """What the vote emits: N with quality 2, no base without depth, no more errors than depth."""
    e = np.minimum(e, d)
    nocall = (b == _N) | (d == 0)
    b[nocall] = _N; q[nocall] = 2
    e[d == 0] = 0
    return b.astype(np.uint8), q.astype(np.uint8), d.astype(np.uint16), e.astype(np.uint16)


def _random_unit(rng, L):
    dmax = int(rng.choice([3, 12, 40, 300, 65535]))
    d = rng.integers(0 if rng.random() < 0.3 else 1, dmax + 1, L)
    escale = float(rng.choice([0.0, 0.05, 0.3, 0.6]))
    e = np.floor(d * rng.random(L) * escale).astype(np.int64)
    b = rng.choice(_ACGT, L)
    b[rng.random(L) < float(rng.choice([0.0, 0.03, 0.3]))] = _N
    lo = int(rng.choice([2, 20, 30]))
    q = rng.integers(lo, 94, L)
    return _vote_like(rng, b, q, d, e)


def _plain_unit(L, depth, qual, n_count=0):
    """Depth `depth`, no errors, quality `qual`, the first n_count bases N."""
    b = np.resize(_ACGT, L).copy()
    b[:n_count] = _N
    q = np.full(L, qual, np.int64)
    return _vote_like(None, b, q, np.full(L, depth, np.int64), np.zeros(L, np.int64))


def _filter_units(rng, p):
    """One batch of units for settings `p`: random units over the length classes plus units planted on every
    threshold of `p`."""
    min_reads, mbq, mre, mbe, min_mean, nc, tags = p
    rows = []
    # per-base error rate: e/d equal to, one error below and one above max_base_error_rate, at many depths (the
    # depths above 32767 are where the i16 clamp of cd / ce decides)
    ladder = [1, 2, 3, 4, 7, 10, 12, 20, 30, 99, 100, 255, 256, 300, 1000, 3000, 9999, 32766, 32767, 32768,
              40000, 50000, 65534, 65535]
    pos = []
    for d in ladder:
        e0 = int(Fraction(d) * Fraction(mbe))
        pos += [(d, e) for e in (e0 - 1, e0, e0 + 1) if 0 <= e <= d]
    pos = np.array(pos, np.int64)
    for k in range(0, len(pos), 24):
        L = len(pos[k:k + 24])
        rows.append(_vote_like(rng, rng.choice(_ACGT, L), rng.integers(40, 94, L), pos[k:k + 24, 0], pos[k:k + 24, 1]))
    # cE: te / td exactly max_read_error_rate (float32 rounds 1/10 and 1/3 up, 7/10 down), and 70000001 / 1e8 against
    # 0.7 (above it, but float32 rounds it to 0.7f < 0.7)
    fr = Fraction(mre).limit_denominator(100)
    rows.append(_vote_like(rng, rng.choice(_ACGT, 40), rng.integers(40, 94, 40), np.full(40, fr.denominator),
                           np.full(40, fr.numerator)))
    if mre == 0.7:
        L = 2000
        e = np.full(L, 35000); e[0] += 1
        rows.append(_vote_like(rng, rng.choice(_ACGT, L), rng.integers(40, 94, L), np.full(L, 50000), e))
    if mre == 0.0:
        e = np.zeros(30, np.int64); e[7] = 1
        rows.append(_vote_like(rng, rng.choice(_ACGT, 30), rng.integers(40, 94, 30), np.full(30, 9), e))
    # mean quality exactly at min_mean_base_quality and one quality step below it
    m = int(min_mean) if min_mean >= 0 else 30
    for L in (20, 37):
        rows.append(_plain_unit(L, 50, m))
        b, q, d, e = _plain_unit(L, 50, m)
        q[3] -= 1
        rows.append((b, q, d, e))
    # all-N units (non_n = 0), with and without depth
    rows.append(_plain_unit(15, 0, 2, 15))
    rows.append(_plain_unit(16, 6, 2, 16))
    # no-call gate exactly at the threshold and one N above it (fraction and count mode)
    if nc >= 1.0:
        for n in (int(nc), int(nc) + 1):
            rows.append(_plain_unit(30, 50, 60, n))
    else:
        for L in (20, 40, 100):
            n = int(Fraction(nc).limit_denominator(100) * L)
            rows.append(_plain_unit(L, 50, 60, n))
            rows.append(_plain_unit(L, 50, 60, n + 1))
    # several gates failing at once: shallow, error-rich, low quality and mostly N
    b, q, d, e = _plain_unit(60, 1, 5, 40)
    e[:] = d
    rows.append(_vote_like(rng, b, q, d, e))
    rows.append(_plain_unit(60, 50, 5, 40))
    # random units over the length classes (1-9, 255-257, 2047-2049, about 5000, empty) and enough of them for
    # several chunks of 256 units
    lengths = ([int(x) for x in rng.integers(1, 10, 40)] + [255, 256, 257, 2047, 2048, 2049, 4999, 5003] +
               [0] * 12 + [int(x) for x in rng.integers(10, 300, 300)])
    rng.shuffle(lengths)
    for L in lengths:
        rows.append(_random_unit(rng, L))
    order = rng.permutation(len(rows))
    return [rows[i] for i in order]


def _layout(rows):
    """Unit table (rows dense, each padded to 8) and the host columns, padding holding the fill."""
    units = np.zeros(len(rows) + 1, dtype=UNIT)
    off = 0
    for i, r in enumerate(rows):
        units[i]["out_off"] = off; units[i]["cons_len"] = len(r[0])
        off += (len(r[0]) + 7) // 8 * 8
    units[len(rows)]["out_off"] = off
    n = max(off, 8)
    cols = [np.full(n, FILL8, np.uint8), np.full(n, FILL8, np.uint8), np.full(n, FILL16, np.uint16),
            np.full(n, FILL16, np.uint16)]
    owned = np.zeros(n, bool)
    for i, r in enumerate(rows):
        o, L = int(units[i]["out_off"]), len(r[0])
        for c, x in zip(cols, r):
            c[o:o + L] = x
        owned[o:o + L] = True
    return units, cols, owned


def _filter_reference(rows, p, seen):
    """Each unit as the record the simplex caller writes, through the record oracle's filter.  Returns masked bases,
    qualities, status and masked count per unit; notes in `seen` which edges the batch reached."""
    min_reads, mbq, mre, mbe, min_mean, nc, tags = p
    th = R.FilterThresholds(min_reads, mre, mbe)
    min_bq = None if mbq < 0 else mbq
    min_mean_q = None if min_mean < 0 else min_mean
    out = []
    for b, q, d, e in rows:
        L = len(b)
        if L == 0:
            out.append((b, q, NO_RECORD, 0))
            seen.add("empty")
            continue
        td, te = int(d.astype(np.int64).sum()), int(e.astype(np.int64).sum())
        ce = float(np.float32(te) / np.float32(td)) if td else 0.0
        tag_list = [(b"cD", "S", int(d.max())), (b"cE", "f", ce)]
        dt, et = np.minimum(d, 32767).astype(np.int64), np.minimum(e, 32767).astype(np.int64)
        if tags:
            tag_list += [(b"cd", "Bs", [int(x) for x in dt]), (b"ce", "Bs", [int(x) for x in et])]
        rec = bytearray(make_record(name=b"u", flags=4, ref_id=-1, pos=-1, cigar=[], seq=b.tobytes(),
                                    quals=[int(x) for x in q], tags=tag_list))
        masked = R.mask_bases(rec, th, min_bq)
        v = R.Rec(bytes(rec))
        mb, mq = np.frombuffer(bytes(v.sequence()), np.uint8), np.array(list(v.quals()), np.uint8)
        n_count, mean = R.compute_read_stats(bytes(rec))
        st = R.filter_read(v.aux(), th)
        if st == R.FILTER_PASS and not R.check_no_call_and_quality(bytes(rec), min_mean_q, nc):
            st = 3 if (min_mean_q is not None and mean < min_mean_q) else 4
        out.append((mb, mq, st, masked))
        # which edges this unit reached
        seen.add(("status", st))
        if tags:
            for k in np.flatnonzero(dt > 0):
                r = float(et[k]) / float(dt[k])
                if r == mbe:
                    seen.add(("base_rate_eq", mbe, int(dt[k])))
                elif r > mbe and float(et[k] - 1) / float(dt[k]) <= mbe:
                    seen.add(("base_rate_above", mbe, int(dt[k])))
                elif r < mbe and float(et[k] + 1) / float(dt[k]) > mbe:
                    seen.add(("base_rate_below", mbe, int(dt[k])))
                if d[k] > 32767 and (float(e[k]) / float(d[k]) > mbe) != (r > mbe):
                    seen.add("clamp_decides")
        if td and (ce > mre) != (te / td > mre):
            seen.add(("ce_f32_fails" if ce > mre else "ce_f32_passes", mre))
        non_n = L - n_count
        qsum = sum(int(x) for x, y in zip(mq, mb) if y != _N)
        if non_n == 0:
            seen.add("all_n")
        elif min_mean_q is not None and st not in (1, 2):
            if qsum == min_mean_q * non_n:
                seen.add("mean_eq")
            elif qsum == min_mean_q * non_n - 1:
                seen.add("mean_one_below")
        if st not in (1, 2) and (min_mean_q is None or mean >= min_mean_q):
            if nc >= 1.0 and n_count == nc:
                seen.add(("nocall_count_eq", nc))
            elif nc < 1.0 and n_count / L == nc:
                seen.add("nocall_fraction_eq")
        fails = [int(d.max()) < min_reads, ce > mre, min_mean_q is not None and mean < min_mean_q,
                 (n_count > nc) if nc >= 1.0 else (n_count / L > nc)]
        if sum(fails) >= 2:
            seen.add(("several_gates", st))
    return out


def _run_filter(fg, eng, db, cols, fp, n_units):
    import torch
    status = torch.full((n_units,), 77, dtype=torch.uint8, device=DEV)
    masked = torch.full((n_units,), -1, dtype=torch.int32, device=DEV)
    b, c = db.struct(), cols.struct()
    eng.stats_reset()
    st = eng._lib.fgb_filter_simplex_device(eng._h, C.byref(b), C.byref(c), C.byref(fp), C.c_void_p(status.data_ptr()),
                                            C.c_void_p(masked.data_ptr()), C.c_void_p(_stream()))
    assert st == 0
    torch.cuda.synchronize()
    return status.cpu().numpy(), masked.cpu().numpy().view(np.uint32), eng.stats()


def filter_forms(fg, p, seed, seen, shifts=None):
    """One setting of the filter grid: the fallback kernel on misaligned columns against the record oracle, the word
    kernel on aligned columns against the fallback, and the counters of both."""
    rng = np.random.default_rng(seed)
    rows = _filter_units(rng, p)
    want = _filter_reference(rows, p, seen)
    units, host, owned = _layout(rows)
    n = len(host[0])
    db = _UnitsOnly(fg, units, DEV)
    eng = fg.Engine(0, 45, 40, 1, 2)
    fp = fg.lib.FgbFilterParams(p[0], p[1], p[2], p[3], p[4], p[5], p[6])
    sh8, sh16 = shifts or (1 + seed % 7, 1 + (3 * seed) % 7)
    results = []
    for form in ((0, 0), (sh8, sh16)):
        cols = _Cols(fg, n, *form)
        cols.load(*host)
        assert cols.misaligned() == (form != (0, 0))
        status, masked, stats = _run_filter(fg, eng, db, cols, fp, len(rows))
        cols.assert_fill_outside(owned)
        (gb, gq), (gd, ge) = cols.host()
        assert np.array_equal(gd, host[2]) and np.array_equal(ge, host[3])      # depth / errors are read only
        results.append((gb, gq, status, masked, stats))
    eng.close()
    (wb, wq, ws, wm, wstats), (fb, fq, fs, fm, fstats) = results
    for u, (mb, mq, st, nm) in enumerate(want):
        o, L = int(units[u]["out_off"]), len(rows[u][0])
        assert fs[u] == st, (p, u, L, fs[u], st)
        assert fm[u] == nm, (p, u, L, fm[u], nm)
        assert np.array_equal(fb[o:o + L], mb) and np.array_equal(fq[o:o + L], mq), (p, u, L)
    assert np.array_equal(wb, fb) and np.array_equal(wq, fq)
    assert np.array_equal(ws, fs) and np.array_equal(wm, fm)
    records = sum(1 for r in rows if len(r[0]))
    assert fstats["filter_records"] == records and fstats["filter_passed"] == int((fs == 0).sum())
    assert fstats["filter_bases_masked"] == int(fm[fs != NO_RECORD].astype(np.int64).sum())
    for k in ("filter_records", "filter_passed", "filter_bases_masked"):
        assert wstats[k] == fstats[k], k
    return len(rows)


def test_filter_fallback_kernel_grid(fg):
    """K4 on misaligned columns (filter_simplex_kernel) and on aligned ones (the word kernel) over a grid of settings,
    against the record oracle's mask_bases / filter_read / no-call and mean-quality checks on the record the simplex
    caller would write."""
    seen = set()
    n_units = [filter_forms(fg, p, 11 + i, seen) for i, p in enumerate(FILTER_GRID)]
    assert min(n_units) > 256                                            # several chunks of the word kernel
    for rate in (0.1, 0.25, 1 / 3, 0.0):
        for kind in ("base_rate_eq", "base_rate_above", "base_rate_below"):
            depths = {x[2] for x in seen if isinstance(x, tuple) and x[:2] == (kind, rate)}
            if kind == "base_rate_below" and rate == 0.0:
                continue                                                 # nothing is below a zero rate
            assert len(depths) >= 5, (kind, rate, sorted(depths))
    assert "clamp_decides" in seen
    assert ("ce_f32_fails", 0.1) in seen and ("ce_f32_fails", 1 / 3) in seen and ("ce_f32_passes", 0.7) in seen
    assert {"all_n", "empty", "mean_eq", "mean_one_below", "nocall_fraction_eq"} <= seen
    assert ("nocall_count_eq", 1.0) in seen and ("nocall_count_eq", 3.0) in seen
    assert {("status", s) for s in (0, 1, 2, 3, 4)} <= seen
    assert {("several_gates", s) for s in (1, 2, 3)} <= seen


# ============================ K2: the duplex combine ======================================================
def _duplex_workload(rng):
    """Real molecules with all four arms, IUPAC and lower-case source bases, plus: a molecule with more than 255
    pooled reads, molecules with strands of 300-1300 bases, a job that uses one unit on both sides and jobs whose units
    lie far apart."""
    units, pairs = _duplex_molecules(rng, 120, depth_hi=8, len_lo=20, len_hi=150, iupac=True)
    base = len(units)
    for k in range(4):                                      # 140 + 140 pooled reads
        units.append(_family(rng, 140, 150, err=0.02)[0])
    pairs += [(base + 0, base + 3), (base + 1, base + 2)]
    for m in range(3):                                      # long strands
        u0 = len(units)
        for k in range(4):
            units.append(_family(rng, int(rng.integers(2, 5)), int(rng.integers(300, 1300)))[0])
        pairs += [(u0 + 0, u0 + 3), (u0 + 1, u0 + 2)]
    pairs += [(5, 5), (0, len(units) - 1), (len(units) - 2, 9)]
    return units, pairs


def _duplex_jobs(fg, batch, pairs):
    cons_len = batch.units["cons_len"]
    jobs = np.zeros(len(pairs), dtype=fg.DUPLEX_JOB_DTYPE)
    off = 0
    for j, (ua, ub) in enumerate(pairs):
        jobs[j] = (ua, ub, off)
        off += (max(int(cons_len[ua]), int(cons_len[ub])) + 7) // 8 * 8
    return jobs, max(off, 8)


def _duplex_oracle(batch, units, pairs, ss_oracle):
    """orc_duplex_job over the oracle's SS columns: per job (status, base, qual, errors)."""
    L = O.load()
    ob, oq, od, oe = ss_oracle
    cons_len, out_off = batch.units["cons_len"], batch.units["out_off"]
    res = []
    for ua, ub in pairs:
        la, lb = int(cons_len[ua]), int(cons_len[ub])
        oa, obo = int(out_off[ua]), int(out_off[ub])
        rows = units[ua] + units[ub]
        keep = [np.frombuffer(r[0], np.uint8).copy() for r in rows]
        ptrs = (C.c_void_p * len(rows))(*[k.ctypes.data for k in keep])
        lens = (C.c_size_t * len(rows))(*[len(r[0]) for r in rows])
        cap = max(la, lb, 1)
        rb = np.zeros(cap, np.uint8); rq = np.zeros(cap, np.uint8); re_ = np.zeros(cap, np.uint16)
        olen = C.c_size_t()
        st = L.orc_duplex_job(ob[oa:].ctypes.data, oq[oa:].ctypes.data, od[oa:].ctypes.data,
                              oe[oa:].ctypes.data, la, ob[obo:].ctypes.data, oq[obo:].ctypes.data,
                              od[obo:].ctypes.data, oe[obo:].ctypes.data, lb, ptrs, lens, len(rows),
                              rb.ctypes.data, rq.ctypes.data, re_.ctypes.data, C.addressof(olen))
        n = olen.value
        res.append((st, rb[:n].copy(), rq[:n].copy(), re_[:n].copy()))
    return res


class _DuplexOut:
    def __init__(self, fg, n_out, n_jobs, sh8, sh16):
        import torch
        self.cols = _Cols(fg, n_out, sh8, sh16, depth=False)
        self.raw_status = torch.full((n_jobs + 8,), 77, dtype=torch.uint8, device=DEV)
        self.status = self.raw_status[sh8:sh8 + n_jobs]
        self.sh8 = sh8

    def args(self):
        return self.cols.base, self.cols.qual, self.cols.errors, self.status

    def host(self):
        (b, q), (e,) = self.cols.host()
        return b, q, e, self.status.cpu().numpy()


def _check_duplex(out, jobs, want, strict, cons_len):
    """Every job equals the oracle; nothing outside the jobs' rows was written (`strict`: outside the output row
    proper; else outside the row's 8-aligned slot, which a word kernel may fill)."""
    gb, gq, ge, gs = out.host()
    owned = np.zeros(out.cols.n, bool)
    for j, (st, rb, rq, re_) in enumerate(want):
        o, n = int(jobs[j]["out_off"]), len(rb)
        assert gs[j] == st, (j, gs[j], st)
        assert np.array_equal(gb[o:o + n], rb) and np.array_equal(gq[o:o + n], rq), j
        assert np.array_equal(ge[o:o + n], re_), j
        slot = n if strict else (max(int(cons_len[jobs[j]["unit_a"]]), int(cons_len[jobs[j]["unit_b"]])) + 7) // 8 * 8
        owned[o:o + slot] = True
    out.cols.assert_fill_outside(owned)
    return gb, gq, ge, gs


def duplex_forms(fg, units, pairs, sh8=3, sh16=5):
    """K2 on misaligned source bases, SS columns and outputs (duplex_combine_kernel) against the oracle and against
    the word kernel on the aligned copies; then fgb_vote_duplex_device with misaligned outputs (vote, then the fallback
    kernel) against the fused form.  Returns the arms seen."""
    import torch
    batch = fg.pack_source_reads(units, 1)
    cons_len = batch.units["cons_len"]
    eng = fg.Engine(0, 45, 40, 1, 2)
    db = fg.DeviceBatch(batch, DEV)
    ss = fg.DeviceColumns(batch.n_out, DEV)
    eng.vote_device(db, ss, _stream())
    torch.cuda.synchronize()
    oracle_ss = O.simplex_batch(batch, 45, 40, 1, 2)[:4]
    g = ss.to_host()
    for sl in batch.unit_slices():
        assert all(np.array_equal(x[sl], y[sl]) for x, y in zip((g.base, g.qual, g.depth, g.errors), oracle_ss))
    want = _duplex_oracle(batch, units, pairs, oracle_ss)
    jobs, n_out = _duplex_jobs(fg, batch, pairs)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(DEV)
    # the same source bases and SS columns behind misaligned pointers
    raw_bases = torch.zeros(db.bases.numel() + 16, dtype=torch.uint8, device=DEV)
    db_mis = copy.copy(db)
    db_mis.bases = raw_bases[sh8:sh8 + db.bases.numel()]
    db_mis.bases.copy_(db.bases)
    ss_mis = _Cols(fg, ss.base.numel(), sh8, sh16)
    ss_mis.load(ss.base, ss.qual, ss.depth, ss.errors)
    assert _ptr_misaligned(db_mis.bases, 8) and ss_mis.misaligned()
    runs = []
    for d, s, sh in ((db, ss, (0, 0)), (db_mis, ss_mis, (1 + (sh8 + 1) % 7, 1 + sh16 % 7))):
        out = _DuplexOut(fg, n_out, len(pairs), *sh)
        eng.stats_reset()
        eng.duplex_combine_device(d, s, tj, len(pairs), *out.args(), _stream())
        torch.cuda.synchronize()
        runs.append((_check_duplex(out, jobs, want, d is db_mis, cons_len), eng.stats()))
    assert out.cols.misaligned()
    (aligned, s_al), (fallback, s_fb) = runs
    for j in range(len(pairs)):
        o, n = int(jobs[j]["out_off"]), len(want[j][1])
        assert all(np.array_equal(x[o:o + n], y[o:o + n]) for x, y in zip(aligned[:3], fallback[:3])), j
    assert np.array_equal(aligned[3], fallback[3])
    assert s_al["combined_jobs"] == s_fb["combined_jobs"] == len(pairs)
    # fgb_vote_duplex_device: fused with aligned outputs, vote + fallback kernel with misaligned ones
    tiles, class_tiles, tile_jobs, job_index, n_attached = fg.plan_tiles_jobs(batch, jobs)
    assert n_attached > 0
    t8 = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(DEV)
    db_f = copy.copy(db)
    db_f.tiles, db_f.n_tiles, db_f.class_tiles = t8(tiles), len(tiles), class_tiles
    d_tj, d_ji = t8(tile_jobs), t8(job_index)
    fused = []
    for sh in ((0, 0), (1 + (sh8 + 3) % 7, 1 + (sh16 + 1) % 7)):
        out = _DuplexOut(fg, n_out, len(pairs), *sh)
        ss2 = fg.DeviceColumns(batch.n_out, DEV)
        eng.stats_reset()
        eng.vote_duplex_device(db_f, ss2, tj, len(pairs), d_tj, d_ji, *out.args(), _stream())
        torch.cuda.synchronize()
        g2 = ss2.to_host()
        assert all(np.array_equal(x, y) for x, y in zip((g.base, g.qual, g.depth, g.errors),
                                                       (g2.base, g2.qual, g2.depth, g2.errors)))
        fused.append((_check_duplex(out, jobs, want, sh != (0, 0), cons_len), eng.stats()))
    assert out.cols.misaligned()
    (f_al, fs_al), (f_mis, fs_mis) = fused
    for j in range(len(pairs)):
        o, n = int(jobs[j]["out_off"]), len(want[j][1])
        assert all(np.array_equal(x[o:o + n], y[o:o + n]) for x, y in zip(f_al[:3], f_mis[:3])), j
    assert np.array_equal(f_al[3], f_mis[3]) and int(f_mis[3].max()) <= 3
    assert fs_al["combined_jobs"] == fs_mis["combined_jobs"] == len(pairs)
    assert fs_al["units"] == fs_mis["units"] == len(units)
    eng.close()
    return {w[0] for w in want}


def test_duplex_fallback_kernel(fg):
    rng = np.random.default_rng(61)
    units, pairs = _duplex_workload(rng)
    sizes = [len(units[a]) + len(units[b]) for a, b in pairs]
    assert max(sizes) > 255
    assert duplex_forms(fg, units, pairs) == {0, 1, 2, 3}


# ============================ K3: the CODEC combine =======================================================
def codec_forms(fg, seed, sh8=5, sh16=3):
    """K3 on misaligned SS and output columns (codec_combine_kernel) against the oracle's padded combine and against
    the word kernel on aligned copies, for both parameter sets."""
    import torch
    L = O.load()
    L.orc_codec_combine.restype = None
    L.orc_codec_mask.restype = None
    rng = np.random.default_rng(seed)
    units, jobs, (sb, sq, sd, se), ooff = _codec_job_mix(fg, rng)
    n_jobs = len(jobs)
    db = _UnitsOnly(fg, units, DEV)
    eng = fg.Engine(0, 45, 40, 1, 0)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(DEV)
    statuses = set()
    for ss_q, outer_q, outer_len, max_dis, max_rate in ((-1, -1, 0, 0xFFFFFFFF, 1.0), (10, 7, 9, 12, 0.3)):
        cp = fg.lib.FgbCodecParams(ss_q, outer_q, outer_len, max_dis, max_rate)
        runs = []
        for form in ((0, 0), (sh8, sh16)):
            ss = _Cols(fg, len(sb), *form)
            ss.load(sb, sq, sd, se)
            out = _Cols(fg, ooff + 8, *((0, 0) if form == (0, 0) else (1 + (sh8 + 1) % 7, 1 + (sh16 + 2) % 7)))
            assert ss.misaligned() == out.misaligned() == (form != (0, 0))
            st = torch.full((n_jobs,), 255, dtype=torch.uint8, device=DEV)
            dis = torch.full((n_jobs,), -1, dtype=torch.int32, device=DEV); dup = torch.full_like(dis, -1)
            eng.stats_reset()
            eng.codec_combine_device(db, ss, tj, n_jobs, cp, out, st, dis, dup, _stream())
            torch.cuda.synchronize()
            (gb, gq), (gd, ge) = out.host()
            runs.append(((gb, gq, gd, ge, st.cpu().numpy(), dis.cpu().numpy(), dup.cpu().numpy()), eng.stats(), out))
        (w, ws, _), (f, fs, fout) = runs
        gb, gq, gd, ge, gs, gdis, gdup = f
        owned = np.zeros(ooff + 8, bool)
        tot_dup = tot_dis = 0
        for m in range(n_jobs):
            rb, rq, rd, re_, nb, nd = _codec_job_reference(L, (sb, sq, sd, se), units[2 * m], units[2 * m + 1], jobs[m],
                                                           (ss_q, outer_q, outer_len))
            o, n = int(jobs[m]["out_off"]), int(jobs[m]["len"])
            assert np.array_equal(gb[o:o + n], rb) and np.array_equal(gq[o:o + n], rq), m
            assert np.array_equal(gd[o:o + n], rd) and np.array_equal(ge[o:o + n], re_), m
            assert gdup[m] == nb and gdis[m] == nd, m
            want = 0
            if nb > 0:
                want = 1 if nd > max_dis else (2 if nd / nb > max_rate else 0)
            assert gs[m] == want, m
            statuses.add(want)
            owned[o:o + n] = True
            tot_dup += nb; tot_dis += nd
        fout.assert_fill_outside(owned)
        for x, y in zip(w, f):
            assert np.array_equal(x, y)
        assert fs["duplex_bases"] == tot_dup and fs["duplex_disagreements"] == tot_dis and fs["combined_jobs"] == n_jobs
        for k in ("duplex_bases", "duplex_disagreements", "combined_jobs"):
            assert ws[k] == fs[k], k
    eng.close()
    return statuses


def test_codec_fallback_kernel(fg):
    assert codec_forms(fg, 78) == {0, 1, 2}


# ============================ the vote refuses pointers it cannot use ======================================
def test_vote_refuses_misaligned_pointers(fg):
    """fgb_vote_device and fgb_vote_duplex_device return FGB_ERR_LAYOUT with a message, launch nothing, and the same
    handle then votes an aligned batch correctly."""
    import torch
    rng = np.random.default_rng(71)
    units, pairs = _duplex_molecules(rng, 40)
    batch = fg.pack_source_reads(units, 1)
    jobs, n_out = _duplex_jobs(fg, batch, pairs)
    eng = fg.Engine(0, 45, 40, 1, 2)
    lib = eng._lib
    db = fg.DeviceBatch(batch, DEV)
    ss = fg.DeviceColumns(batch.n_out, DEV)
    tiles, class_tiles, tile_jobs, job_index, _ = fg.plan_tiles_jobs(batch, jobs)
    t8 = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(DEV)
    db_f = copy.copy(db)
    db_f.tiles, db_f.n_tiles, db_f.class_tiles = t8(tiles), len(tiles), class_tiles
    tj, d_tj, d_ji = t8(jobs), t8(tile_jobs), t8(job_index)
    o_base = torch.zeros(n_out, dtype=torch.uint8, device=DEV); o_qual = torch.zeros_like(o_base)
    o_err = torch.zeros(n_out, dtype=torch.int16, device=DEV)
    dout = fg.lib.FgbDuplexOut(o_base.data_ptr(), o_qual.data_ptr(), o_err.data_ptr(), None)
    cases = ([("bases", k) for k in (1, 4, 8)] + [("quals", k) for k in (1, 8)] + [("reads", 8), ("units", 8),
             ("tiles", 8)] + [("base", k) for k in (1, 4)] + [("qual", 2)] + [("depth", k) for k in (2, 8)] +
             [("errors", k) for k in (2, 6, 8)])
    n_launch = eng.launch_count()
    refused = 0
    for field, k in cases:
        for duplex in (False, True):
            b = (db_f if duplex else db).struct()
            c = ss.struct()
            tgt = b if field in ("bases", "quals", "reads", "units", "tiles") else c
            setattr(tgt, field, getattr(tgt, field) + k)
            if duplex:
                st = lib.fgb_vote_duplex_device(eng._h, C.byref(b), C.byref(c), C.c_void_p(tj.data_ptr()), len(pairs),
                                                C.c_void_p(d_tj.data_ptr()), C.c_void_p(d_ji.data_ptr()), C.byref(dout),
                                                C.c_void_p(_stream()))
            else:
                st = lib.fgb_vote_device(eng._h, C.byref(b), C.byref(c), C.c_void_p(_stream()))
            assert st == fg.lib.FGB_ERR_LAYOUT, (field, k, duplex, st)
            buf = C.create_string_buffer(256)
            lib.fgb_last_error(eng._h, buf, 256)
            msg = buf.value.decode()
            assert field in msg and "aligned" in msg, (field, msg)
            assert eng.launch_count() == n_launch
            refused += 1
    assert refused == 2 * len(cases)
    torch.cuda.synchronize()
    eng.vote_device(db, ss, _stream())
    torch.cuda.synchronize()
    assert eng.launch_count() > n_launch
    ob, oq, od, oe, _ = O.simplex_batch(batch, 45, 40, 1, 2)
    g = ss.to_host()
    for sl in batch.unit_slices():
        assert np.array_equal(g.base[sl], ob[sl]) and np.array_equal(g.qual[sl], oq[sl])
        assert np.array_equal(g.depth[sl], od[sl]) and np.array_equal(g.errors[sl], oe[sl])
    assert eng.stats()["units"] == len(units)
    eng.close()
