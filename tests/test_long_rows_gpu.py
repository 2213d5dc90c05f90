"""The consensus path on reads up to the 65 535-base limit, on the GPU, against the project's oracles
(tests/long_rows.py builds the workloads; tests/test_long_rows.py checks them without a GPU).

Forms that only long rows reach, and the test that reaches each:
- shallow-class direct tiles (`vote_tile<GlMem>` in the shallow kernel, and its slow pass): 1-4-read units whose
  rows span more than one stage -- test_vote_forms_at_long_rows, test_tiles_beyond_4_gib;
- general-class direct tiles by length (5-23 reads) -- test_vote_forms_at_long_rows, test_tiles_beyond_4_gib;
- deep-class direct tiles of short-read-count units -- test_vote_forms_at_long_rows;
- direct tiles without the uniform-items hint (cons_len > 32 768: the unit is found by binary search), and warp-queue
  overflow into the in-place HBM path -- test_vote_forms_at_long_rows;
- queue entries with positions above 32 767 (units whose first 33 000 positions are clean, so that nothing is queued
  before them), in the shallow, general and deep kernels -- test_vote_forms_at_long_rows;
- staged regular tiles of one or two units at the byte cap (ten items per voting thread) -- test_vote_forms_at_long_rows;
- row offsets above 2^32 in direct and staged tiles -- test_tiles_beyond_4_gib;
- duplex molecules whose strands do not fit one stage (the standalone pending combine) beside ones that do (the fused
  epilogue) -- test_duplex_on_long_strands;
- CODEC combine jobs of 8 k to 65 535 positions -- test_codec_combine_on_long_jobs;
- the row builder on 8 k-65 535-base rows with quality bytes >= 128 -- test_row_builder_at_long_rows;
- device record assembly (K5) with cd / ce arrays of tens of thousands of entries, the filter epilogue (K4), host
  assembly with a total depth past 2^24 -- test_simplex_caller_on_long_reads_*."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import long_rows as LR                       # noqa: E402
from tests import oracle_lib as O                       # noqa: E402
from tests.test_vote_settings import _compare, _duplex_against_oracle   # noqa: E402

pytestmark = pytest.mark.gpu

# (pre, post, min_reads, min_consensus_base_quality): the defaults, a min_reads = 3 / high-quality gate, and a
# post-UMI rate of Q1, where no quality threshold is finite and every position takes the exact vote
SETTINGS = [(45, 40, 1, 2), (30, 20, 3, 40), (45, 1, 1, 2)]


@pytest.fixture(scope="module")
def ladder(fg):
    return LR.ladder_batch(fg, seed=2)


def _vote(fg, batch, way, pre, post, min_reads, mcq, db=None):
    import torch
    eng = fg.Engine(0, pre, post, min_reads, mcq)
    try:
        if way == "submit":
            out = eng.vote(batch)
        else:
            db = db if db is not None else fg.DeviceBatch(batch, "cuda:0")
            if way == "unsorted":
                db.class_tiles = (0, 0, 0)         # every tile through the general kernel
            dc = fg.DeviceColumns(batch.n_out, "cuda:0")
            eng.vote_device(db, dc, torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            out = dc.to_host()
        return out, eng.stats()
    finally:
        eng.close()


@pytest.mark.parametrize("pre,post,min_reads,mcq", SETTINGS, ids=lambda v: str(v))
def test_vote_forms_at_long_rows(fg, ladder, pre, post, min_reads, mcq):
    """The whole ladder through the class kernels, through the general kernel alone and through the host-buffer
    submit: bases, qualities, depths, errors and counters bit-identical to the oracle."""
    _, units, specs = ladder
    batch = fg.pack_source_reads(units, min_reads)
    f = LR.forms(fg, batch)
    want = {("shallow", True, False, True), ("shallow", True, False, False), ("general", True, False, False),
            ("deep", True, False, False), ("deep", True, False, True)}
    if min_reads == 1:
        want |= {(c, False, True, True) for c in ("shallow", "general", "deep")}
    assert want <= f, sorted(want - f)
    ref = O.simplex_batch(batch, pre, post, min_reads, mcq, 8)
    for way in ("sorted", "unsorted", "submit"):
        out, stats = _vote(fg, batch, way, pre, post, min_reads, mcq)
        _compare(out, ref, batch, stats, f"{way} {pre}/{post}/{min_reads}/{mcq}")


def test_tiles_beyond_4_gib(fg):
    """Shallow-direct, general-direct, deep-direct and staged long units whose rows lie above 2^32 in a sparse
    device-resident column give what the same units give packed at offset 0.  The column is filled at the rows and,
    as a decoy, where 32-bit row offsets would land: there every row reads a confident, unanimous C.  (Zero bytes
    would not do: the fast passes decide nothing on them, and the slow pass reads the rows again from their full
    offsets, so a truncated offset in a fast pass would go unseen.)"""
    import torch
    free = torch.cuda.mem_get_info()[0]
    if free < 12 * 2**30:
        pytest.skip(f"needs ~12 GiB of free device memory for two 4 GiB columns; {free / 2**30:.1f} GiB free")
    rng = np.random.default_rng(9)
    shapes = [(2, [30001, 29000]), (6, [9000] * 6), (30, [1200] * 30), (1, [20000]), (1, [40000]), (3, [5000] * 3)]
    units = [LR.long_unit(rng, d, lens, LR.default_dissent(max(lens))) for d, lens in shapes]
    batch = fg.pack_source_reads(units, 1)
    ref = O.simplex_batch(batch, 45, 40, 1, 2, 8)
    base = 2**32 + 4096                   # a 32-bit row offset would land at 4096 + offset, in the decoy
    far = fg.PackedBatch(None, None, batch.reads.copy(), batch.units.copy(), batch.n_units, batch.n_reads,
                         base + batch.n_bytes, batch.n_out)
    far.reads[:far.n_reads] += np.uint64(base << 16)
    f = LR.forms(fg, far)
    assert {("shallow", True, False, True), ("general", True, False, True), ("deep", True, False, True),
            ("shallow", False, True, True), ("shallow", True, False, False)} <= f, sorted(f)
    assert (far.tiles["byte_begin"] >= 2**32).all()
    dev = "cuda:0"
    db = fg.DeviceBatch.__new__(fg.DeviceBatch)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)
    try:
        n = base + len(batch.bases)
        db.bases = torch.zeros(n, dtype=torch.uint8, device=dev)
        db.quals = torch.zeros(n, dtype=torch.uint8, device=dev)
        db.bases[base:].copy_(torch.from_numpy(batch.bases))
        db.quals[base:].copy_(torch.from_numpy(batch.quals))
        decoy = slice(base - 2**32, base - 2**32 + len(batch.bases))
        db.bases[decoy].fill_(ord("C"))
        db.quals[decoy].fill_(40)
        db.host, db.device = far, dev
        db.reads, db.units = t(far.reads), t(far.units)
        sorted_tiles, db.class_tiles = fg.engine.sort_tiles_by_class(far.tiles)
        db.tiles, db.n_tiles = t(sorted_tiles), len(far.tiles)
        out, stats = _vote(fg, far, "sorted", 45, 40, 1, 2, db)
        _compare(out, ref, batch, stats, "rows above 2^32, class kernels")
        out, stats = _vote(fg, far, "unsorted", 45, 40, 1, 2, db)
        _compare(out, ref, batch, stats, "rows above 2^32, general kernel")
    finally:
        del db
        torch.cuda.empty_cache()


@pytest.mark.parametrize("fused", [True, False])
def test_duplex_on_long_strands(fg, fused):
    """Molecules whose strands are 1-4 reads of 2-12 kb, of unequal lengths: pairs that fit one stage are combined
    in the vote kernels' epilogue, the others by the pending combine; both paths against orc_duplex_job."""
    rng = np.random.default_rng(13)
    units, pairs = [], []
    for m in range(24):
        for _ in range(2):
            if m % 3 == 0:                                   # two single reads that share a stage
                d, lens = 1, [int(rng.integers(2000, 9000))]
            else:
                d = int(rng.integers(1, 5))
                lens = [int(x) for x in rng.integers(2000, 12001, size=d)]
            units.append(LR.long_unit(rng, d, lens, LR.default_dissent(max(lens))))
        pairs.append((len(units) - 2, len(units) - 1))
    batch = fg.pack_source_reads(units, 1)
    jobs = np.zeros(len(pairs), dtype=fg.DUPLEX_JOB_DTYPE)
    for j, (a, b) in enumerate(pairs):
        jobs[j] = (a, b, 0)
    _, _, _, _, n_attached = fg.plan_tiles_jobs(batch, jobs)
    assert 0 < n_attached < len(pairs), n_attached
    _duplex_against_oracle(fg, units, pairs, fused, 45, 40, 2)


def test_codec_combine_on_long_jobs(fg):
    """CODEC combine jobs of 8 k to 65 535 output positions, every orientation, with pads, output rows 8-aligned
    and not, against the oracle's padded combine + mask."""
    import torch
    from tests.test_combine_parity import _UnitsOnly, _codec_job_reference
    L = O.load()
    L.orc_codec_combine.restype = None
    L.orc_codec_mask.restype = None
    rng = np.random.default_rng(17)
    n_jobs = 24
    units = np.zeros(2 * n_jobs + 1, dtype=fg.UNIT_DTYPE)
    jobs = np.zeros(n_jobs, dtype=fg.CODEC_JOB_DTYPE)
    off = ooff = 0
    for m in range(n_jobs):
        n = LR.MAX_READ_LEN - m if m < 4 else int(rng.integers(8192, LR.MAX_READ_LEN + 1))
        for s in range(2):
            l = int(rng.integers(n // 2, n + 1)) if m % 3 else n
            units[2 * m + s]["out_off"], units[2 * m + s]["cons_len"] = off, l
            off += (l + 7) // 8 * 8
        la, lb = int(units[2 * m]["cons_len"]), int(units[2 * m + 1]["cons_len"])
        jobs[m]["unit_a"], jobs[m]["unit_b"], jobs[m]["len"] = 2 * m, 2 * m + 1, n
        jobs[m]["rc_a"], jobs[m]["rc_b"], jobs[m]["rc_out"] = (m >> 0) & 1, (m >> 1) & 1, (m >> 2) & 1
        jobs[m]["pad_a_left"] = int(rng.integers(0, n - la + 1))
        jobs[m]["pad_b_left"] = int(rng.integers(0, n - lb + 1))
        if m % 4 == 3:
            ooff += int(rng.integers(1, 8))                 # this job's output row is not 8-aligned
        jobs[m]["out_off"] = ooff
        ooff = (ooff + n + 7) // 8 * 8
    units[2 * n_jobs]["out_off"] = off
    sb = rng.choice(np.frombuffer(b"ACGTN", np.uint8), size=off + 16, p=[0.24, 0.24, 0.24, 0.24, 0.04])
    sq = rng.integers(0, 94, size=off + 16).astype(np.uint8)
    sd = rng.integers(1, 300, size=off + 16).astype(np.uint16)
    se = np.minimum(sd, rng.integers(0, 6, size=off + 16)).astype(np.uint16)
    dev = "cuda:0"
    ss = fg.DeviceColumns(len(sb), dev)
    ss.base.copy_(torch.from_numpy(sb)); ss.qual.copy_(torch.from_numpy(sq))
    ss.depth.copy_(torch.from_numpy(sd.view(np.int16))); ss.errors.copy_(torch.from_numpy(se.view(np.int16)))
    db = _UnitsOnly(fg, units, dev)
    eng = fg.Engine(0, 45, 40, 1, 0)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(dev)
    try:
        for ss_q, outer_q, outer_len, max_dis, max_rate in ((-1, -1, 0, 0xFFFFFFFF, 1.0), (10, 7, 9, 300, 0.01)):
            out = fg.DeviceColumns(ooff + 8, dev)
            out.base.fill_(0x55); out.qual.fill_(0x55); out.depth.fill_(0x5555); out.errors.fill_(0x5555)
            st = torch.full((n_jobs,), 255, dtype=torch.uint8, device=dev)
            dis = torch.zeros(n_jobs, dtype=torch.int32, device=dev); dup = torch.zeros_like(dis)
            cp = fg.lib.FgbCodecParams(ss_q, outer_q, outer_len, max_dis, max_rate)
            eng.codec_combine_device(db, ss, tj, n_jobs, cp, out, st, dis, dup, torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            g = out.to_host()
            gs, gdis, gdup = st.cpu().numpy(), dis.cpu().numpy(), dup.cpu().numpy()
            written = np.zeros(ooff + 8, bool)
            for m in range(n_jobs):
                rb, rq, rd, re_, nb, nd = _codec_job_reference(L, (sb, sq, sd, se), units[2 * m], units[2 * m + 1],
                                                               jobs[m], (ss_q, outer_q, outer_len))
                o, n = int(jobs[m]["out_off"]), int(jobs[m]["len"])
                for name, a, b in (("base", g.base, rb), ("qual", g.qual, rq), ("depth", g.depth, rd),
                                   ("errors", g.errors, re_)):
                    bad = np.flatnonzero(a[o:o + n] != b)
                    assert bad.size == 0, (m, name, n, bad[:5])
                assert gdup[m] == nb and gdis[m] == nd, m
                want = 0 if nb == 0 else 1 if nd > max_dis else 2 if nd / nb > max_rate else 0
                assert gs[m] == want, m
                written[o:o + n] = True
            assert (g.base[~written] == 0x55).all() and (g.depth[~written] == 0x5555).all()
    finally:
        eng.close()


# ---- the row builder ------------------------------------------------------------------------------------------------
ROW_LENS = (8193, 8200, 16384, 30001, 40961, 65534, 65535, 65535)


def _long_records(rng):
    """Records of 8 193-65 535 bases on both strands, with quality bytes over 0-255 and runs of 0xFF (a record
    with missing qualities), and the kept row length of each."""
    from tests.bam_builder import make_record
    recs, rows = [], []
    for i, L in enumerate(ROW_LENS):
        seq = LR.ACGT[rng.integers(0, 4, size=L)].copy()
        m = rng.random(L) < 0.05
        seq[m] = np.frombuffer(b"NRYKM", np.uint8)[rng.integers(0, 5, size=int(m.sum()))]
        q = rng.integers(0, 256, size=L).astype(np.uint8)
        for _ in range(4):
            a = int(rng.integers(0, L - 1))
            q[a:a + int(rng.integers(1, 3000))] = 0xFF
        if i == 5:
            q[:] = 0xFF
        rev = i % 2 == 1
        recs.append(make_record(name=b"long%d" % i + b"x" * i, flags=16 if rev else 0, pos=100, seq=seq.tobytes(),
                                quals=q.tobytes(), tags=[(b"MI", "Z", b"7")]))
        final_len = L if i % 3 == 0 else int(rng.integers(L // 2, L + 1))
        rows.append((L, rev, final_len, seq, q))
    return recs, rows


def _check_rows(hb, hq, rows, min_q, guard=None):
    from tests.test_records_input import _expected_row
    off = 0
    for r, (L, rev, fl, seq, q) in enumerate(rows):
        eb, eq = _expected_row(L, rev, fl, seq, q, min_q)
        assert np.array_equal(hb[off:off + fl], eb), (r, L, rev, fl, min_q)
        assert np.array_equal(hq[off:off + fl], eq), (r, L, rev, fl, min_q)
        padded = (fl + 7) // 8 * 8
        assert not hb[off + fl:off + padded].any() and not hq[off + fl:off + padded].any()     # zeroed row padding
        off += padded
    if guard is not None:
        assert (hb[off:] == guard).all() and (hq[off:] == guard).all()        # nothing written past the last row


@pytest.mark.parametrize("min_q", [0, 10, 127, 128, 200])
def test_row_builder_at_long_rows(fg, min_q):
    """fgb_unpack_records_device and fgb_unpack_bam4_device on rows of 8 193-65 535 bases (both strands, odd
    lengths, quality bytes >= 128 that pass any min_q <= 127) against the per-base rule."""
    import torch
    rng = np.random.default_rng(100 + min_q)
    recs, rows = _long_records(rng)
    assert any((q >= 128).any() for *_, q in rows) and any((q == 0xFF).all() for *_, q in rows)
    R = len(recs)
    reads = np.zeros(R + 2, dtype=np.uint64)
    off_row = 0
    for r, (_, _, fl, _, _) in enumerate(rows):
        reads[r] = (off_row << 16) | fl
        off_row += (fl + 7) // 8 * 8
    dev = "cuda:0"
    lib = fg.lib.load()
    eng = fg.Engine(0, 45, 40, 1, 2)
    d_reads = torch.from_numpy(reads.view(np.uint8).copy()).to(dev)
    batch = fg.lib.FgbBatch(0, R, off_row, 0, 0, None, None, d_reads.data_ptr(), None, None)
    try:
        # records form: the rows' bases and qualities straight from the BAM records
        blob = np.frombuffer(b"".join(recs), np.uint8)
        rec_off = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.uint64)
        raw = np.zeros(R, dtype=fg.RAW_READ_DTYPE)
        for r, (rec, (L, rev, _, _, _)) in enumerate(zip(recs, rows)):
            raw[r] = (int(rec_off[r]) + 32 + rec[8] + 4 * int.from_bytes(rec[12:14], "little"), L, 1 if rev else 0)
        d_blob = torch.from_numpy(np.concatenate([blob, np.zeros(64, np.uint8)])).to(dev)
        d_raw = torch.from_numpy(raw.view(np.uint8).reshape(-1).copy()).to(dev)
        d_b = torch.full((off_row + 64,), 0xAA, dtype=torch.uint8, device=dev)
        d_q = torch.full((off_row + 64,), 0xAA, dtype=torch.uint8, device=dev)
        rc = fg.lib.FgbRecordColumns(len(blob) + 64, d_blob.data_ptr(), d_raw.data_ptr(), min_q)
        assert lib.fgb_unpack_records_device(eng._h, C.byref(batch), C.byref(rc), C.c_void_p(d_b.data_ptr()),
                                             C.c_void_p(d_q.data_ptr()), None) == 0
        torch.cuda.synchronize()
        assert lib.fgb_wait(eng._h) == 0
        _check_rows(d_b.cpu().numpy(), d_q.cpu().numpy(), rows, min_q, guard=0xAA)
        # BAM4 form: 4-bit sequence and raw qualities, spans on even nibbles
        code = {c: i for i, c in enumerate(b"=ACMGRSVTWYHKDBN")}
        nibs, quals, raw4 = [], [], np.zeros(R, dtype=fg.RAW_READ_DTYPE)
        o = 0
        for r, (L, rev, _, seq, q) in enumerate(rows):
            raw4[r] = (o, L, 1 if rev else 0)
            nibs.append(np.array([code.get(int(b), 15) for b in seq], np.uint8)); quals.append(q)
            o += L
            if o % 2:
                nibs.append(np.zeros(1, np.uint8)); quals.append(np.zeros(1, np.uint8)); o += 1
        nib, allq = np.concatenate(nibs), np.concatenate(quals)
        seq4 = ((nib[0::2] << 4) | nib[1::2]).astype(np.uint8)
        d_seq = torch.from_numpy(np.concatenate([seq4, np.zeros(32, np.uint8)])).to(dev)
        d_q4 = torch.from_numpy(np.concatenate([allq, np.zeros(32, np.uint8)])).to(dev)
        d_raw4 = torch.from_numpy(raw4.view(np.uint8).reshape(-1).copy()).to(dev)
        d_b.fill_(0xAA); d_q.fill_(0xAA)
        rc4 = fg.lib.FgbRawColumns(o, d_seq.data_ptr(), d_q4.data_ptr(), d_raw4.data_ptr(), min_q)
        assert lib.fgb_unpack_bam4_device(eng._h, C.byref(batch), C.byref(rc4), C.c_void_p(d_b.data_ptr()),
                                          C.c_void_p(d_q.data_ptr()), None) == 0
        torch.cuda.synchronize()
        assert lib.fgb_wait(eng._h) == 0
        _check_rows(d_b.cpu().numpy(), d_q.cpu().numpy(), rows, min_q, guard=0xAA)
    finally:
        eng.close()


# ---- the record-level simplex caller ---------------------------------------------------------------------------------
BIG_FAMILY = ("frag", 260, (LR.MAX_READ_LEN - 200, LR.MAX_READ_LEN), None)    # > 255 reads, total depth > 2^24


def _gpu_caller_output(fg, groups, n_threads=8):
    from fgumi_b200 import benchlegs
    blob, off, grp = LR.flatten(groups)
    gpu = benchlegs._Caller(fg.lib.load(), 0, n_threads)
    try:
        p, n, cnt = gpu.process(blob.ctypes.data, off.ctypes.data, grp.ctypes.data, len(groups))
        return C.string_at(p, n), cnt
    finally:
        gpu.close()


def test_simplex_caller_on_long_reads_device_assembly(fg, monkeypatch, capfd):
    """Families of 1-255 reads of 1 kb-65 535 bases, both strands, overlapping mates: records assembled on the
    device, byte-identical to the host code over the CPU oracle's vote and to the record oracle."""
    from tests.test_callers_at_depth import assert_same_stream
    from tests.test_long_rows import cpu_caller_output, record_oracle_output
    groups = LR.long_families(81)
    monkeypatch.setenv("FGB_CALLER_TRACE", "1")
    capfd.readouterr()
    got, cnt = _gpu_caller_output(fg, groups)
    err = capfd.readouterr().err
    assert "records assembled on the device" in err, err[-2000:]
    want, cnt2 = cpu_caller_output(groups)
    assert cnt == cnt2 >= len(groups)
    assert_same_stream(got, want)
    sub = [g for g in groups if len(g) <= 64]
    head = record_oracle_output(sub)[0]
    assert_same_stream(_gpu_caller_output(fg, sub)[0], head)


def test_simplex_caller_on_long_reads_trim_and_overlap(fg, monkeypatch, capfd):
    """The same families with quality trimming, per-base tags and the overlapping-bases pre-pass, against the record
    oracle's pre-pass and caller."""
    from tests.test_callers_at_depth import assert_same_stream, run_caller, simplex_caller, vanilla_oracle
    groups = LR.long_families(82)
    want, count, oracle, ov = vanilla_oracle(groups, True, overlap=True, trim=True)
    monkeypatch.setenv("FGB_CALLER_TRACE", "1")
    capfd.readouterr()
    got, st, err = run_caller(lambda: simplex_caller(fg, True, 4, trim=True, consensus_call_overlapping_bases=True),
                              groups, capfd)
    assert "records assembled on the device" in err, err[-2000:]
    assert got.count == count
    assert_same_stream(got.data, want)
    assert st["overlapping_bases"] == ov.stats()[0] > 20000


def test_simplex_caller_on_long_reads_filter(fg, monkeypatch, capfd):
    """The filter epilogue (K4) on long consensus reads: per-unit sums of up to 65 535 x depth."""
    from oracle import record_oracle as R
    from tests.test_callers_at_depth import assert_same_stream, run_caller, simplex_caller, vanilla_oracle
    groups = LR.long_families(83)
    unfiltered = vanilla_oracle(groups, True)[0]
    flt = R.SimplexFilterOracle(R.FilterThresholds(2, 0.05, 0.1), 10, None, 0.3)
    want, kept = flt.filter_stream(unfiltered)
    f = fg.ConsensusFilter(min_reads=2, max_read_error_rate=0.05, max_base_error_rate=0.1, min_base_quality=10,
                           max_no_call_fraction=0.3)
    got, st, _ = run_caller(lambda: simplex_caller(fg, True, 3, filter=f), groups, capfd)
    assert got.count == kept
    assert_same_stream(got.data, want)
    assert st["filter_records"] == flt.total and st["filter_passed"] == flt.passed
    assert st["filter_bases_masked"] == flt.bases_masked


def test_simplex_caller_on_long_reads_host_assembly(fg, monkeypatch, capfd):
    """One family of 260 reads near the limit next to the others: the batch is assembled on the host from 16-bit
    columns, and the family's total depth passes 2^24, where cE's f32 ratio rounds."""
    from tests.test_callers_at_depth import assert_same_stream
    from tests.test_long_rows import cpu_caller_output
    groups = LR.long_families(84, LR.LONG_FAMILIES[:4] + (BIG_FAMILY,))
    assert BIG_FAMILY[1] * BIG_FAMILY[2][0] > 2**24
    monkeypatch.setenv("FGB_CALLER_TRACE", "1")
    capfd.readouterr()
    got, cnt = _gpu_caller_output(fg, groups)
    err = capfd.readouterr().err
    assert "records assembled on the device" not in err, err[-2000:]
    want, cnt2 = cpu_caller_output(groups)
    assert cnt == cnt2 >= len(groups)
    assert_same_stream(got, want)
