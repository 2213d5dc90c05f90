"""BASELINE.json's configurations at FULL size on one H100 (80 GB), checked through size-independent
properties plus an exact oracle comparison on a random sample of families (the oracle cannot vote
10 M families in seconds, but it can vote a few thousand of them drawn from the very same batch):

  cfg 2  simplex  10 M families, depth 8, 150 bp, error 1e-3
  cfg 3  duplex   5 M molecules, 4+4 reads per strand  (20 M single-strand units -> 10 M duplex reads)
  cfg 4  CODEC    2 M molecules, depth 2-20 per strand, 2 x 150 bp
  cfg 5  simplex  6.25 M families (one rank's shard of 100 M over 16 GPUs), Zipf depth 1-100

Besides the sample, one contiguous slice of every vote (up to 2 M source rows: 250 k families at depth 8) is
compared with a full oracle pass, every unit and position.

Properties: device counters equal the descriptor sums; results do not depend on how the batch is cut
into launches (prefix sub-batch == prefix of the full result); a second launch is bit-identical;
depth/error invariants hold everywhere.  FGB_FULL_SCALE (default 1.0) shrinks every size."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import oracle_lib as O

pytestmark = pytest.mark.gpu
SCALE = float(os.environ.get("FGB_FULL_SCALE", "1.0"))
L = 150
DEV = "cuda:0"


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as graft
    graft.build()
    import fgumi_b200
    return fgumi_b200


def _sample_rows(torch, tb, units_idx):
    """Source rows of the sampled units, copied from device memory -> [[(bases, quals), ...], ...]."""
    host = tb.host
    rb = host.units["read_begin"].astype(np.int64)
    Lp = (L + 7) // 8 * 8
    rows = np.concatenate([np.arange(rb[u], rb[u + 1]) for u in units_idx])
    idx = torch.from_numpy(rows).to(DEV)
    b = tb.bases.reshape(-1, Lp)[idx, :L].cpu().numpy()
    q = tb.quals.reshape(-1, Lp)[idx, :L].cpu().numpy()
    out, k = [], 0
    for u in units_idx:
        n = int(rb[u + 1] - rb[u])
        out.append([(b[k + i].tobytes(), q[k + i].tobytes()) for i in range(n)])
        k += n
    return out


def _gather_cols(torch, cols, offs, n):
    """Elements [off, off+n) of every output column for each off, as host arrays [len(offs), n]."""
    idx = (torch.from_numpy(np.asarray(offs, dtype=np.int64)).to(DEV)[:, None] +
           torch.arange(n, device=DEV)[None, :])
    return [c[idx].cpu().numpy() for c in cols]


def _check_sample_against_oracle(fg, torch, tb, out, sample, min_reads, min_q):
    units = _sample_rows(torch, tb, sample)
    pb = fg.pack_source_reads(units, min_reads)
    ob, oq, od, oe, cl = O.simplex_batch(pb, 45, 40, min_reads, min_q, 8)
    offs = tb.host.units["out_off"][sample].astype(np.int64)
    gb, gq, gd, ge = _gather_cols(torch, (out.base, out.qual, out.depth, out.errors), offs, L)
    for k, sl in enumerate(pb.unit_slices()):
        n = sl.stop - sl.start
        assert n == int(tb.host.units["cons_len"][sample[k]])
        assert np.array_equal(gb[k][:n], ob[sl]), sample[k]
        assert np.array_equal(gq[k][:n], oq[sl]), sample[k]
        assert np.array_equal(gd[k][:n].view(np.uint16), od[sl]), sample[k]
        assert np.array_equal(ge[k][:n].view(np.uint16), oe[sl]), sample[k]
    return pb, (ob, oq, od, oe)


def _check_slice_against_oracle(fg, torch, tb, out, depths, min_reads, min_q, max_rows=2_000_000, where=0.37):
    """EVERY unit of one contiguous slice of the batch (up to `max_rows` source rows, starting `where` of the way
    in) against a full oracle pass over the same rows copied back from device memory: all four columns, every
    called position.  The sampled comparison above draws units from everywhere; this one leaves no gaps."""
    from fgumi_b200 import synth
    host = tb.host
    U = host.n_units
    rb = host.units["read_begin"].astype(np.int64)
    Lp, Lo = (L + 7) // 8 * 8, (L + 7) // 8 * 8
    u0 = int(U * where)
    u1 = int(np.searchsorted(rb, rb[u0] + max_rows, side="right")) - 1
    u1 = max(u0 + 1, min(U, u1))
    pb = synth.make_descriptors(depths[u0:u1], L, min_reads)
    r0, r1 = int(rb[u0]), int(rb[u1])
    pad = np.zeros(16, np.uint8)
    pb.bases = np.concatenate([tb.bases.reshape(-1)[r0 * Lp:r1 * Lp].cpu().numpy(), pad])
    pb.quals = np.concatenate([tb.quals.reshape(-1)[r0 * Lp:r1 * Lp].cpu().numpy(), pad])
    ob, oq, od, oe, cl = O.simplex_batch(pb, 45, 40, min_reads, min_q, max(1, min(32, os.cpu_count() or 1)))
    o0 = int(host.units["out_off"][u0])
    n = (u1 - u0) * Lo
    assert int(host.units["out_off"][u1]) - o0 == n and pb.n_out == n
    assert np.array_equal(cl, host.units["cons_len"][u0:u1])
    valid = (np.arange(Lo)[None, :] < cl.astype(np.int64)[:, None]).reshape(-1)
    for name, g, o in (("base", out.base, ob), ("qual", out.qual, oq), ("depth", out.depth, od), ("errors", out.errors, oe)):
        got = g[o0:o0 + n].cpu().numpy()
        if got.dtype != o.dtype:
            got = got.view(o.dtype)
        bad = np.flatnonzero((got != o[:n]) & valid)
        assert bad.size == 0, (name, u0 + int(bad[0]) // Lo, int(bad[0]) % Lo, bad.size)
    _LAST_SLICE.clear()
    _LAST_SLICE.update(u0=u0, u1=u1, pb=pb, cols=(ob, oq, od, oe, cl))
    return u1 - u0


_LAST_SLICE = {}      # the slice the last _vote_and_check compared in full, with the oracle's columns for it


def _invariants(torch, out, depth_max):
    d, e = out.depth.view(torch.int16), out.errors.view(torch.int16)
    assert int(d.max()) <= depth_max and int(d.min()) >= 0
    assert bool((e <= d).all())
    q = out.qual
    assert int(q.max()) <= 93


def _vote_and_check(fg, torch, tb, depths, min_reads=1, min_q=2, n_sample=1500, seed=0):
    from fgumi_b200 import synth
    eng = fg.Engine(0, 45, 40, min_reads, min_q)
    out = fg.DeviceColumns(tb.host.n_out, DEV)
    s = torch.cuda.current_stream().cuda_stream
    eng.vote_device(tb, out, s)
    torch.cuda.synchronize()
    st = eng.stats()
    U = tb.host.n_units
    assert st["units"] == U and st["input_reads"] == int(depths.sum())
    assert st["positions"] == int(tb.host.units["cons_len"][:U].astype(np.int64).sum())
    _invariants(torch, out, int(depths.max()))
    # a second launch is bit-identical
    out2 = fg.DeviceColumns(tb.host.n_out, DEV)
    eng.vote_device(tb, out2, s)
    torch.cuda.synchronize()
    for a, b in ((out.base, out2.base), (out.qual, out2.qual), (out.depth, out2.depth), (out.errors, out2.errors)):
        assert torch.equal(a, b)
    del out2
    # the prefix voted as its own (differently tiled) batch equals the prefix of the full result
    P = max(1, U // 7)
    sub_host = synth.make_descriptors(depths[:P], L, min_reads)
    sub = synth.TorchBatch(tb.bases, tb.quals, tb.reads, tb.units.clone(),
                           torch.from_numpy(sub_host.tiles.view(np.uint8).reshape(-1)).to(DEV), sub_host)
    # the sub-batch needs its own sentinel unit: reuse the descriptor array the planner saw
    sub.units = torch.from_numpy(sub_host.units.view(np.uint8).reshape(-1)).to(DEV)
    outp = fg.DeviceColumns(sub_host.n_out, DEV)
    eng.vote_device(sub, outp, s)
    torch.cuda.synchronize()
    n = sub_host.n_out
    assert torch.equal(outp.base[:n], out.base[:n]) and torch.equal(outp.qual[:n], out.qual[:n])
    assert torch.equal(outp.depth[:n], out.depth[:n]) and torch.equal(outp.errors[:n], out.errors[:n])
    del outp
    rng = np.random.default_rng(seed)
    sample = np.sort(rng.choice(U, size=min(n_sample, U), replace=False))
    _check_sample_against_oracle(fg, torch, tb, out, sample, min_reads, min_q)
    _check_slice_against_oracle(fg, torch, tb, out, depths, min_reads, min_q)
    return eng, out


def test_config2_simplex_10m_depth8(fg):
    import torch
    from fgumi_b200 import synth
    U = max(1000, int(10_000_000 * SCALE))
    depths = np.full(U, 8, dtype=np.int64)
    tb = synth.device_batch(torch, DEV, depths, L, 1e-3, seed=42)
    eng, out = _vote_and_check(fg, torch, tb, depths, seed=2)
    st = eng.stats()
    assert st["exact_positions"] < st["positions"] // 10_000     # the proofs decide almost everything
    eng.close()


def test_config5_zipf_shard(fg):
    import torch
    from fgumi_b200 import synth
    U = max(1000, int(6_250_000 * SCALE))          # ~120 M source rows (37 GB) + two output sets
    depths = synth.zipf_depths(U, 1, 100, 1.0, seed=42 + 3)          # rank 3's shard: seed 42+rank
    tb = synth.device_batch(torch, DEV, depths, L, 1e-3, seed=45)
    eng, out = _vote_and_check(fg, torch, tb, depths, n_sample=600, seed=5)
    eng.close()


def test_config3_duplex_5m_molecules(fg):
    import torch
    from fgumi_b200 import synth
    M = max(500, int(5_000_000 * SCALE))
    U = 4 * M                                                         # AB-R1, AB-R2, BA-R1, BA-R2
    depths = np.full(U, 4, dtype=np.int64)
    m = np.arange(M, dtype=np.int64)
    tid = np.empty(U, dtype=np.int64)                                 # AB-R1 & BA-R2 see one template,
    tid[0::4], tid[3::4] = 2 * m, 2 * m                               # AB-R2 & BA-R1 the other
    tid[1::4], tid[2::4] = 2 * m + 1, 2 * m + 1
    tb = synth.device_batch(torch, DEV, depths, L, 1e-3, seed=43, template_ids=tid)
    eng, ss = _vote_and_check(fg, torch, tb, depths, min_reads=1, min_q=2, n_sample=400, seed=3)
    Lo = (L + 7) // 8 * 8
    jobs = np.zeros(2 * M, dtype=fg.DUPLEX_JOB_DTYPE)
    jobs["unit_a"][0::2], jobs["unit_b"][0::2] = 4 * m, 4 * m + 3    # duplex_caller.rs:1999-2012
    jobs["unit_a"][1::2], jobs["unit_b"][1::2] = 4 * m + 1, 4 * m + 2
    jobs["out_off"] = np.arange(2 * M, dtype=np.uint64) * np.uint64(Lo)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(DEV)
    n_out = 2 * M * Lo
    o_base = torch.zeros(n_out, dtype=torch.uint8, device=DEV)
    o_qual = torch.zeros(n_out, dtype=torch.uint8, device=DEV)
    o_err = torch.zeros(n_out, dtype=torch.int16, device=DEV)
    o_st = torch.full((2 * M,), 255, dtype=torch.uint8, device=DEV)
    eng.stats_reset()
    eng.duplex_combine_device(tb, ss, tj, 2 * M, o_base, o_qual, o_err, o_st,
                              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert eng.stats()["combined_jobs"] == 2 * M
    assert int(o_st.max()) == 0 and int(o_st.min()) == 0              # every molecule has both strands
    # strands share a template and errors are rare: nearly every duplex base is called
    called = (o_base.reshape(-1, Lo)[:, :L] != ord("N")).float().mean().item()
    assert called > 0.99
    # sampled jobs against the oracle (SS columns from the oracle vote of the same rows)
    rng = np.random.default_rng(33)
    sj = np.sort(rng.choice(2 * M, size=min(400, 2 * M), replace=False))
    lib = O.load()
    ua, ub = jobs["unit_a"][sj].astype(np.int64), jobs["unit_b"][sj].astype(np.int64)
    both = np.stack([ua, ub], 1).reshape(-1)
    units = _sample_rows(torch, tb, both)
    pb = fg.pack_source_reads(units, 1)
    ob, oq, od, oe, cl = O.simplex_batch(pb, 45, 40, 1, 2, 8)
    gb, gq, ge = _gather_cols(torch, (o_base, o_qual, o_err), jobs["out_off"][sj].astype(np.int64), L)
    oo = pb.units["out_off"]
    for k in range(len(sj)):
        a, b = 2 * k, 2 * k + 1
        rows = units[a] + units[b]
        keep = [np.frombuffer(r[0], np.uint8).copy() for r in rows]
        ptrs = (C.c_void_p * len(rows))(*[x.ctypes.data for x in keep])
        lens = (C.c_size_t * len(rows))(*[len(r[0]) for r in rows])
        rb = np.zeros(L, np.uint8); rq = np.zeros(L, np.uint8); re_ = np.zeros(L, np.uint16)
        olen = C.c_size_t()
        oa, obo = int(oo[a]), int(oo[b])
        st = lib.orc_duplex_job(ob[oa:].ctypes.data, oq[oa:].ctypes.data, od[oa:].ctypes.data,
                                oe[oa:].ctypes.data, int(cl[a]), ob[obo:].ctypes.data, oq[obo:].ctypes.data,
                                od[obo:].ctypes.data, oe[obo:].ctypes.data, int(cl[b]), ptrs, lens, len(rows),
                                rb.ctypes.data, rq.ctypes.data, re_.ctypes.data, C.addressof(olen))
        n = olen.value
        assert st == 0 and n == L
        assert np.array_equal(gb[k][:n], rb[:n]) and np.array_equal(gq[k][:n], rq[:n])
        assert np.array_equal(ge[k][:n].view(np.uint16), re_[:n])
    # the combine in the vote kernels' epilogue (fgb_plan_tiles_jobs + fgb_vote_duplex_device): every called position
    # of all 10 M jobs, and the SS columns, equal the two-kernel form's; every job ran in the epilogue
    tiles, class_tiles, tile_jobs, job_index, n_attached = fg.plan_tiles_jobs(tb.host, jobs)
    assert n_attached == 2 * M
    t8 = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(DEV)
    tbf = synth.TorchBatch(tb.bases, tb.quals, tb.reads, tb.units, t8(tiles), tb.host, class_tiles)
    tbf.n_tiles = len(tiles)
    d_tj, d_ji = t8(tile_jobs), t8(job_index)
    ss2 = fg.DeviceColumns(tb.host.n_out, DEV)
    f_base = torch.zeros_like(o_base); f_qual = torch.zeros_like(o_qual); f_err = torch.zeros_like(o_err)
    f_st = torch.full((2 * M,), 77, dtype=torch.uint8, device=DEV)
    eng.stats_reset()
    eng.vote_duplex_device(tbf, ss2, tj, 2 * M, d_tj, d_ji, f_base, f_qual, f_err, f_st,
                           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    s2 = eng.stats()
    assert s2["combined_jobs"] == 2 * M and s2["units"] == U and int(f_st.max()) == 0
    valid = lambda x: x.reshape(-1, Lo)[:, :L]
    for got, want in ((f_base, o_base), (f_qual, o_qual), (f_err, o_err), (ss2.base[:U * Lo], ss.base[:U * Lo]),
                      (ss2.qual[:U * Lo], ss.qual[:U * Lo]), (ss2.depth[:U * Lo], ss.depth[:U * Lo]),
                      (ss2.errors[:U * Lo], ss.errors[:U * Lo])):
        assert torch.equal(valid(got), valid(want))
    del ss2, f_base, f_qual, f_err, tbf
    # ... and EVERY job of a contiguous run inside the slice the vote check compared in full (the oracle's own SS
    # columns for those units are at hand): up to 20 000 jobs, all three columns, every position
    u0, u1, spb, (sb_, sq_, sd_, se_, scl) = (_LAST_SLICE[k] for k in ("u0", "u1", "pb", "cols"))
    j0, j1 = (u0 + 3) // 4 * 2, min(u1 // 4 * 2, (u0 + 3) // 4 * 2 + 20_000)
    assert j1 > j0
    soo = spb.units["out_off"].astype(np.int64)
    srb = spb.units["read_begin"].astype(np.int64)
    Lp = (L + 7) // 8 * 8
    srows = spb.bases[: spb.n_reads * Lp].reshape(-1, Lp)
    gb = o_base[j0 * Lo:j1 * Lo].cpu().numpy().reshape(-1, Lo)
    gq = o_qual[j0 * Lo:j1 * Lo].cpu().numpy().reshape(-1, Lo)
    ge = o_err[j0 * Lo:j1 * Lo].cpu().numpy().view(np.uint16).reshape(-1, Lo)
    rb = np.zeros(L, np.uint8); rq = np.zeros(L, np.uint8); re_ = np.zeros(L, np.uint16)
    olen = C.c_size_t()
    for j in range(j0, j1):
        a, b = int(jobs["unit_a"][j]) - u0, int(jobs["unit_b"][j]) - u0
        ridx = list(range(srb[a], srb[a + 1])) + list(range(srb[b], srb[b + 1]))
        ptrs = (C.c_void_p * len(ridx))(*[srows[r].ctypes.data for r in ridx])
        lens = (C.c_size_t * len(ridx))(*([L] * len(ridx)))
        oa, obo = int(soo[a]), int(soo[b])
        st = lib.orc_duplex_job(sb_[oa:].ctypes.data, sq_[oa:].ctypes.data, sd_[oa:].ctypes.data,
                                se_[oa:].ctypes.data, int(scl[a]), sb_[obo:].ctypes.data, sq_[obo:].ctypes.data,
                                sd_[obo:].ctypes.data, se_[obo:].ctypes.data, int(scl[b]), ptrs, lens, len(ridx),
                                rb.ctypes.data, rq.ctypes.data, re_.ctypes.data, C.addressof(olen))
        n = olen.value
        assert st == 0 and n == L, j
        k = j - j0
        assert np.array_equal(gb[k][:n], rb[:n]) and np.array_equal(gq[k][:n], rq[:n]), j
        assert np.array_equal(ge[k][:n], re_[:n]), j
    eng.close()


def test_config4_codec_2m_molecules(fg):
    import torch
    from fgumi_b200 import synth
    M = max(500, int(2_000_000 * SCALE))
    rng = np.random.default_rng(44)
    k = rng.integers(2, 21, size=M)                                   # pairs per molecule, U[2,20]
    depths = np.repeat(k, 2).astype(np.int64)                         # unit 2m = R1s, 2m+1 = R2s
    tb = synth.device_batch(torch, DEV, depths, L, 1e-3, seed=44)
    eng, ss = _vote_and_check(fg, torch, tb, depths, min_reads=1, min_q=0, n_sample=300, seed=4)
    insert = np.clip(np.round(rng.normal(300, 50, size=M)), L, 2 * L).astype(np.int64)   # Lc = insert
    Lc_pad = (insert + 7) // 8 * 8
    jobs = np.zeros(M, dtype=fg.CODEC_JOB_DTYPE)
    r1_neg = rng.random(M) < 0.5
    jobs["unit_a"], jobs["unit_b"] = 2 * np.arange(M), 2 * np.arange(M) + 1
    jobs["out_off"][1:] = np.cumsum(Lc_pad)[:-1]
    jobs["len"] = insert
    jobs["rc_a"], jobs["rc_b"], jobs["rc_out"] = r1_neg, ~r1_neg, r1_neg
    jobs["pad_a_left"] = np.where(r1_neg, insert - L, 0)
    jobs["pad_b_left"] = np.where(~r1_neg, insert - L, 0)             # R2 negative when R1 is not
    n_out = int(Lc_pad.sum())
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(DEV)
    out = fg.DeviceColumns(n_out, DEV)
    st = torch.full((M,), 255, dtype=torch.uint8, device=DEV)
    dis = torch.zeros(M, dtype=torch.int32, device=DEV)
    dup = torch.zeros(M, dtype=torch.int32, device=DEV)
    cp = fg.lib.FgbCodecParams(-1, -1, 5, 0xFFFFFFFF, 1.0)
    eng.stats_reset()
    eng.codec_combine_device(tb, ss, tj, M, cp, out, st, dis, dup, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    s = eng.stats()
    assert s["combined_jobs"] == M and int(st.max()) == 0
    assert s["duplex_bases"] == int(dup.sum().item()) and s["duplex_disagreements"] == int(dis.sum().item())
    overlap = int((2 * L - insert).sum())                             # 2L - Lc positions per molecule
    assert 0.97 * overlap < s["duplex_bases"] <= overlap              # minus the few no-call positions
    # sampled molecules against the oracle
    sm = np.sort(rng.choice(M, size=min(300, M), replace=False))
    both = np.stack([2 * sm, 2 * sm + 1], 1).reshape(-1)
    units = _sample_rows(torch, tb, both)
    pb = fg.pack_source_reads(units, 1)
    ob, oq, od, oe, cl = O.simplex_batch(pb, 45, 40, 1, 0, 8)
    oo = pb.units["out_off"]
    lib = O.load()
    gs, gdis, gdup = st.cpu().numpy(), dis.cpu().numpy(), dup.cpu().numpy()
    for i, m in enumerate(sm):
        clen = int(insert[m]); a, b = 2 * i, 2 * i + 1
        rb = np.zeros(clen, np.uint8); rq = np.zeros(clen, np.uint8)
        rd = np.zeros(clen, np.uint16); re_ = np.zeros(clen, np.uint16)
        nb, nd = C.c_uint64(), C.c_uint64()
        oa, obo = int(oo[a]), int(oo[b])
        rs = lib.orc_codec_job(ob[oa:].ctypes.data, oq[oa:].ctypes.data, od[oa:].ctypes.data,
                               oe[oa:].ctypes.data, int(cl[a]), ob[obo:].ctypes.data, oq[obo:].ctypes.data,
                               od[obo:].ctypes.data, oe[obo:].ctypes.data, int(cl[b]), int(r1_neg[m]),
                               int(not r1_neg[m]), clen, -1, -1, 5, 2 ** 62, 1.0, rb.ctypes.data,
                               rq.ctypes.data, rd.ctypes.data, re_.ctypes.data, C.addressof(nb), C.addressof(nd))
        g = _gather_cols(torch, (out.base, out.qual, out.depth, out.errors), [int(jobs["out_off"][m])], clen)
        assert gs[m] == rs and gdis[m] == nd.value and gdup[m] == nb.value
        assert np.array_equal(g[0][0], rb) and np.array_equal(g[1][0], rq)
        assert np.array_equal(g[2][0].view(np.uint16), rd) and np.array_equal(g[3][0].view(np.uint16), re_)
    eng.close()
