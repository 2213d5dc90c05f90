"""GPU parity of the strand-combine kernels (K2 duplex, K3 CODEC) through the C-ABI against the
oracle.  Pure integer work: everything must match bit-exact."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as graft
    graft.build()
    import fgumi_b200
    return fgumi_b200


def _family(rng, depth, length, err=0.05, n_rate=0.03, all_n=False, qlo=5, qhi=41):
    tmpl = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=length)
    rows = []
    for _ in range(depth):
        b = tmpl.copy()
        m = rng.random(length) < err
        b[m] = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=int(m.sum()))
        q = rng.integers(qlo, qhi + 1, size=length).astype(np.uint8)
        nm = rng.random(length) < n_rate
        if all_n:
            nm[:] = True
        b[nm] = ord("N")
        q[nm] = 2
        rows.append((b.tobytes(), q.tobytes()))
    return rows, tmpl


def _vote(fg, units, min_cons_q):
    """Single-strand vote on the GPU (device-resident) + the oracle's SS columns."""
    import torch
    batch = fg.pack_source_reads(units, 1)
    eng = fg.Engine(0, 45, 40, 1, min_cons_q)
    db = fg.DeviceBatch(batch, "cuda:0")
    ss = fg.DeviceColumns(batch.n_out, "cuda:0")
    eng.vote_device(db, ss, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ob, oq, od, oe, _ = O.simplex_batch(batch, 45, 40, 1, min_cons_q)
    g = ss.to_host()
    n = batch.n_out
    for sl in batch.unit_slices():
        assert np.array_equal(g.base[sl], ob[sl]) and np.array_equal(g.qual[sl], oq[sl])
        assert np.array_equal(g.depth[sl], od[sl]) and np.array_equal(g.errors[sl], oe[sl])
    return eng, batch, db, ss, (ob, oq, od, oe)


def _duplex_against_oracle(fg, units, pairs, fused, min_cons_q=2, want_status=True):
    """Vote `units`, combine `pairs` (standalone K2, or in the vote kernels' epilogue with `fused`) and compare every
    job with the oracle's duplex_consensus over the oracle's own SS columns.  Returns the set of arms seen."""
    import torch
    L = O.load()
    dev = "cuda:0"
    batch = fg.pack_source_reads(units, 1)
    cons_len = batch.units["cons_len"]
    out_off = batch.units["out_off"]
    jobs = np.zeros(len(pairs), dtype=fg.DUPLEX_JOB_DTYPE)
    off = 0
    for j, (ua, ub) in enumerate(pairs):
        jobs[j] = (ua, ub, off)
        off += (max(int(cons_len[ua]), int(cons_len[ub])) + 7) // 8 * 8
    n_out = max(off, 8)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(dev)
    o_base = torch.zeros(n_out, dtype=torch.uint8, device=dev)
    o_qual = torch.zeros(n_out, dtype=torch.uint8, device=dev)
    o_err = torch.zeros(n_out, dtype=torch.int16, device=dev)
    o_st = torch.full((len(pairs),), 77, dtype=torch.uint8, device=dev)
    eng = fg.Engine(0, 45, 40, 1, min_cons_q)
    db = fg.DeviceBatch(batch, dev)
    ss = fg.DeviceColumns(batch.n_out, dev)
    stream = torch.cuda.current_stream().cuda_stream
    n_attached = None
    if fused:
        tiles, class_tiles, tile_jobs, job_index, n_attached = fg.plan_tiles_jobs(batch, jobs)
        t8 = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)
        db.tiles, db.n_tiles, db.class_tiles = t8(tiles), len(tiles), class_tiles
        d_tj, d_ji = t8(tile_jobs), t8(job_index)
        eng.vote_duplex_device(db, ss, tj, len(pairs), d_tj, d_ji, o_base, o_qual, o_err,
                               o_st if want_status else None, stream)
    else:
        eng.vote_device(db, ss, stream)
        eng.duplex_combine_device(db, ss, tj, len(pairs), o_base, o_qual, o_err, o_st, stream)
    torch.cuda.synchronize()
    ob, oq, od, oe, _ = O.simplex_batch(batch, 45, 40, 1, min_cons_q)
    g = ss.to_host()
    for sl in batch.unit_slices():
        assert np.array_equal(g.base[sl], ob[sl]) and np.array_equal(g.qual[sl], oq[sl])
        assert np.array_equal(g.depth[sl], od[sl]) and np.array_equal(g.errors[sl], oe[sl])
    gb, gq = o_base.cpu().numpy(), o_qual.cpu().numpy()
    ge, gs = o_err.cpu().numpy().view(np.uint16), o_st.cpu().numpy()
    st_ = eng.stats()
    assert st_["combined_jobs"] == len(pairs)
    assert st_["units"] == len(units)
    eng.close()
    seen = set()
    for j, (ua, ub) in enumerate(pairs):
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
        seen.add(st)
        if want_status:
            assert gs[j] == st, (j, gs[j], st)
        o = int(jobs[j]["out_off"]); n = olen.value
        assert np.array_equal(gb[o:o + n], rb[:n]), j
        assert np.array_equal(gq[o:o + n], rq[:n]), j
        assert np.array_equal(ge[o:o + n], re_[:n]), j
    return seen, n_attached


def _duplex_molecules(rng, n_mol, depth_hi=6, len_lo=20, len_hi=90, iupac=False):
    units = []
    for m in range(n_mol):
        # AB-R1, AB-R2, BA-R1, BA-R2 single-strand families; a few strands carry no coverage at all
        for k in range(4):
            depth = int(rng.integers(1, depth_hi))
            length = int(rng.integers(len_lo, len_hi))
            dead = (m % 17 == 3 and k >= 2) or (m % 23 == 5 and k < 2) or (m % 29 == 7)
            rows, _ = _family(rng, depth, length, all_n=dead)
            if iupac and m % 5 == 1:      # codes the vote ignores but the exact recount counts (and a lower-case base)
                b = bytearray(rows[0][0])
                b[int(rng.integers(0, len(b)))] = ord("R")
                b[int(rng.integers(0, len(b)))] = ord("a")
                rows[0] = (bytes(b), rows[0][1])
            units.append(rows)
    # duplex R1 = AB-R1 (+) BA-R2, duplex R2 = AB-R2 (+) BA-R1   (duplex_caller.rs:1999-2012)
    pairs = []
    for m in range(n_mol):
        pairs.append((4 * m + 0, 4 * m + 3))
        pairs.append((4 * m + 1, 4 * m + 2))
    return units, pairs


@pytest.mark.parametrize("fused", [False, True])
def test_duplex_combine_matches_oracle(fg, fused):
    rng = np.random.default_rng(31)
    units, pairs = _duplex_molecules(rng, 300)
    seen, n_attached = _duplex_against_oracle(fg, units, pairs, fused)
    assert seen == {0, 1, 2, 3}     # every arm of duplex_consensus was exercised
    if fused:
        assert n_attached == len(pairs)      # a molecule's four small units always fit one stage


@pytest.mark.parametrize("fused", [False, True])
def test_duplex_combine_mixed_classes_and_odd_jobs(fg, fused):
    """Strand depths from 1 to 40 (shallow, general and deep units inside one molecule), 150-base reads, codes outside
    A/C/G/T/N in the source rows, jobs in shuffled order, and jobs whose units lie far apart (never attached to a
    tile: the standalone kernel takes them after the vote)."""
    rng = np.random.default_rng(32)
    units, pairs = _duplex_molecules(rng, 160, depth_hi=41, len_lo=120, len_hi=151, iupac=True)
    n_mol = len(units) // 4
    for m in range(0, n_mol - 40, 7):                           # far-apart partners (and a repeated unit)
        pairs.append((4 * m, 4 * (m + 37) + 2))
    pairs.append((5, 5))
    order = rng.permutation(len(pairs))
    pairs = [pairs[i] for i in order]
    seen, n_attached = _duplex_against_oracle(fg, units, pairs, fused)
    assert {0, 1, 2} <= seen
    if fused:
        assert 3 * n_mol // 2 <= n_attached < len(pairs)


def test_duplex_epilogue_without_status_column(fg):
    """fgb_duplex_out.status may be NULL: the epilogue then keeps its pending marks in a buffer of the engine."""
    rng = np.random.default_rng(34)
    units, pairs = _duplex_molecules(rng, 150)
    seen, _ = _duplex_against_oracle(fg, units, pairs, True, want_status=False)
    assert seen == {0, 1, 2, 3}


def test_duplex_epilogue_uniform_molecules(fg):
    """BASELINE config 3's shape in small: 4 + 4 reads per strand, 150 bp, regular tiles of eight molecules."""
    rng = np.random.default_rng(33)
    units = []
    for m in range(700):
        for k in range(4):
            rows, _ = _family(rng, 4, 150, err=0.01, n_rate=0.002, qlo=20, qhi=40)
            units.append(rows)
    pairs = [p for m in range(700) for p in ((4 * m, 4 * m + 3), (4 * m + 1, 4 * m + 2))]
    seen, n_attached = _duplex_against_oracle(fg, units, pairs, True)
    assert seen == {0} and n_attached == len(pairs)


def test_duplex_known_answers(fg):
    """duplex_caller.rs:2494-2575 through the GPU: single-read strands with min_consensus_base_quality
    0 keep (base, LUT[q]); the KAT vectors use the raw combine rule, so feed quals whose LUT image is
    the wanted value."""
    import torch
    sq = O.tables(45, 40)[3]
    inv = {int(v): q for q, v in enumerate(sq)}          # LUT[q] -> q (any preimage)
    want = [20, 30, 37, 38]
    qa = bytes(inv[v] for v in want)
    units = [[(b"ACGT", qa)], [(b"ACGT", qa)], [(b"TGCA", bytes(inv[v] for v in (10, 15, 20, 25)))],
             [(b"TGCA", qa)]]
    eng, batch, db, ss, (ob, oq, od, oe) = _vote(fg, units, 0)
    jobs = np.zeros(3, dtype=fg.DUPLEX_JOB_DTYPE)
    jobs[0] = (0, 1, 0); jobs[1] = (0, 2, 8); jobs[2] = (0, 3, 16)
    dev = "cuda:0"
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(dev)
    o_base = torch.zeros(24, dtype=torch.uint8, device=dev)
    o_qual = torch.zeros(24, dtype=torch.uint8, device=dev)
    o_err = torch.zeros(24, dtype=torch.int16, device=dev)
    eng.duplex_combine_device(db, ss, tj, 3, o_base, o_qual, o_err, None,
                              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    eng.close()
    gb, gq = o_base.cpu().numpy(), o_qual.cpu().numpy()
    assert bytes(gb[0:4]) == b"ACGT" and list(gq[0:4]) == [min(93, 2 * v) for v in want]   # agreement
    assert bytes(gb[8:12]) == b"ACGT" and list(gq[8:12]) == [10, 15, 17, 13]              # higher wins
    assert bytes(gb[16:20]) == b"NNNN" and list(gq[16:20]) == [2, 2, 2, 2]                # equal quals


def test_codec_combine_matches_oracle(fg):
    import torch
    rng = np.random.default_rng(41)
    L = O.load()
    units, meta = [], []
    n_mol = 400
    for m in range(n_mol):
        k = int(rng.integers(1, 7))
        l1, l2 = int(rng.integers(12, 70)), int(rng.integers(12, 70))
        err = 0.3 if m % 11 == 4 else 0.04          # some molecules trip the disagreement gates
        r1, t1 = _family(rng, k, l1, err=err)
        # R2 shares sequence context with R1 (reverse complement of an overlapping window)
        r2, _ = _family(rng, k, l2, err=err)
        units += [r1, r2]
        cons_length = max(l1, l2) + int(rng.integers(0, 30))
        meta.append((bool(rng.integers(0, 2)), cons_length))
    eng, batch, db, ss, (ob, oq, od, oe) = _vote(fg, units, 0)
    cons_len = batch.units["cons_len"]; out_off = batch.units["out_off"]
    jobs = np.zeros(n_mol, dtype=fg.CODEC_JOB_DTYPE)
    off = 0
    for m, (r1_neg, clen) in enumerate(meta):
        la, lb = int(cons_len[2 * m]), int(cons_len[2 * m + 1])
        r2_neg = not r1_neg                       # FR pair
        jobs[m]["unit_a"] = 2 * m; jobs[m]["unit_b"] = 2 * m + 1
        jobs[m]["out_off"] = off; jobs[m]["len"] = clen
        jobs[m]["rc_a"] = r1_neg; jobs[m]["rc_b"] = not r1_neg; jobs[m]["rc_out"] = r1_neg
        jobs[m]["pad_a_left"] = clen - la if r1_neg else 0       # pad_consensus(.., r1_is_negative)
        jobs[m]["pad_b_left"] = clen - lb if r2_neg else 0
        off += (clen + 7) // 8 * 8
    for ss_q, outer_q, outer_len, max_dis, max_rate in ((-1, -1, 0, 1 << 30, 1.0), (10, 5, 7, 6, 0.2)):
        dev = "cuda:0"
        tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(dev)
        out = fg.DeviceColumns(off, dev)
        st = torch.full((n_mol,), 255, dtype=torch.uint8, device=dev)
        dis = torch.zeros(n_mol, dtype=torch.int32, device=dev)
        dup = torch.zeros(n_mol, dtype=torch.int32, device=dev)
        cp = fg.lib.FgbCodecParams(ss_q, outer_q, outer_len, min(max_dis, 0xFFFFFFFF), max_rate)
        eng.stats_reset()
        eng.codec_combine_device(db, ss, tj, n_mol, cp, out, st, dis, dup,
                                 torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        g = out.to_host()
        gs, gdis, gdup = st.cpu().numpy(), dis.cpu().numpy(), dup.cpu().numpy()
        tot_dup = tot_dis = 0
        statuses = set()
        for m, (r1_neg, clen) in enumerate(meta):
            ua, ub = 2 * m, 2 * m + 1
            la, lb = int(cons_len[ua]), int(cons_len[ub]); oa, obo = int(out_off[ua]), int(out_off[ub])
            rb = np.zeros(clen, np.uint8); rq = np.zeros(clen, np.uint8)
            rd = np.zeros(clen, np.uint16); re_ = np.zeros(clen, np.uint16)
            nb, nd = C.c_uint64(), C.c_uint64()
            rs = L.orc_codec_job(ob[oa:].ctypes.data, oq[oa:].ctypes.data, od[oa:].ctypes.data,
                                 oe[oa:].ctypes.data, la, ob[obo:].ctypes.data, oq[obo:].ctypes.data,
                                 od[obo:].ctypes.data, oe[obo:].ctypes.data, lb, int(r1_neg),
                                 int(not r1_neg), clen, ss_q, outer_q, outer_len,
                                 min(max_dis, 2 ** 62), max_rate, rb.ctypes.data, rq.ctypes.data,
                                 rd.ctypes.data, re_.ctypes.data, C.addressof(nb), C.addressof(nd))
            o = int(jobs[m]["out_off"])
            assert gs[m] == rs, m
            assert gdis[m] == nd.value and gdup[m] == nb.value, m
            assert np.array_equal(g.base[o:o + clen], rb), m
            assert np.array_equal(g.qual[o:o + clen], rq), m
            assert np.array_equal(g.depth[o:o + clen], rd), m
            assert np.array_equal(g.errors[o:o + clen], re_), m
            tot_dup += nb.value; tot_dis += nd.value
            statuses.add(rs)
        s = eng.stats()
        assert s["duplex_bases"] == tot_dup and s["duplex_disagreements"] == tot_dis
        if max_dis < 100:
            assert statuses == {0, 1, 2}
    eng.close()


class _UnitsOnly:
    """fgb_batch that carries just a unit table (all the CODEC combine reads of it)."""

    def __init__(self, fg, units, device):
        import torch
        self.units = torch.from_numpy(units.view(np.uint8).reshape(-1).copy()).to(device)
        self.n_units = len(units) - 1
        self._fg = fg

    def struct(self):
        z = 0
        return self._fg.lib.FgbBatch(self.n_units, 0, 0, 0, 0, z, z, z, self.units.data_ptr(), z, (C.c_uint64 * 3)(0, 0, 0))


_COMP = np.arange(256, dtype=np.uint8)
for _x, _y in zip(b"ACGTacgt", b"TGCATGCA"):
    _COMP[_x] = _y


def _codec_job_reference(L, cols, ua, ub, job, cp):
    """One fgb_codec_job through the oracle's padded combine + mask (orient / pad / re-orient done here with numpy:
    codec_caller.rs:507-520, 980-1023, 783-784)."""
    sb, sq, sd, se = cols
    ss_q, outer_q, outer_len = cp
    n = int(job["len"])

    def padded(u, pad, rc):
        o, l = int(u["out_off"]), int(u["cons_len"])
        b, q, d, e = sb[o:o + l], sq[o:o + l], sd[o:o + l], se[o:o + l]
        if rc:
            b, q, d, e = _COMP[b[::-1]], q[::-1], d[::-1], e[::-1]
        pb = np.full(n, ord("n"), np.uint8); pq = np.zeros(n, np.uint8)
        pd_ = np.zeros(n, np.uint16); pe = np.zeros(n, np.uint16)
        k = max(0, min(l, n - pad))
        pb[pad:pad + k], pq[pad:pad + k], pd_[pad:pad + k], pe[pad:pad + k] = b[:k], q[:k], d[:k], e[:k]
        return pb, pq, pd_, pe
    A = padded(ua, int(job["pad_a_left"]), bool(job["rc_a"]))
    B = padded(ub, int(job["pad_b_left"]), bool(job["rc_b"]))
    ob = np.zeros(n, np.uint8); oq = np.zeros(n, np.uint8); od = np.zeros(n, np.uint16); oe = np.zeros(n, np.uint16)
    nb, nd = C.c_uint64(), C.c_uint64()
    if n:
        L.orc_codec_combine(A[0].ctypes.data, A[1].ctypes.data, A[2].ctypes.data, A[3].ctypes.data,
                            B[0].ctypes.data, B[1].ctypes.data, B[2].ctypes.data, B[3].ctypes.data, n,
                            ob.ctypes.data, oq.ctypes.data, od.ctypes.data, oe.ctypes.data, C.addressof(nb), C.addressof(nd))
        L.orc_codec_mask(ob.ctypes.data, oq.ctypes.data, n, A[0].ctypes.data, B[0].ctypes.data, ss_q, outer_q, outer_len)
    if job["rc_out"]:
        ob, oq, od, oe = _COMP[ob[::-1]], oq[::-1], od[::-1], oe[::-1]
    return ob, oq, od, oe, nb.value, nd.value


def _codec_job_mix(fg, rng):
    """A unit table, CODEC jobs and single-strand host columns: every orientation combination, arbitrary pads, lengths
    from 0 to 1300, some output rows that are not 8-aligned, a few bases outside A/C/G/T/N and large depths / errors.
    Returns (units, jobs, (base, qual, depth, errors), output elements the jobs' rows span)."""
    n_jobs = 32 * 9 + 5
    UNIT = np.dtype([("out_off", "<u8"), ("read_begin", "<u4"), ("cons_len", "<u4")])
    units = np.zeros(2 * n_jobs + 1, dtype=UNIT)
    jobs = np.zeros(n_jobs, dtype=fg.CODEC_JOB_DTYPE)
    off = 0; ooff = 0
    for m in range(n_jobs):
        kind = m % 13
        for s in range(2):
            l = int(rng.integers(1, 200)) if kind != 7 else int(rng.integers(300, 1300))
            if kind == 9 and s == 1:
                l = 0
            units[2 * m + s]["out_off"] = off; units[2 * m + s]["cons_len"] = l
            off += (l + 7) // 8 * 8
        la, lb = int(units[2 * m]["cons_len"]), int(units[2 * m + 1]["cons_len"])
        n = max(la, lb) + int(rng.integers(0, 40))
        if kind == 5:
            n = max(0, min(la, lb) - int(rng.integers(0, 10)))      # strands longer than the consensus
        if kind == 11:
            n = 0
        jobs[m]["unit_a"], jobs[m]["unit_b"] = 2 * m, 2 * m + 1
        jobs[m]["len"] = n
        jobs[m]["rc_a"], jobs[m]["rc_b"], jobs[m]["rc_out"] = rng.integers(0, 2, 3)
        jobs[m]["pad_a_left"] = int(rng.integers(0, max(1, n - la + 1 if n >= la else 8)))
        jobs[m]["pad_b_left"] = int(rng.integers(0, max(1, n - lb + 1 if n >= lb else 8)))
        if kind == 3:
            ooff += int(rng.integers(1, 8))                          # this job's output row is not 8-aligned
        jobs[m]["out_off"] = ooff
        ooff += n if kind == 3 else (n + 7) // 8 * 8
        if kind == 3:
            ooff = (ooff + 7) // 8 * 8
    units[2 * n_jobs]["out_off"] = off
    sb = rng.choice(np.frombuffer(b"ACGTN", np.uint8), size=off + 16, p=[0.23, 0.23, 0.23, 0.23, 0.08])
    sq = rng.integers(0, 94, size=off + 16).astype(np.uint8)
    sq[rng.random(off + 16) < 0.1] = 2
    sd = rng.integers(0, 40, size=off + 16).astype(np.uint16)
    se = np.minimum(sd, rng.integers(0, 6, size=off + 16)).astype(np.uint16)
    big = rng.random(off + 16) < 0.01
    sd[big] = 65000; se[big] = rng.integers(0, 65536, size=int(big.sum()))
    for m in range(n_jobs):                                         # exotic bases in a few jobs
        if m % 13 == 2:
            o, l = int(units[2 * m]["out_off"]), int(units[2 * m]["cons_len"])
            if l:
                sb[o + int(rng.integers(0, l))] = rng.choice(np.frombuffer(b"acgtnRY", np.uint8))
    return units, jobs, (sb, sq, sd, se), ooff


def test_codec_combine_generic_jobs(fg):
    """Every orientation combination, arbitrary pads (strands may stick out of the consensus), lengths from 0 to
    beyond a thousand, output rows that are not 8-aligned (scalar jobs inside a word-kernel launch), single-strand
    columns with bases outside A/C/G/T/N (redo path), large depths / errors (u16 wrap-around): the kernel against the
    oracle's padded combine + mask with orientation done in numpy."""
    import torch
    L = O.load()
    L.orc_codec_combine.restype = None
    L.orc_codec_mask.restype = None
    rng = np.random.default_rng(77)
    dev = "cuda:0"
    units, jobs, (sb, sq, sd, se), ooff = _codec_job_mix(fg, rng)
    n_jobs = len(jobs)
    ss = fg.DeviceColumns(len(sb), dev)
    ss.base.copy_(torch.from_numpy(sb)); ss.qual.copy_(torch.from_numpy(sq))
    ss.depth.copy_(torch.from_numpy(sd.view(np.int16))); ss.errors.copy_(torch.from_numpy(se.view(np.int16)))
    db = _UnitsOnly(fg, units, dev)
    eng = fg.Engine(0, 45, 40, 1, 0)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(dev)
    for ss_q, outer_q, outer_len, max_dis, max_rate in ((-1, -1, 0, 0xFFFFFFFF, 1.0), (10, 7, 9, 12, 0.3)):
        out = fg.DeviceColumns(ooff + 8, dev)
        out.base.fill_(0x55); out.qual.fill_(0x55); out.depth.fill_(0x5555); out.errors.fill_(0x5555)
        st = torch.full((n_jobs,), 255, dtype=torch.uint8, device=dev)
        dis = torch.zeros(n_jobs, dtype=torch.int32, device=dev); dup = torch.zeros_like(dis)
        cp = fg.lib.FgbCodecParams(ss_q, outer_q, outer_len, max_dis, max_rate)
        eng.stats_reset()
        eng.codec_combine_device(db, ss, tj, n_jobs, cp, out, st, dis, dup, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        g = out.to_host()
        gs, gdis, gdup = st.cpu().numpy(), dis.cpu().numpy(), dup.cpu().numpy()
        written = np.zeros(ooff + 8, bool)
        tot_dup = tot_dis = 0
        for m in range(n_jobs):
            rb, rq, rd, re_, nb, nd = _codec_job_reference(L, (sb, sq, sd, se), units[2 * m], units[2 * m + 1], jobs[m],
                                                           (ss_q, outer_q, outer_len))
            o, n = int(jobs[m]["out_off"]), int(jobs[m]["len"])
            assert np.array_equal(g.base[o:o + n], rb), (m, m % 13)
            assert np.array_equal(g.qual[o:o + n], rq), (m, m % 13)
            assert np.array_equal(g.depth[o:o + n], rd), (m, m % 13)
            assert np.array_equal(g.errors[o:o + n], re_), (m, m % 13)
            assert gdup[m] == nb and gdis[m] == nd, (m, m % 13)
            want = 0
            if nb > 0:
                want = 1 if nd > max_dis else (2 if nd / nb > max_rate else 0)
            assert gs[m] == want, (m, m % 13)
            written[o:o + n] = True
            tot_dup += nb; tot_dis += nd
        # nothing outside the jobs' own rows is touched
        assert np.all(g.base[~written[:len(g.base)]] == 0x55) and np.all(g.qual[~written[:len(g.qual)]] == 0x55)
        assert np.all(g.depth[~written[:len(g.depth)]] == 0x5555) and np.all(g.errors[~written[:len(g.errors)]] == 0x5555)
        s = eng.stats()
        assert s["duplex_bases"] == tot_dup and s["duplex_disagreements"] == tot_dis and s["combined_jobs"] == n_jobs
    eng.close()
