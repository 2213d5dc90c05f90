"""GPU parity of every vote kernel form across error-rate and quality settings, at the edges of the host-built proof
tables (host_tables.cpp).

Each table the vote trusts without looking -- qt, qt3, sumt, pair_q, the dominant-winner proof and its depth limit
nmax2 -- is a function of (error_rate_pre_umi, error_rate_post_umi), and whether a proven call is written or masked
to N depends on min_reads and min_consensus_base_quality.  One seeded workload reaches the shallow, general and deep
kernels in each of their forms (lane groups, flat single-unit tiles, direct oversize units; regular and ragged rows)
at depths around the class, stage and nmax2 limits, and sweeps every majority quality 1..93 so that every threshold
of every table is crossed without the test knowing where it is.  The outputs (bases, qualities, depths, errors) and
the counters must be bit-identical to the CPU oracle, through the class kernels, through the general kernel alone
and through the host-buffer submit; duplex molecules built from the same depths go through both duplex paths."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O

pytestmark = pytest.mark.gpu

ACGT = np.frombuffer(b"ACGT", np.uint8)
IUPAC = np.frombuffer(b"RYKMSWBDHV", np.uint8)
LOWER = np.frombuffer(b"acgtn", np.uint8)
STAGE_READS = 512          # read descriptors per shared-memory stage (fgb_config.h kTileMaxReads)


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as graft
    graft.build()
    import fgumi_b200
    return fgumi_b200


def _tables(fg, pre, post):
    """(qt[256], fast_qual, nmax2) as the engine builds them."""
    lib = fg.lib.load()
    qt = np.zeros(256, np.uint8)
    fq = C.c_uint32()
    assert lib.fgb_host_tables(pre, post, None, None, None, None, qt.ctypes.data, C.addressof(fq)) == 0
    dfix = np.zeros(96, np.int32)
    g2 = C.c_int32()
    nmax2 = C.c_uint32()
    assert lib.fgb_host_proof_tables(pre, post, dfix.ctypes.data, C.addressof(g2), C.addressof(nmax2)) == 0
    return qt, fq.value, nmax2.value


def _min_cons_q(spec, fast_qual):
    """min_consensus_base_quality of a settings row: a number, or relative to phred(pre) ("fq", "fq+1")."""
    if isinstance(spec, int):
        return spec
    return fast_qual + (1 if spec == "fq+1" else 0)


class _Cycle:
    """Majority quality 1..93 and dissent count 0..4, each advanced once per position."""

    def __init__(self):
        self.i = 0

    def next(self):
        q, k = 1 + self.i % 93, self.i % 5
        self.i += 1
        return q, k


def _unit(rng, depth, lens, cyc):
    """One unit of `depth` rows with the given lengths.  Per position: a template base carried by the majority at
    the position's majority quality (a tenth of the majority rows higher), 0-4 dissenting rows -- read 0 among them
    a quarter of the time -- that are either all A/C/G/T at qualities >= the majority's (the near-unanimous proof's
    case) or any of A/C/G/T, N, IUPAC and lowercase at any quality, and now and then a row at Q0 or above Q93."""
    P = max(lens)
    tmpl = rng.choice(ACGT, size=P)
    B = np.repeat(tmpl[None, :], depth, 0)
    Q = np.empty((depth, P), np.uint8)
    for p in range(P):
        qm, k = cyc.next()
        Q[:, p] = qm
        hi = np.flatnonzero(rng.random(depth) < 0.1)
        Q[hi, p] = rng.integers(qm, 94, size=hi.size)
        k = min(k, depth)
        if k:
            rows = rng.choice(depth, size=k, replace=False)
            if 0 not in rows and rng.random() < 0.25:
                rows[0] = 0
            acgt_only = rng.random() < 0.6
            others = ACGT[ACGT != tmpl[p]]
            for r in rows:
                x = 0.0 if acgt_only else rng.random()
                b = (rng.choice(others) if x < 0.4 else ord("N") if x < 0.6 else rng.choice(IUPAC) if x < 0.8
                     else rng.choice(LOWER))
                B[r, p] = b
                Q[r, p] = rng.integers(qm, 94) if acgt_only or rng.random() < 0.6 else rng.integers(1, 94)
        if rng.random() < 0.05:
            Q[rng.integers(depth), p] = rng.choice([0, 94, 120, 255])
    return [(B[r, :lens[r]].tobytes(), Q[r, :lens[r]].tobytes()) for r in range(depth)]


def _depth_ladder(nmax2):
    """Class limits (4/5, 23/24/25), the flat form's 64, 255 (the last depth with its own table entries), the stage's
    512 read descriptors, and nmax2 / nmax2 + 1 where they fall in 2..512."""
    ds = {2, 3, 4, 5, 23, 24, 25, 63, 64, 65, 254, 255, 256, 511, 512, 513}
    ds |= {d for d in (nmax2, nmax2 + 1) if 2 <= d <= 512}
    return sorted(ds)


def _workload(rng, ladder, reps=3):
    """Units of every ladder depth in a regular half (one read length per depth, 16-24) and a ragged half (lengths
    16-24 per read).  Each depth comes as a run of `reps` units (multi-unit tiles where a stage holds them) and as
    `reps` units isolated between units of another class (single-unit tiles: the flat form from 64 reads), started
    on alternating read parities.  Returns (units, per-unit (depth, ragged) list)."""
    units, meta = [], []
    n_reads = 0

    def add(depth, ragged, cyc):
        nonlocal n_reads
        if ragged:
            lens = [int(x) for x in rng.integers(16, 25, size=depth)]
            if depth > 1 and len(set(lens)) == 1:
                lens[0] = 16 if lens[0] != 16 else 17
        else:
            lens = [L] * depth
        units.append(_unit(rng, depth, lens, cyc))
        meta.append((depth, ragged))
        n_reads += depth

    for ragged in (False, True):
        for i, d in enumerate(ladder):
            L = (16, 20, 24, 17, 23)[i % 5]
            cyc = _Cycle()
            for _ in range(reps):
                add(d, ragged, cyc)
            sep = (5, 6) if d <= 4 else (2, 3)
            for r in range(reps):
                s = sep[0] if (n_reads + sep[0]) % 2 == r % 2 else sep[1]
                add(s, ragged, _Cycle())
                add(d, ragged, cyc)
    return units, meta


def _assert_forms(fg, batch, meta, min_reads):
    """Every kernel form is reached in regular and in ragged form, and a unit is voted from HBM exactly when its
    reads do not fit one stage's descriptors (one fewer when it starts at an odd read index).  A unit with fewer
    than min_reads reads calls no position, so its tile is not regular: min_reads = 25 leaves only the deep class
    regular."""
    tiles = fg.plan_tiles(batch)
    forms = set()
    direct_seen = set()
    for t in tiles:
        f = int(t["flags"])
        cls, direct, regular = (f >> 4) & 3, bool(f & 1), bool(f & 2)
        u0, nu = int(t["unit_begin"]), int(t["n_units"])
        if direct:
            forms.add(("direct", meta[u0][1]))
        elif cls == 2:
            forms.add(("lanes" if nu > 1 else "flat" if t["n_reads"] >= 64 else "single", regular))
        else:
            forms.add(("shallow" if cls == 1 else "general", regular))
        for u in range(u0, u0 + nu):
            d = meta[u][0]
            rb = int(batch.units["read_begin"][u])
            assert direct == (d + (rb & 1) > STAGE_READS), (u, d, rb, f)
            if d >= STAGE_READS - 1:
                direct_seen.add((d, rb & 1, direct))
    want = {(k, r) for k in ("shallow", "general", "lanes", "flat") for r in (True, False)}
    want |= {("direct", False), ("direct", True)}
    if min_reads > 4:
        want -= {("shallow", True), ("general", True)}
    assert want <= forms, sorted(want - forms)
    assert {(511, 1, False), (512, 0, False), (512, 1, True), (513, 0, True)} <= direct_seen, sorted(direct_seen)


def _compare(out, ref, batch, stats, tag):
    ob, oq, od, oe, _ = ref
    n = batch.n_out
    mask = np.zeros(max(n, 1), bool)
    for sl in batch.unit_slices():
        mask[sl] = True
    mask = mask[:n]
    for name, g, r in (("bases", out.base, ob), ("qualities", out.qual, oq), ("depths", out.depth, od),
                       ("errors", out.errors, oe)):
        g, r = g[:n][mask], r[:n][mask]
        bad = np.flatnonzero(g != r)
        assert bad.size == 0, f"{tag}: {bad.size} {name} differ, first at {bad[:5]}: {g[bad[:5]]} vs {r[bad[:5]]}"
    assert stats["positions"] == int(mask.sum()), tag
    assert stats["nocall_positions"] == int((ob[:n][mask] == ord("N")).sum()), tag
    assert stats["units"] == batch.n_units, tag
    assert stats["input_reads"] == batch.n_reads, tag


# (pre, post, min_reads, min_consensus_base_quality); "fq" = phred(pre), the quality every proven call carries
SETTINGS = [
    (45, 40, 1, 2), (45, 40, 25, 30),
    (30, 20, 1, "fq+1"), (30, 20, 3, "fq"),          # proven calls masked to N/Q2 / kept
    (10, 45, 1, "fq+1"), (10, 45, 25, "fq"),
    (93, 93, 1, 2), (85, 93, 3, 2), (80, 93, 1, 20), (80, 10, 1, 2),   # nmax2 inside the depth range
    (3, 3, 1, 2), (2, 2, 3, 2), (0, 40, 1, 2),       # one step of the unanimous table, phred(pre) clamped to 2
    (45, 1, 1, 2), (45, 0, 1, 2),                    # every D negative; tables not finite (no proof at all)
]


@pytest.mark.parametrize("pre,post,min_reads,mcq", SETTINGS, ids=lambda v: str(v))
def test_vote_forms_across_settings(fg, pre, post, min_reads, mcq):
    import torch
    qt, fast_qual, nmax2 = _tables(fg, pre, post)
    min_cons_q = _min_cons_q(mcq, fast_qual)
    # sanity: the settings sit where they are meant to
    if post == 0:
        assert nmax2 == 0
    if post == 1:
        assert (qt == 255).all()
    if mcq == "fq+1":
        assert min_cons_q > fast_qual and (qt[2:] <= 93).any()
    rng = np.random.default_rng(pre * 1000 + post * 10 + min_reads)
    units, meta = _workload(rng, _depth_ladder(nmax2))
    batch = fg.pack_source_reads(units, min_reads)
    _assert_forms(fg, batch, meta, min_reads)
    ref = O.simplex_batch(batch, pre, post, min_reads, min_cons_q, 8)

    for way in ("sorted", "unsorted", "submit"):
        eng = fg.Engine(0, pre, post, min_reads, min_cons_q)
        try:
            if way == "submit":
                out = eng.vote(batch)
            else:
                db = fg.DeviceBatch(batch, "cuda:0")
                if way == "unsorted":
                    db.class_tiles = (0, 0, 0)     # every tile through the general kernel
                dc = fg.DeviceColumns(batch.n_out, "cuda:0")
                eng.vote_device(db, dc, torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
                out = dc.to_host()
            stats = eng.stats()
        finally:
            eng.close()
        _compare(out, ref, batch, stats, f"{way} pre={pre} post={post} min_reads={min_reads} min_cons_q={min_cons_q}")


@pytest.mark.parametrize("pre,post", [(85, 93), (45, 40)])
def test_deep_lane_groups_across_the_end_of_qt3(fg, pre, post):
    """One deep tile of lane groups narrower than a warp whose units lie on both sides of an end of the near-unanimous
    table: depth nmax2 beside nmax2 + 1 where nmax2 is inside the deep class, else depth 24 beside 256 (qt3 ends at
    255).  The lane groups of one warp then disagree on whether the dissent counters are folded; the deep kernel used
    to fold them under that per-group condition with full-warp shuffles, and left positions unwritten."""
    import torch
    nmax2 = _tables(fg, pre, post)[2]
    depths = [nmax2, nmax2 + 1] * 2 if 24 <= nmax2 < 255 else [24, 256, 24, 24]
    rng = np.random.default_rng(11)
    units = [_unit(rng, d, [24] * d, _Cycle()) for d in depths]
    batch = fg.pack_source_reads(units, 1)
    tiles = fg.plan_tiles(batch)
    assert len(tiles) == 1 and (int(tiles[0]["flags"]) >> 4) & 3 == 2 and not tiles[0]["flags"] & 1
    ref = O.simplex_batch(batch, pre, post, 1, 2, 8)
    eng = fg.Engine(0, pre, post, 1, 2)
    try:
        db = fg.DeviceBatch(batch, "cuda:0")
        dc = fg.DeviceColumns(batch.n_out, "cuda:0")
        eng.vote_device(db, dc, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        out = dc.to_host()
        stats = eng.stats()
    finally:
        eng.close()
    _compare(out, ref, batch, stats, f"deep tile of depths {depths} at pre={pre} post={post}")


def test_flat_tiles_reuse_their_slots(fg):
    """A thousand single-unit deep tiles (200 reads of 56 bases: two would overflow a stage), several per CTA, so the
    flat form's double-buffered reduction slots are reused: each must be back to its identities before the next tile.
    About one dissenting A/C/G/T row per position at qualities above qt3 keeps most positions on the near-unanimous
    proof, whose error count a stale counter would change."""
    import torch
    rng = np.random.default_rng(12)
    U, D, L = 1000, 200, 56
    tmpl = rng.integers(0, 4, size=(U, 1, L), dtype=np.uint8)
    idx = np.broadcast_to(tmpl, (U, D, L)).copy()
    dis = rng.random((U, D, L)) < 1.0 / D
    idx[dis] = (idx[dis] + rng.integers(1, 4, size=int(dis.sum()), dtype=np.uint8)) & 3
    bases = ACGT[idx]
    quals = rng.integers(30, 41, size=(U, D, L), dtype=np.uint8)
    batch = fg.pack_uniform(bases, quals, 1)
    tiles = fg.plan_tiles(batch)
    assert len(tiles) == U and all((int(t["flags"]) >> 4) & 3 == 2 and t["n_units"] == 1 for t in tiles)
    ref = O.simplex_batch(batch, 45, 40, 1, 2, 8)
    eng = fg.Engine(0, 45, 40, 1, 2)
    try:
        db = fg.DeviceBatch(batch, "cuda:0")
        dc = fg.DeviceColumns(batch.n_out, "cuda:0")
        eng.vote_device(db, dc, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        out = dc.to_host()
        stats = eng.stats()
    finally:
        eng.close()
    assert (ref[3][:batch.n_out] > 0).mean() > 0.3          # the error counts are not all zero
    _compare(out, ref, batch, stats, "flat tiles")


# ---- duplex: the vote kernels' duplex epilogue and the standalone combine, at other settings than (45, 40) -------


def _duplex_against_oracle(fg, units, pairs, fused, pre, post, min_cons_q):
    """Vote `units` and combine `pairs` -- in the vote kernels' epilogue (`fused`) or with the standalone combine --
    at (pre, post, min_cons_q); every single-strand column and every job must equal the oracle's."""
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
    eng = fg.Engine(0, pre, post, 1, min_cons_q)
    try:
        db = fg.DeviceBatch(batch, dev)
        ss = fg.DeviceColumns(batch.n_out, dev)
        stream = torch.cuda.current_stream().cuda_stream
        if fused:
            tiles, class_tiles, tile_jobs, job_index, _ = fg.plan_tiles_jobs(batch, jobs)
            t8 = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)
            db.tiles, db.n_tiles, db.class_tiles = t8(tiles), len(tiles), class_tiles
            eng.vote_duplex_device(db, ss, tj, len(pairs), t8(tile_jobs), t8(job_index), o_base, o_qual, o_err,
                                   o_st, stream)
        else:
            eng.vote_device(db, ss, stream)
            eng.duplex_combine_device(db, ss, tj, len(pairs), o_base, o_qual, o_err, o_st, stream)
        torch.cuda.synchronize()
        st_ = eng.stats()
    finally:
        eng.close()
    ob, oq, od, oe, _ = O.simplex_batch(batch, pre, post, 1, min_cons_q, 8)
    g = ss.to_host()
    for sl in batch.unit_slices():
        assert np.array_equal(g.base[sl], ob[sl]) and np.array_equal(g.qual[sl], oq[sl]), sl
        assert np.array_equal(g.depth[sl], od[sl]) and np.array_equal(g.errors[sl], oe[sl]), sl
    assert st_["combined_jobs"] == len(pairs)
    assert st_["units"] == len(units)
    gb, gq = o_base.cpu().numpy(), o_qual.cpu().numpy()
    ge, gs = o_err.cpu().numpy().view(np.uint16), o_st.cpu().numpy()
    for j, (ua, ub) in enumerate(pairs):
        la, lb = int(cons_len[ua]), int(cons_len[ub])
        oa, obo = int(out_off[ua]), int(out_off[ub])
        rows = units[ua] + units[ub]
        keep = [np.frombuffer(r[0], np.uint8).copy() for r in rows]
        ptrs = (C.c_void_p * len(rows))(*[k.ctypes.data for k in keep])
        lens = (C.c_size_t * len(rows))(*[len(r[0]) for r in rows])
        cap = max(la, lb, 1)
        rb = np.zeros(cap, np.uint8)
        rq = np.zeros(cap, np.uint8)
        re_ = np.zeros(cap, np.uint16)
        olen = C.c_size_t()
        st = L.orc_duplex_job(ob[oa:].ctypes.data, oq[oa:].ctypes.data, od[oa:].ctypes.data,
                              oe[oa:].ctypes.data, la, ob[obo:].ctypes.data, oq[obo:].ctypes.data,
                              od[obo:].ctypes.data, oe[obo:].ctypes.data, lb, ptrs, lens, len(rows),
                              rb.ctypes.data, rq.ctypes.data, re_.ctypes.data, C.addressof(olen))
        assert gs[j] == st, (j, gs[j], st)
        o, n = int(jobs[j]["out_off"]), olen.value
        assert np.array_equal(gb[o:o + n], rb[:n]), j
        assert np.array_equal(gq[o:o + n], rq[:n]), j
        assert np.array_equal(ge[o:o + n], re_[:n]), j


@pytest.mark.parametrize("pre,post,mcq", [(45, 40, 2), (30, 20, "fq+1"), (85, 93, 2), (45, 1, 2)],
                         ids=lambda v: str(v))
def test_duplex_strands_from_the_depth_ladder(fg, pre, post, mcq):
    """Molecules whose two strands take depths from the ladder (shallow to oversize, nmax2 on either side), regular
    and ragged: the fused and the standalone duplex paths must both equal the oracle's duplex_consensus."""
    _, fast_qual, nmax2 = _tables(fg, pre, post)
    min_cons_q = _min_cons_q(mcq, fast_qual)
    ladder = _depth_ladder(nmax2)
    rng = np.random.default_rng(7000 + pre * 100 + post)
    units, pairs = [], []
    for i, da in enumerate(ladder):
        for shift in (0, 1, len(ladder) // 2):
            db = ladder[(i + shift) % len(ladder)]
            ragged = (i + shift) % 2 == 1
            cyc = _Cycle()
            for d in (da, db):
                L = int(rng.integers(16, 25))
                lens = [int(x) for x in rng.integers(16, 25, size=d)] if ragged else [L] * d
                units.append(_unit(rng, d, lens, cyc))
            pairs.append((len(units) - 2, len(units) - 1))
    for fused in (True, False):
        _duplex_against_oracle(fg, units, pairs, fused, pre, post, min_cons_q)
