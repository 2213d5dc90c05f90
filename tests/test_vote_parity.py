"""GPU parity: the sm_90a vote (through the C-ABI) against the CPU oracle on identical inputs.

Bar (BASELINE.json north_star): consensus bases, depths, errors and lengths bit-exact; consensus
qualities within +-1 phred (the tests additionally report how many differ at all — expected 0)."""
import numpy as np
import pytest

from tests import oracle_lib as O

pytestmark = pytest.mark.gpu

QUAL_TOL = 1   # phred units, stated by BASELINE.json


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as graft
    graft.build()
    import fgumi_b200
    return fgumi_b200


def check(fg, batch, pre=45, post=40, min_reads=1, min_cons_q=2, device_path=False, threads=4):
    eng = fg.Engine(0, pre, post, min_reads, min_cons_q)
    try:
        if device_path:
            import torch
            db = fg.DeviceBatch(batch, "cuda:0")
            dc = fg.DeviceColumns(batch.n_out, "cuda:0")
            eng.vote_device(db, dc, torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            out = dc.to_host()
        else:
            out = eng.vote(batch)
        stats = eng.stats()
    finally:
        eng.close()
    ob, oq, od, oe, cl = O.simplex_batch(batch, pre, post, min_reads, min_cons_q, threads)
    assert np.array_equal(cl, batch.units["cons_len"][: batch.n_units])
    n = batch.n_out
    # compare only real positions (rows are padded to 4)
    mask = np.zeros(max(n, 1), bool)
    for sl in batch.unit_slices():
        mask[sl] = True
    mask = mask[:n]
    gb, gq, gd, ge = out.base[:n][mask], out.qual[:n][mask], out.depth[:n][mask], out.errors[:n][mask]
    rb, rq, rd, re_ = ob[:n][mask], oq[:n][mask], od[:n][mask], oe[:n][mask]
    assert np.array_equal(gb, rb), f"{(gb != rb).sum()} consensus bases differ"
    assert np.array_equal(gd, rd), "depths differ"
    assert np.array_equal(ge, re_), "errors differ"
    dq = np.abs(gq.astype(int) - rq.astype(int))
    assert dq.max(initial=0) <= QUAL_TOL, f"max |dq| = {dq.max()}"
    assert (dq != 0).sum() == 0, f"{(dq != 0).sum()} qualities differ by 1 (within tolerance, but unexpected)"
    assert stats["positions"] == int(mask.sum())
    assert stats["units"] == batch.n_units
    return stats


def test_known_answer_vectors(fg):
    """The reference's own KATs (SURVEY §8c) pushed through the GPU path."""
    q = lambda v, n: bytes([v] * n)
    units = [
        [(b"GATTACA", q(10, 7))] * 2,                                   # vanilla_caller.rs:2083
        [(b"GATTACA", q(10, 7)), (b"GATTACA", q(10, 7)), (b"GATTTCA", q(10, 7))],  # :2117
        [(b"A" * 10, q(30, 10))] * 3 + [(b"AAAAACAAAA", q(30, 10))],    # :2396
        [(b"GATNACAG", q(20, 8)), (b"GATGACAG", q(20, 8)), (b"GATGACAG", q(20, 8)),
         (b"GATTACAG", q(20, 8))],                                      # :2473
        [(b"A" * 10, q(30, 10)), (b"A" * 8, q(30, 8)), (b"A" * 6, q(30, 6))],   # :2157
        [(b"A", q(37, 1))], [(b"AA", q(37, 2))] * 2, [(b"ACG", q(37, 3))] * 3,   # Appendix B
        [(b"C" * 5, q(20, 5))] * 300,                                   # deep pileup
        [(b"AC", bytes([20, 20])), (b"CA", bytes([20, 20]))],           # exact tie -> N
    ]
    for pre, post, mr, mq in ((45, 40, 1, 0), (93, 93, 1, 0), (50, 50, 1, 2), (45, 40, 2, 40)):
        usable = [u for u in units if len(u) >= mr]
        check(fg, fg.pack_source_reads(usable, mr), pre, post, mr, mq)


def test_config1_plumbing_depth3(fg):
    """BASELINE config 1: 1k molecules -> 2k units (R1, R2), depth 3, 150 bp, no errors."""
    from fgumi_b200 import synth
    b1, q1 = synth.host_pileup(1000, 3, 150, 0.0, seed=42)
    b2, q2 = synth.host_pileup(1000, 3, 150, 0.0, seed=43, r2=True)
    bases = np.stack([b1, b2], 1).reshape(2000, 3, 150)
    quals = np.stack([q1, q2], 1).reshape(2000, 3, 150)
    st = check(fg, fg.pack_uniform(bases, quals, 1))
    assert st["input_reads"] == 6000


@pytest.mark.parametrize("depth,err,seed", [(8, 1e-3, 1), (8, 0.05, 2), (4, 1e-2, 3), (2, 1e-2, 4),
                                           (1, 0.0, 5), (33, 0.02, 6), (100, 1e-3, 7)])
def test_uniform_depths(fg, depth, err, seed):
    from fgumi_b200 import synth
    n = 3000 if depth <= 8 else 300
    bases, quals = synth.host_pileup(n, depth, 150, err, seed=seed)
    st = check(fg, fg.pack_uniform(bases, quals, 1), device_path=(seed % 2 == 0))
    if depth == 8 and err == 1e-3:
        # the fast path must carry the clean data: < 3 % of positions may need the f64 path
        assert st["exact_positions"] < 0.03 * st["positions"]


def test_heavy_disagreement_and_ns(fg):
    from fgumi_b200 import synth
    bases, quals = synth.host_pileup(1500, 6, 150, 0.25, seed=11, n_rate=0.1)
    check(fg, fg.pack_uniform(bases, quals, 1))
    check(fg, fg.pack_uniform(bases, quals, 3), min_reads=3, min_cons_q=30)


def _ragged_units(rng, n_units, max_depth, lmin, lmax, alphabet=b"ACGTN", qlo=2, qhi=45):
    units = []
    for _ in range(n_units):
        d = int(rng.integers(1, max_depth + 1))
        tmpl = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=lmax)
        rows = []
        for _ in range(d):
            ln = int(rng.integers(lmin, lmax + 1))
            b = tmpl[:ln].copy()
            m = rng.random(ln) < 0.08
            b[m] = rng.choice(np.frombuffer(alphabet, np.uint8), size=int(m.sum()))
            qv = rng.integers(qlo, qhi + 1, size=ln).astype(np.uint8)
            rows.append((b.tobytes(), qv.tobytes()))
        units.append(rows)
    return units


def test_ragged_lengths_and_depths(fg):
    rng = np.random.default_rng(5)
    units = _ragged_units(rng, 800, 12, 1, 170)
    check(fg, fg.pack_source_reads(units, 1))
    units2 = [u for u in units if len(u) >= 2]
    check(fg, fg.pack_source_reads(units2, 2), min_reads=2, min_cons_q=10)


def test_odd_alphabet_and_qualities(fg):
    """lowercase bases, IUPAC codes, quality bytes above 93 and 0xFF."""
    rng = np.random.default_rng(6)
    units = _ragged_units(rng, 400, 9, 5, 60, alphabet=b"ACGTNacgtnRYKM.", qlo=0, qhi=255)
    check(fg, fg.pack_source_reads(units, 1), min_cons_q=0)


def test_order_sensitive_ties(fg):
    """SURVEY H1: two competing bases carrying the same multiset of qualities — the call depends
    on the f64 accumulation order, so the GPU must replay the reference's order exactly."""
    rng = np.random.default_rng(8)
    units = []
    for _ in range(3000):
        k = int(rng.integers(1, 6))
        qs = rng.integers(5, 45, size=k)
        obs = [(ord("A"), int(x)) for x in qs] + [(ord("C"), int(x)) for x in rng.permutation(qs)]
        order = rng.permutation(len(obs))
        rows = [(bytes([obs[i][0]]) * 3, bytes([obs[i][1]]) * 3) for i in order]
        units.append(rows)
    # (winner selection and the tie rule run on the exact f64 sums; the quality of a non-tied call
    #  comes from the certified tail or the f64 tail, whichever the position admits)
    check(fg, fg.pack_source_reads(units, 1), min_cons_q=0)


def test_zipf_depths(fg):
    from fgumi_b200 import synth
    rng = np.random.default_rng(9)
    depths = synth.zipf_depths(400, 1, 100, 1.0, seed=9)
    units = []
    for d in depths:
        b, q = synth.host_pileup(1, int(d), 150, 5e-3, seed=int(rng.integers(1 << 30)))
        units.append([(b[0, r].tobytes(), q[0, r].tobytes()) for r in range(int(d))])
    check(fg, fg.pack_source_reads(units, 1))


def test_deep_units_between_shallow_ones(fg):
    """Deep units (32-100 reads: tiles of a few dozen items, the whole-warp resolver) interleaved with
    shallow ones: regular and ragged, heavy dissent (long warp queues), Ns, low qualities, min_reads
    gates."""
    from fgumi_b200 import synth
    rng = np.random.default_rng(31)
    units = []
    for d, err in ((40, 1e-3), (3, 1e-2), (100, 5e-3), (33, 0.2), (1, 0.0), (64, 1e-3), (65, 0.05), (32, 0.0), (31, 0.01)):
        b, q = synth.host_pileup(1, d, 150, err, seed=int(rng.integers(1 << 30)))
        units.append([(b[0, r].tobytes(), q[0, r].tobytes()) for r in range(d)])
    batch = fg.pack_source_reads(units, 1)
    check(fg, batch)
    check(fg, batch, device_path=True)
    ragged = _ragged_units(rng, 60, 90, 1, 170)
    ragged = [u for u in ragged if len(u) >= 20]
    check(fg, fg.pack_source_reads(ragged, 1))
    check(fg, fg.pack_source_reads(ragged, 25), min_reads=25, min_cons_q=20)
    odd = _ragged_units(rng, 30, 80, 30, 60, alphabet=b"ACGTNacgtRY.", qlo=0, qhi=120)
    odd = [u for u in odd if len(u) >= 32]
    check(fg, fg.pack_source_reads(odd, 1))


def test_oversize_units_take_direct_path(fg):
    """Units too big for a shared-memory stage are voted straight from HBM."""
    from fgumi_b200 import synth
    cap = fg.lib.load().fgb_tile_capacity_bytes()
    d_big = cap // 152 + 40
    units = []
    for d, seed in ((3, 1), (d_big, 2), (5, 3), (600, 4), (2, 5)):
        b, q = synth.host_pileup(1, d, 150, 0.02, seed=seed)
        units.append([(b[0, r].tobytes(), q[0, r].tobytes()) for r in range(d)])
    batch = fg.pack_source_reads(units, 1)
    tiles = fg.plan_tiles(batch)
    assert (tiles["flags"] & 1).sum() == 2
    check(fg, batch)
    check(fg, batch, device_path=True)


def test_empty_and_tiny_batches(fg):
    eng = fg.Engine(0)
    out = eng.vote(fg.pack_source_reads([], 1))
    assert eng.stats()["units"] == 0
    eng.close()
    check(fg, fg.pack_source_reads([[(b"A", bytes([30]))]], 1))
    check(fg, fg.pack_source_reads([[(b"ACG", bytes([30] * 3))] * 2], 1))


def test_multi_chunk_submit(fg):
    """A host batch larger than one pipeline chunk (96 MiB per column) is split at tile boundaries."""
    from fgumi_b200 import synth
    bases, quals = synth.host_pileup(4000, 8, 150, 2e-3, seed=21)
    reps = 24   # 4000*24 units * 8 reads * 152 B = 116.7 MB per column
    bases = np.tile(bases, (reps, 1, 1))
    quals = np.tile(quals, (reps, 1, 1))
    st = check(fg, fg.pack_uniform(bases, quals, 1), threads=8)
    assert st["units"] == 4000 * reps


def test_pack8_submit_matches_byte_submit(fg):
    """PACK8 transfer format: same results as the two-column submit, half the H2D bytes."""
    rng = np.random.default_rng(88)
    units = []
    for _ in range(3000):
        depth = int(rng.integers(1, 12))
        L = int(rng.integers(5, 200))
        rows = []
        for _ in range(depth):
            ln = int(rng.integers(max(1, L - 20), L + 1))
            b = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=ln)
            q = rng.integers(0, 62, size=ln).astype(np.uint8)
            m = rng.random(ln) < 0.05
            b[m] = ord("N"); q[m] = 2
            rows.append((b.tobytes(), q.tobytes()))
        units.append(rows)
    batch = fg.pack_source_reads(units, 1)
    packed = fg.pack8_encode(batch.bases, batch.quals)
    assert packed is not None and packed.size == batch.bases.size
    eng = fg.Engine(0, 45, 40, 1, 2)
    want = eng.vote(batch)
    got = fg.HostColumns.alloc(batch.n_out)
    eng.submit_pack8(batch, packed, got)
    eng.wait()
    eng.close()
    for sl in batch.unit_slices():
        assert np.array_equal(got.base[sl], want.base[sl]) and np.array_equal(got.qual[sl], want.qual[sl])
        assert np.array_equal(got.depth[sl], want.depth[sl]) and np.array_equal(got.errors[sl], want.errors[sl])
    # and against the oracle directly
    ob, oq, od, oe, _ = O.simplex_batch(batch, 45, 40, 1, 2)
    for sl in batch.unit_slices():
        assert np.array_equal(got.base[sl], ob[sl]) and np.array_equal(got.qual[sl], oq[sl])


def test_bam4_submit_builds_source_reads_on_device(fg):
    """BAM4 transfer format (SURVEY §8f N1): the device decodes the 4-bit sequence, orients the read
    and applies the min-input-quality mask of create_source_read (vanilla_caller.rs:893-916); the
    result must equal a vote over rows prepared by the record oracle's create_source_read."""
    from oracle import record_oracle as R
    from tests.bam_builder import make_record
    rng = np.random.default_rng(99)
    alphabet = np.frombuffer(b"ACGTACGTACGTACGTNRYM=", np.uint8)
    opt = R.VanillaOptions(min_reads=1, min_input_base_quality=12, trim=False)
    raw_units, row_units = [], []
    for _ in range(2500):
        depth = int(rng.integers(1, 10))
        L = int(rng.integers(8, 180))
        ru, ou = [], []
        for _ in range(depth):
            ln = int(rng.integers(max(1, L - 15), L + 1))
            seq = alphabet[rng.integers(0, alphabet.size, size=ln)].tobytes()
            q = rng.integers(2, 45, size=ln).astype(np.uint8).tobytes()
            rev = bool(rng.integers(0, 2))
            clip = int(rng.integers(0, 6)) if rng.random() < 0.3 else 0
            rec = R.Rec(make_record(name=b"r", flags=R.REVERSE if rev else 0, pos=10, seq=seq, quals=q))
            sr = R.create_source_read(rec, 0, clip, opt)
            if sr is None:
                continue
            ru.append((seq, q, rev, len(sr.bases)))
            ou.append((bytes(sr.bases), bytes(sr.quals)))
        if ru:
            raw_units.append(ru); row_units.append(ou)
    layout, raw = fg.pack_raw_reads(raw_units, 1, opt.min_input_base_quality)
    eng = fg.Engine(0, 45, 40, 1, 2)
    got = fg.HostColumns.alloc(layout.n_out)
    eng.submit_bam4(layout, raw, got)
    eng.wait()
    want_batch = fg.pack_source_reads(row_units, 1)
    assert np.array_equal(want_batch.units["out_off"], layout.units["out_off"])
    ob, oq, od, oe, _ = O.simplex_batch(want_batch, 45, 40, 1, 2)
    for sl in want_batch.unit_slices():
        assert np.array_equal(got.base[sl], ob[sl]) and np.array_equal(got.qual[sl], oq[sl])
        assert np.array_equal(got.depth[sl], od[sl]) and np.array_equal(got.errors[sl], oe[sl])
    # CODEC-style rows: a clipped raw span, orientation only, no masking (codec_caller.rs:414-469)
    raw_units, row_units = [], []
    for _ in range(600):
        ru, ou = [], []
        for _ in range(int(rng.integers(1, 6))):
            ln = int(rng.integers(10, 120))
            seq = alphabet[rng.integers(0, 4, size=ln)].tobytes()
            q = rng.integers(2, 45, size=ln).astype(np.uint8).tobytes()
            rev = bool(rng.integers(0, 2))
            a = int(rng.integers(0, 4)) * 2                 # kept span starts on an even raw index
            b = ln - int(rng.integers(0, 5))
            ks, kq = seq[a:b], q[a:b]
            ru.append((ks, kq, rev, len(ks)))
            rows_b = bytes(R.reverse_complement(ks)) if rev else ks
            ou.append((rows_b, kq[::-1] if rev else kq))
        raw_units.append(ru); row_units.append(ou)
    layout, raw = fg.pack_raw_reads(raw_units, 1, 0)
    got = fg.HostColumns.alloc(layout.n_out)
    eng.submit_bam4(layout, raw, got)
    eng.wait()
    eng.close()
    want_batch = fg.pack_source_reads(row_units, 1)
    ob, oq, od, oe, _ = O.simplex_batch(want_batch, 45, 40, 1, 2)
    for sl in want_batch.unit_slices():
        assert np.array_equal(got.base[sl], ob[sl]) and np.array_equal(got.qual[sl], oq[sl])
        assert np.array_equal(got.depth[sl], od[sl]) and np.array_equal(got.errors[sl], oe[sl])


def test_submit_ex_narrow_outputs(fg):
    """fgb_submit_ex with FGB_OUT_U8: depth / errors arrive as u8 columns and equal the u16 ones; a
    unit deeper than 255 reads is refused."""
    rng = np.random.default_rng(123)
    units = []
    for _ in range(1500):
        depth = int(rng.integers(1, 30))
        L = int(rng.integers(10, 160))
        rows = []
        for _ in range(depth):
            b = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=L)
            q = rng.integers(2, 45, size=L).astype(np.uint8)
            rows.append((b.tobytes(), q.tobytes()))
        units.append(rows)
    batch = fg.pack_source_reads(units, 1)
    eng = fg.Engine(0, 45, 40, 1, 2)
    want = eng.vote(batch)
    n = batch.n_out
    for packed in (None, fg.pack8_encode(batch.bases, batch.quals)):
        got = fg.HostColumns(np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.full(n, 255, np.uint8),
                             np.full(n, 255, np.uint8))
        eng.submit_ex(batch, got, packed=packed, narrow=True)
        eng.wait()
        for sl in batch.unit_slices():
            assert np.array_equal(got.base[sl], want.base[sl]) and np.array_equal(got.qual[sl], want.qual[sl])
            assert np.array_equal(got.depth[sl], want.depth[sl]) and np.array_equal(got.errors[sl], want.errors[sl])
    deep = fg.pack_source_reads([[(b"ACGT", bytes([30] * 4))] * 256], 1)
    out = fg.HostColumns(np.zeros(8, np.uint8), np.zeros(8, np.uint8), np.zeros(8, np.uint8), np.zeros(8, np.uint8))
    with pytest.raises(fg.lib.FgbError):
        eng.submit_ex(deep, out, narrow=True)
    eng.close()


@pytest.mark.parametrize("pre,post", [(45, 40), (30, 20), (60, 50), (93, 93), (10, 45), (50, 10)])
def test_small_depth_dissent_stress(fg, pre, post):
    """Shallow pileups with dissent and the whole quality range leave the integer proofs and are
    decided by the certified single-precision tail or, near a rounding boundary, by the f64 tail.
    Qualities must still be identical to the oracle's, not merely within +-1."""
    rng = np.random.default_rng(1000 + pre * 100 + post)
    units = []
    for _ in range(20000):
        depth = int(rng.integers(2, 7))
        L = 64
        tmpl = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=L)
        rows = []
        for _ in range(depth):
            b = tmpl.copy()
            m = rng.random(L) < 0.25
            b[m] = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=int(m.sum()))
            q = rng.integers(1, 94, size=L).astype(np.uint8)
            rows.append((b.tobytes(), q.tobytes()))
        units.append(rows)
    batch = fg.pack_source_reads(units, 1)
    eng = fg.Engine(0, pre, post, 1, 2)
    got = eng.vote(batch)
    st = eng.stats()
    eng.close()
    ob, oq, od, oe, _ = O.simplex_batch(batch, pre, post, 1, 2, 8)
    n = batch.n_out
    assert np.array_equal(got.base[:n], ob[:n])
    assert np.array_equal(got.qual[:n], oq[:n])
    assert np.array_equal(got.depth[:n], od[:n]) and np.array_equal(got.errors[:n], oe[:n])
    # the certified tail decides almost everything the proofs leave open
    assert st["exact_positions"] < 0.05 * st["positions"]


def test_bam4_bad_raw_span_is_reported_at_wait(fg):
    """A raw span that runs past the columns is caught by the unpack kernel (the read is skipped) and
    surfaces as FGB_ERR_LAYOUT from the next fgb_wait; the handle stays usable."""
    units = [[(b"ACGTACGTAC", bytes([30] * 10), False, 10)] * 3 for _ in range(50)]
    layout, raw = fg.pack_raw_reads(units, 1, 10)
    eng = fg.Engine(0, 45, 40, 1, 2)
    out = fg.HostColumns.alloc(layout.n_out)
    raw.raw_reads["raw_len"][7] = 4          # shorter than its 10-base row
    eng.submit_bam4(layout, raw, out)
    with pytest.raises(fg.lib.FgbError) as ei:
        eng.wait()
    assert ei.value.status == fg.lib.FGB_ERR_LAYOUT
    raw.raw_reads["raw_len"][7] = 10
    eng.submit_bam4(layout, raw, out)
    eng.wait()
    assert bytes(out.base[:10]) == b"ACGTACGTAC"
    eng.close()
