"""GPU parity of the general vote kernel's early stage release: undecided positions of units with at most 24 reads are
copied into per-warp pileup slots, the stage is released, and the slots are resolved afterwards.  Every case runs
through `vote_kernel` and is compared with the CPU oracle bit for bit (bases, qualities, depths, errors) together with
the position and no-call counters.  The cases reach the slot path and each fallback: full slots, an overflowing warp
queue, units deeper than a slot, shallow-class units and an oversize (direct) unit in an unsorted batch, the literal
f64 path from a slot, and ragged reads whose uncovered rows are left out of the gathered pileup."""
import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_vote_parity import _ragged_units

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fg():
    import __graft_entry__ as graft
    graft.build()
    import fgumi_b200
    return fgumi_b200


def check(fg, batch, pre=45, post=40, min_reads=1, min_cons_q=2, unsorted=False):
    """Device-resident vote of `batch`; with `unsorted` every tile goes to the general kernel (class_tiles = 0)."""
    import torch
    eng = fg.Engine(0, pre, post, min_reads, min_cons_q)
    try:
        db = fg.DeviceBatch(batch, "cuda:0")
        if unsorted:
            db.class_tiles = (0, 0, 0)
        dc = fg.DeviceColumns(batch.n_out, "cuda:0")
        eng.vote_device(db, dc, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        out = dc.to_host()
        stats = eng.stats()
    finally:
        eng.close()
    ob, oq, od, oe, _ = O.simplex_batch(batch, pre, post, min_reads, min_cons_q, 8)
    n = batch.n_out
    mask = np.zeros(max(n, 1), bool)
    for sl in batch.unit_slices():
        mask[sl] = True
    mask = mask[:n]
    assert np.array_equal(out.base[:n][mask], ob[:n][mask]), "consensus bases differ"
    assert np.array_equal(out.qual[:n][mask], oq[:n][mask]), "consensus qualities differ"
    assert np.array_equal(out.depth[:n][mask], od[:n][mask]), "depths differ"
    assert np.array_equal(out.errors[:n][mask], oe[:n][mask]), "errors differ"
    assert stats["positions"] == int(mask.sum())
    assert stats["nocall_positions"] == int((ob[:n][mask] == ord("N")).sum())
    assert stats["units"] == batch.n_units
    return stats


def _noisy_units(rng, n_units, depths, L, err, qlo, qhi):
    units = []
    for _ in range(n_units):
        d = int(rng.integers(depths[0], depths[1] + 1))
        tmpl = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=L)
        rows = []
        for _ in range(d):
            b = tmpl.copy()
            m = rng.random(L) < err
            b[m] = rng.choice(np.frombuffer(b"ACGTN", np.uint8), size=int(m.sum()))
            q = rng.integers(qlo, qhi + 1, size=L).astype(np.uint8)
            rows.append((b.tobytes(), q.tobytes()))
        units.append(rows)
    return units


@pytest.mark.parametrize("err,seed", [(0.02, 1), (0.3, 2)])
def test_general_depths_fill_and_overflow_slots(fg, err, seed):
    """Depth 5-23 at low qualities: at 2 % dissent a warp's queue fills and passes its 16 slots, at 30 % it also
    passes the 96-entry queue (positions resolved in place during the fast pass)."""
    rng = np.random.default_rng(seed)
    units = _noisy_units(rng, 3000, (5, 23), 150, err, 2, 30)
    st = check(fg, fg.pack_source_reads(units, 1))
    check(fg, fg.pack_source_reads(units, 6), min_reads=6, min_cons_q=20)
    assert st["exact_positions"] > 0


def test_unsorted_batch_mixes_depths_in_general_kernel(fg):
    """class_tiles = (0, 0, 0): shallow (1-4 reads), general and deep (25-40 reads, too deep for a slot) tiles and one
    oversize unit voted from HBM, all through the general kernel."""
    from fgumi_b200 import synth
    rng = np.random.default_rng(3)
    units = []
    for lo, hi in ((1, 4), (5, 23), (25, 40), (1, 4), (24, 24)):
        units += _noisy_units(rng, 400 if hi <= 23 else 60, (lo, hi), 150, 0.05, 2, 40)
    cap = fg.lib.load().fgb_tile_capacity_bytes()
    b, q = synth.host_pileup(1, cap // 152 + 40, 150, 0.02, seed=4)
    units.insert(500, [(b[0, r].tobytes(), q[0, r].tobytes()) for r in range(b.shape[1])])
    batch = fg.pack_source_reads(units, 1)
    assert (fg.plan_tiles(batch)["flags"] & 1).sum() == 1
    check(fg, batch, unsorted=True)
    check(fg, fg.pack_source_reads(units, 3), min_reads=3, min_cons_q=25, unsorted=True)


def test_order_sensitive_ties_from_slots(fg):
    """Two bases with the same multiset of qualities in 6-22 reads: whether the f64 sums tie depends on the order they
    are added in, so the f64 path must see the slot's observations in read order."""
    rng = np.random.default_rng(8)
    units = []
    for _ in range(3000):
        k = int(rng.integers(3, 12))
        qs = rng.integers(5, 45, size=k)
        obs = [(ord("A"), int(x)) for x in qs] + [(ord("C"), int(x)) for x in rng.permutation(qs)]
        order = rng.permutation(len(obs))
        units.append([(bytes([obs[i][0]]) * 20, bytes([obs[i][1]]) * 20) for i in order])
    check(fg, fg.pack_source_reads(units, 1), min_cons_q=0)


@pytest.mark.parametrize("pre,post", [(45, 40), (93, 93), (10, 45), (50, 10)])
def test_general_depth_dissent_near_boundaries(fg, pre, post):
    """Dissent over the whole quality range at depth 5-8: integer proofs fail and the f64 tail decides near rounding
    boundaries, from the slots."""
    rng = np.random.default_rng(2000 + pre * 100 + post)
    units = _noisy_units(rng, 4000, (5, 8), 64, 0.25, 1, 93)
    check(fg, fg.pack_source_reads(units, 1))


def test_ragged_reads_leave_the_gathered_pileup(fg):
    """Reads of different lengths: a read that ends before a position is not one of its observations."""
    rng = np.random.default_rng(5)
    units = [u for u in _ragged_units(rng, 2500, 23, 1, 170) if len(u) >= 5]
    check(fg, fg.pack_source_reads(units, 1))
    check(fg, fg.pack_source_reads(units, 4), min_reads=4, min_cons_q=10)
