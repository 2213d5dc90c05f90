"""fgb_sort_records at the sizes users sort.  The inputs reach what only large inputs reach -- both page-locked staging
buffers reused in both directions with a partial last chunk, the staging copies split unevenly over several threads,
an offsets upload of two chunks, runs that each span several chunks merged on the host -- and the record gather at
every alignment, on records of 64 KiB and more and on CIGARs and MC strings of 65 535 operations.

Every record carries a serial in bytes no key reads (tests/sort_cases.py), so a wrong permutation, a lost record or an
unstable tie changes the output bytes.  The references: numpy for the coordinate key, a stable np.lexsort of the
host key words (fgb_host_sort_keys, checked against oracle/sort_oracle.py on a sample of each input) for
template-coordinate, and oracle/sort_oracle.py itself for the mid-size inputs.  The CPU checks of the generators and
references are in tests/test_sort_keys.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sort_oracle as S      # noqa: E402
from tests import sort_cases as SC       # noqa: E402
from tests.sort_cases import HEADER      # noqa: E402

pytestmark = pytest.mark.gpu
TC, CO = "template-coordinate", "coordinate"
CASES = [(TC, b"CB"), (TC, None), (CO, None)]

SEED = 31
BULK_BYTES = 232 << 20        # bulk input: 4 staging chunks each way, and room for 3 runs of more than 64 MiB
BULK_LEAD, BULK_SKEW = 4093, 1  # its rec_off[0], and its bodies array 1 byte into an aligned allocation
RUNS = 3                      # runs of the multi-run case, each more than one staging buffer of records
FAMILY_WINDOW = 200           # records on either side of each run boundary that share one key
MIN_RECORDS = 9_000_000       # minimal records: (n + 1) x 8 bytes of offsets span two staging chunks
THREADS = (1, 3, 16)          # staging copies on 1 thread, 3 uneven pieces, 16 pieces
SAMPLE = 2000                 # records of each large input whose host keys are checked against the oracle
GRID_RUN_BYTES = 600_000      # device_bytes of the gather-edge input sorted in several runs
SMALL_RUN_BYTES = 150_000     # device_bytes of the offset-base input sorted in several runs


@pytest.fixture(scope="module")
def mods():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, sort
    return sort, bamio


def _words(order):
    return 1 if order == CO else 5


def _sorted_ok(mods, out, n, nbytes, order, cell):
    """The output's length and `fgumi sort --verify` on it."""
    sort, bamio = mods
    assert len(out) == nbytes + 4 * n
    ob, ooff = bamio.split_stream(out)
    assert len(ooff) == n + 1
    assert sort.verify(HEADER, ob, ooff, order, cell) == (0, None)


def _keys_match_oracle(sort, bodies, off, which, order, cell):
    """The host keys (the key kernel's code) equal the oracle's on the records `which`."""
    recs = SC.records_of(bodies, off, which)
    b, o = SC.pack(recs)
    got = [tuple(int(x) for x in row) for row in sort.sort_keys(HEADER, b, o, order, cell)]
    assert got == S.keys(recs, HEADER, order, cell)
    if order == CO:
        assert [k[0] for k in got] == SC.coordinate_keys(b, o).tolist()


def _sample(n, seed, extra=()):
    rng = np.random.default_rng(seed)
    return sorted(set(rng.choice(n, SAMPLE, replace=False).tolist()) | set(int(i) for i in extra))


# ---- the bulk input: one run, and several runs of more than one staging buffer --------------------------------------
@pytest.fixture(scope="module")
def bulk():
    """About BULK_BYTES of records tiled from SC.bulk_pool, with one family of equal keys (one pool record, the same
    fixed fields) planted across every run boundary of the multi-run case in both orders."""
    common, rare = SC.bulk_pool(SEED)
    pool = common + rare
    lens = np.array([len(r) for r in pool], np.int64)
    n = int(BULK_BYTES / lens[:len(common)].mean())
    f = SC.bulk_fields(n, SEED, len(common), len(rare))
    fam = int(np.argmin(np.abs(lens[:len(common)] - lens[f["idx"]].mean())))   # about the mean size: boundaries stay

    def budgets(off):   # the first run holds 1.03 / RUNS of the bytes, so the last one holds about 0.94 / RUNS
        off = np.asarray(off, np.int64)
        end = int(np.searchsorted(off, off[0] + (off[-1] - off[0]) * 103 // (100 * RUNS)))
        return {w: SC.budget_for(off, end, w) for w in (1, 5)}

    off0 = np.zeros(n + 1, np.int64)
    off0[1:] = np.cumsum(lens[f["idx"]])
    members = np.zeros(n, bool)
    for w, budget in budgets(off0).items():
        for bd in SC.run_plan(off0, budget, w)[1:-1]:
            members[bd - FAMILY_WINDOW:bd + FAMILY_WINDOW] = True
    f["idx"][members] = fam
    for k, v in (("tid", 1), ("pos", 5), ("strand", 0x10), ("mtid", 1), ("mpos", 9)):
        f[k][members] = v
    bodies, off = SC.materialize(pool, f, BULK_LEAD, BULK_SKEW)
    return dict(bodies=bodies, off=off, family=np.flatnonzero(members), budget=budgets(off),
                rare=np.flatnonzero(f["idx"] >= len(common)), perm={})


def _bulk_perm(mods, bulk, order, cell):
    """The reference order of the bulk input, once per (order, cell), after its keys are checked on a sample."""
    if (order, cell) not in bulk["perm"]:
        bodies, off = bulk["bodies"], bulk["off"]
        n = len(off) - 1
        _keys_match_oracle(mods[0], bodies, off, _sample(n, 1, bulk["rare"]), order, cell)
        keys = SC.coordinate_keys(bodies, off) if order == CO else mods[0].sort_keys(HEADER, bodies, off, order, cell)
        bulk["perm"][(order, cell)] = SC.sorted_order(keys)
    return bulk["perm"][(order, cell)]


def _split(total, threads):
    """par_copy's pieces of a staging chunk of `total` bytes on `threads` threads."""
    return min(threads, max(total >> 22, 1))


@pytest.mark.parametrize("order,cell", CASES)
def test_one_run_at_scale(mods, bulk, order, cell):
    sort = mods[0]
    bodies, off = bulk["bodies"], bulk["off"]
    n, nbytes = len(off) - 1, int(off[-1] - off[0])
    assert bodies.ctypes.data % 4 and off[0] % 4
    assert nbytes >= 160 << 20
    for total in (nbytes, nbytes + 4 * n):        # upload of the records, download of the stream
        chunks = -(-total // SC.STAGE_BYTES)
        last = total - (chunks - 1) * SC.STAGE_BYTES
        assert chunks >= 3, "both staging buffers are reused"
        assert all(last % _split(last, t) for t in THREADS[1:]), "the last chunk splits unevenly"
    assert SC.STAGE_BYTES % _split(SC.STAGE_BYTES, 3)
    perm = _bulk_perm(mods, bulk, order, cell)
    assert len(SC.alignments(off, perm)) == 64
    first = None
    for t in THREADS:
        s = sort.RecordSorter(0, order, cell, device_bytes=0, n_threads=t)
        out = s.sort(HEADER, bodies, off)
        assert s.last_timing()["merge_ms"] == 0
        s.close()
        if first is None:
            SC.assert_stream(out, bodies, off, perm)
            first = out
        elif out != first:
            SC.assert_stream(out, bodies, off, perm)   # names the first wrong record
            pytest.fail(f"n_threads={t} changed the output")
        del out
    _sorted_ok(mods, first, n, nbytes, order, cell)


@pytest.mark.parametrize("order,cell", [(TC, b"CB"), (CO, None)])
def test_runs_larger_than_a_staging_buffer(mods, bulk, order, cell):
    sort = mods[0]
    bodies, off = bulk["bodies"], bulk["off"]
    n, nbytes = len(off) - 1, int(off[-1] - off[0])
    budget = bulk["budget"][_words(order)]
    plan = SC.run_plan(off, budget, _words(order))
    assert len(plan) - 1 >= RUNS
    assert all(int(off[b] - off[a]) > SC.STAGE_BYTES for a, b in zip(plan, plan[1:]))
    fam = bulk["family"]
    for bd in plan[1:-1]:                          # equal keys, different serials, on both sides of every boundary
        assert np.any((fam >= bd - FAMILY_WINDOW) & (fam < bd)) and np.any((fam >= bd) & (fam < bd + FAMILY_WINDOW))
    perm = _bulk_perm(mods, bulk, order, cell)
    s = sort.RecordSorter(0, order, cell, device_bytes=budget, n_threads=16)
    out = s.sort(HEADER, bodies, off)
    assert s.last_timing()["merge_ms"] > 0
    s.close()
    SC.assert_stream(out, bodies, off, perm)
    one = sort.RecordSorter(0, order, cell, n_threads=16).sort(HEADER, bodies, off)
    if out != one:                                  # (no assertion rewriting on two streams of 240 MB)
        SC.assert_stream(one, bodies, off, perm)
        pytest.fail("the one-run output differs from the multi-run output")
    del one
    _sorted_ok(mods, out, n, nbytes, order, cell)


# ---- more than 8 388 607 minimal records: the offsets upload spans two staging chunks ------------------------------
def test_offsets_span_two_staging_chunks(mods):
    sort = mods[0]
    f = SC.bulk_fields(MIN_RECORDS, SEED + 1, 1, 0)
    bodies, off = SC.materialize([SC.minimal_record()], f)
    del f
    n = MIN_RECORDS
    assert (n + 1) * 8 > SC.STAGE_BYTES
    keys = SC.coordinate_keys(bodies, off)
    assert len(np.unique(keys)) * 1000 < n          # heavy ties, every record byte-unique by its serial
    _keys_match_oracle(sort, bodies, off, _sample(n, 2), CO, None)
    perm = SC.sorted_order(keys)
    del keys
    s = sort.RecordSorter(0, CO, None, n_threads=16)
    out = s.sort(HEADER, bodies, off)
    assert s.last_timing()["merge_ms"] == 0
    s.close()
    SC.assert_stream(out, bodies, off, perm)
    _sorted_ok(mods, out, n, int(off[-1]), CO, None)


# ---- the record gather's edges, against the oracle ----------------------------------------------------------------
@pytest.fixture(scope="module")
def grid():
    recs = SC.gather_grid(SEED)
    return recs, SC.pack(recs), {}


@pytest.mark.parametrize("device_bytes", [0, GRID_RUN_BYTES])
@pytest.mark.parametrize("order,cell", CASES)
def test_gather_edges(mods, grid, order, cell, device_bytes):
    sort = mods[0]
    recs, (b, off), want = grid
    if (order, cell) not in want:
        want[(order, cell)] = S.sorted_stream(recs, HEADER, order, cell)
    s = sort.RecordSorter(0, order, cell, device_bytes=device_bytes, n_threads=4)
    out = s.sort(HEADER, b, off)
    assert (s.last_timing()["merge_ms"] > 0) == (device_bytes > 0)
    s.close()
    if out != want[(order, cell)]:
        k = S.keys(recs, HEADER, order, cell)
        SC.assert_stream(out, b, off, np.array(sorted(range(len(recs)), key=k.__getitem__)))
        pytest.fail("output differs from the oracle")
    _sorted_ok(mods, out, len(recs), int(off[-1]), order, cell)


# ---- rec_off[0] != 0 and a bodies pointer that is not 4-aligned, against the oracle ---------------------------------
@pytest.mark.parametrize("device_bytes", [0, SMALL_RUN_BYTES])
@pytest.mark.parametrize("order,cell", [(TC, b"CB"), (CO, None)])
def test_offset_base_and_unaligned_bodies(mods, order, cell, device_bytes):
    sort = mods[0]
    recs = SC.stamp_serials(SC.random_records(5000, seed=SEED + 2))
    b, off = SC.pack_at(recs, 4093, 1)
    assert b.ctypes.data % 4 and off[0] == 4093
    if device_bytes:
        assert len(SC.run_plan(off, device_bytes, _words(order))) - 1 >= 3
    s = sort.RecordSorter(0, order, cell, device_bytes=device_bytes, n_threads=3)
    out = s.sort(HEADER, b, off)
    assert (s.last_timing()["merge_ms"] > 0) == (device_bytes > 0)
    s.close()
    assert out == S.sorted_stream(recs, HEADER, order, cell)
    _sorted_ok(mods, out, len(recs), int(off[-1] - off[0]), order, cell)
