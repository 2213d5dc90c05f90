"""The sort keys, library lookup, output header and `--verify` of `fgumi sort` without a GPU: cases restated from the
reference's tests (sort/keys.rs, sort/inline_buffer.rs, sort/raw.rs, sort/mod.rs, fgumi-raw-bam tags.rs and cigar.rs)
against oracle/sort_oracle.py and fgb_host_sort_keys (the code the key kernel runs), and the two word for word on
random records of every kind."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sort_oracle as S       # noqa: E402
from tests import sort_cases as SC        # noqa: E402
from tests.bam_builder import make_record  # noqa: E402
from tests.sort_cases import HEADER, pack, random_records  # noqa: E402

M64 = (1 << 64) - 1
TC, CO = "template-coordinate", "coordinate"


@pytest.fixture(scope="module")
def srt():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import sort
    return sort


def both(srt, recs, order=TC, cell=b"CB", header=HEADER):
    """The keys of `recs` from the product and the oracle, which must agree word for word."""
    b, off = pack(recs)
    got = [tuple(int(x) for x in row) for row in srt.sort_keys(header, b, off, order, cell, n_threads=3)]
    want = S.keys(recs, header, order, cell)
    assert got == want
    return got


def rec(name=b"r", flags=0, tid=0, pos=100, cigar="10M", mtid=-1, mpos=-1, tags=()):
    return make_record(name=name, flags=flags, ref_id=tid, pos=pos, cigar=cigar, mate_ref_id=mtid, mate_pos=mpos,
                       seq=b"A" * 10, tags=tags)


# ---- coordinate (keys.rs / inline_buffer.rs PackedCoordinateKey) ------------------------------------------------
def test_coordinate_key_packing(srt):
    k = both(srt, [rec(tid=0, pos=0), rec(tid=0, pos=0, flags=0x10), rec(tid=1, pos=100), rec(tid=-1, pos=5),
                   rec(tid=2, pos=7, flags=0x4), rec(tid=0, pos=-1)], CO)
    assert [x[0] for x in k] == [2, 3, (1 << 34) | (101 << 1), M64, (2 << 34) | (8 << 1), 0]
    assert all(x[1:] == (0, 0, 0, 0) for x in k)


def test_coordinate_order_tid_pos_strand(srt):
    recs = [rec(tid=1, pos=5), rec(tid=0, pos=9, flags=0x10), rec(tid=0, pos=9), rec(tid=-1), rec(tid=0, pos=2)]
    k = [x[0] for x in both(srt, recs, CO)]
    assert sorted(range(5), key=lambda i: k[i]) == [4, 2, 1, 0, 3]


# ---- TemplateKey packing and order (inline_buffer.rs) -----------------------------------------------------------
def test_template_key_new_packing():
    k = S.template_key_new(1, 100, False, 2, 200, True, 9, 3, (5, False), 7, True)
    assert k == ((1 << 48) | (2 << 32) | (100 ^ 0x80000000), ((200 ^ 0x80000000) << 32) | (1 << 1) | 0, 9,
                 (3 << 48) | (5 << 1) | 1, (7 << 1) | 1)
    m = S.template_key_new(2 ** 31 - 1, -1, True, 70000, 2 ** 31 - 1, False, 0, 0x1FFFF, (2 ** 50 + 3, True), M64, False)
    assert m[0] == (0xFFFF << 48) | ((70000 & 0xFFFF) << 32) | 0x7FFFFFFF
    assert m[1] == (0xFFFFFFFF << 32) | (0 << 1) | 1
    assert m[3] == (0xFFFF << 48) | ((3 & 0xFFFFFFFFFFFF) << 1)
    assert m[4] == (M64 << 1) & M64
    assert S.template_key_unmapped(5, 6, True) == (M64, M64, 6, 0, 11)


def test_template_key_from_records(srt):
    libs_hdr = HEADER
    mate = rec(name=b"p", flags=0x1 | 0x20 | 0x40, tid=0, pos=100, cigar="3S10M", mtid=0, mpos=300,
               tags=[(b"MC", "Z", b"10M2S"), (b"RG", "Z", b"A"), (b"MI", "Z", b"12/B")])
    k = both(srt, [mate], TC, None, libs_hdr)[0]
    # own 5' = 100 - 3 = 97 forward; mate reverse 5' = 300 + 10 + 2 - 1 = 311; lower first
    assert k == S.template_key_new(0, 97, False, 0, 311, True, 0, 2, (12, False), S.fnv1a64(b"p"), False)


def test_template_order(srt):
    def key(**kw):
        return both(srt, [rec(**kw)], TC)[0]
    assert key(tid=0, pos=5) < key(tid=1, pos=0)
    assert key(tid=0, pos=5, flags=0x10, cigar="1M") < key(tid=0, pos=5)      # reverse before forward
    a = key(tags=[(b"MI", "Z", b"3/A")])
    b = key(tags=[(b"MI", "Z", b"3/B")])
    assert a < b and a[:3] == b[:3]
    lo = key(name=b"x", flags=0x1, tid=0, pos=5, mtid=0, mpos=50, tags=[(b"MC", "Z", b"10M")])
    hi = key(name=b"x", flags=0x1, tid=0, pos=50, mtid=0, mpos=5, tags=[(b"MC", "Z", b"10M")])
    assert lo[:4] == hi[:4] and lo[4] == hi[4] - 1                          # is_upper false before true


def test_core_cmp_ignores_name_hash(srt):
    a, b = rec(name=b"aaa"), rec(name=b"zzz")
    for recs in ([a, b], [b, a]):
        bb, off = pack(recs)
        assert srt.verify(HEADER, bb, off) == (0, None) == S.verify(recs, HEADER, TC)
    bb, off = pack([rec(pos=9), rec(pos=3), rec(pos=4), rec(pos=1)])
    assert srt.verify(HEADER, bb, off) == (2, 1)
    assert srt.verify(HEADER, bb, off, CO) == (2, 1)


# ---- LibraryLookup (raw.rs) -------------------------------------------------------------------------------------
def test_library_lookup(srt):
    assert S.library_lookup(HEADER) == {b"A": 2, b"B": 1, b"C": 0, b"D": 3, b"E": 1}
    for rg, want in ((b"A", 2), (b"B", 1), (b"C", 0), (b"D", 3), (b"E", 1), (b"nope", 0), (None, 0)):
        tags = [(b"RG", "Z", rg)] if rg is not None else []
        k = both(srt, [rec(tags=tags)])[0]
        assert k[3] >> 48 == want, rg


def test_cell_hash(srt):
    with_cb = rec(tags=[(b"CB", "Z", b"ACGT")])
    k = both(srt, [with_cb, with_cb, rec(tags=[(b"CB", "Z", b"TTTT")]), rec()])
    assert k[0][2] != 0 and k[0][2] == k[1][2] != k[2][2] and k[3][2] == 0
    assert both(srt, [with_cb], TC, None)[0][2] == 0                        # no cell tag: 0
    assert both(srt, [with_cb], TC, b"XB")[0][2] == 0                       # another tag: absent
    assert both(srt, [rec(tags=[(b"XB", "Z", b"ACGT")])], TC, b"XB")[0][2] == S.fnv1a64(b"ACGT")


def test_unmapped_with_mapped_mate_and_both_unmapped(srt):
    u = rec(name=b"m", flags=0x1 | 0x4 | 0x80, tid=0, pos=500, cigar=[], mtid=0, mpos=500,
            tags=[(b"MC", "Z", b"5S20M")])
    k = both(srt, [u])[0]
    assert k == S.template_key_new(0, 495, False, 2 ** 31 - 1, 2 ** 31 - 1, False, 0, 0, (0, True),
                                   S.fnv1a64(b"m"), True)
    uu = rec(name=b"m", flags=0x1 | 0x4 | 0x8 | 0x80, tid=-1, pos=-1, cigar=[], tags=[(b"CB", "Z", b"AC")])
    assert both(srt, [uu])[0] == (M64, M64, S.fnv1a64(b"AC"), 0, ((S.fnv1a64(b"m") << 1) & M64) | 1)


# ---- parse_mi_bytes / extract_template_aux_tags (tags.rs) -------------------------------------------------------
@pytest.mark.parametrize("value,want", [(b"123", (123, True)), (b"123/A", (123, True)), (b"123/B", (123, False)),
                                        (b"abc", (0, True)), (b"", (0, True)), (b"/A", (0, True)),
                                        (b"7/C", (7, True)), (b"1x/B", (0, True)),
                                        (b"99999999999999999999999/B", (M64, False))])
def test_parse_mi_z(srt, value, want):
    k = both(srt, [rec(tags=[(b"MI", "Z", value)])])[0]
    assert k[3] == ((want[0] & 0xFFFFFFFFFFFF) << 1) | (not want[1])


@pytest.mark.parametrize("typ,v,want", [("c", -3, 0), ("C", 200, 200), ("s", -1, 0), ("S", 60000, 60000),
                                        ("i", -7, 0), ("i", 123456, 123456), ("I", 4000000000, 4000000000)])
def test_mi_integer_types(srt, typ, v, want):
    k = both(srt, [rec(tags=[(b"MI", typ, v)])])[0]
    assert k[3] == want << 1


def test_aux_scan_rules(srt):
    # a later RG replaces an earlier one while tags are still wanted; the scan ends once all of them are seen
    k = both(srt, [rec(tags=[(b"RG", "Z", b"A"), (b"RG", "Z", b"B")])])[0]
    assert k[3] >> 48 == 1
    k = both(srt, [rec(tags=[(b"MI", "Z", b"1"), (b"RG", "Z", b"A"), (b"MC", "Z", b"1M"), (b"RG", "Z", b"B")])], TC,
             None)[0]
    assert k[3] >> 48 == 2
    # a non-UTF-8 MC counts as absent: the mate position falls back to mate_pos
    m = [(b"MC", "Z", b"\xff5S10M")]
    k = both(srt, [rec(name=b"a", flags=0x1, tid=0, pos=900, mtid=0, mpos=200, tags=m)])[0]
    assert k[0] & 0xFFFFFFFF == 200 ^ 0x80000000
    # an unknown type ends the scan before a later RG
    r = rec(tags=[(b"XX", "i", 1)]) + b"QQ?xyz" + b"RGZA\0"
    assert both(srt, [r])[0][3] >> 48 == 0


# ---- unclipped_5prime_raw / mate_unclipped_5prime (cigar.rs) ----------------------------------------------------
@pytest.mark.parametrize("flags,cigar,want", [(0, "5S10M", 95), (0, "2H3S10M", 95), (0x10, "10M5S", 114),
                                              (0x10, "3S10M2D4M2S1H", 100 + 16 + 3 - 1), (0, "10M", 100),
                                              (0x10, "5S", 99), (0, [], 100)])
def test_unclipped_5prime(srt, flags, cigar, want):
    k = both(srt, [rec(flags=flags, cigar=cigar)])[0]
    assert k[0] & 0xFFFFFFFF == (want & 0xFFFFFFFF) ^ 0x80000000


@pytest.mark.parametrize("mrev,mc,want", [(False, b"5S10M", 995), (False, b"3H2S10M", 995), (True, b"10M5S", 1014),
                                          (True, b"5S10M2D3N1=1X4S2H", 1000 + 17 + 6 - 1), (False, b"10M", 1000),
                                          (True, b"", 999), (False, b"99999999999S", 1000)])
def test_mate_unclipped_5prime(srt, mrev, mc, want):
    r = rec(name=b"q", flags=0x1 | (0x20 if mrev else 0), tid=0, pos=5000, mtid=0, mpos=1000, tags=[(b"MC", "Z", mc)])
    k = both(srt, [r])[0]
    assert k[0] & 0xFFFFFFFF == (want & 0xFFFFFFFF) ^ 0x80000000


def test_name_and_cigar_past_the_record(srt):
    r = bytearray(rec(name=b"abc", flags=0x10, cigar="5M5S"))
    r[8] = 200                                     # the name runs past the record: hashes as empty
    struct.pack_into("<H", r, 12, 50000)           # the CIGAR runs past it: pos unchanged
    k = both(srt, [bytes(r)])[0]
    assert k[4] == (S.fnv1a64(b"") << 1) & M64 and k[0] & 0xFFFFFFFF == 100 ^ 0x80000000


def test_short_record_is_a_layout_error(srt):
    from fgumi_b200 import lib as L
    recs = [rec(), rec(), rec()[:31], rec()]
    b, off = pack(recs)
    lib = L.load()
    o = srt.options(TC)
    keys = np.zeros((4, 5), np.uint64)
    bad = C.c_uint64()
    st = lib.fgb_host_sort_keys(C.byref(o), HEADER, len(HEADER), b.ctypes.data, off.ctypes.data, 4, keys.ctypes.data,
                                C.byref(bad))
    assert st == L.FGB_ERR_LAYOUT and bad.value == 2
    v, f = C.c_uint64(), C.c_uint64()
    st = lib.fgb_host_sort_verify(C.byref(o), HEADER, len(HEADER), b.ctypes.data, off.ctypes.data, 4, C.byref(v),
                                  C.byref(f), C.byref(bad))
    assert st == L.FGB_ERR_LAYOUT and bad.value == 2
    bad_opt = srt.options(TC)
    bad_opt.order = 7
    assert lib.fgb_host_sort_keys(C.byref(bad_opt), HEADER, len(HEADER), b.ctypes.data, off.ctypes.data, 1,
                                  keys.ctypes.data, C.byref(bad)) == L.FGB_ERR_INVALID_ARG


# ---- the whole key function on random records -------------------------------------------------------------------
@pytest.mark.parametrize("order,cell", [(TC, b"CB"), (TC, None), (CO, None)])
def test_random_records_match_the_oracle(srt, order, cell):
    recs = random_records(10000, seed=11)
    both(srt, recs, order, cell)


def test_verify_on_shuffled_and_sorted(srt):
    recs = random_records(3000, seed=5)
    rng = np.random.default_rng(1)
    for order, cell in ((TC, b"CB"), (TC, None), (CO, None)):
        for trial in range(3):
            shuffled = [recs[i] for i in rng.permutation(len(recs))]
            b, off = pack(shuffled)
            assert srt.verify(HEADER, b, off, order, cell) == S.verify(shuffled, HEADER, order, cell)
        ordered = S.sort_records(recs, HEADER, order, cell)
        b, off = pack(ordered)
        assert srt.verify(HEADER, b, off, order, cell) == (0, None) == S.verify(ordered, HEADER, order, cell)


# ---- the output header (sort/mod.rs) ----------------------------------------------------------------------------
def _hd(text):
    return next(ln for ln in text.decode().split("\n") if ln.startswith("@HD")).split("\t")[1:]


def test_sort_header(srt):
    from fgumi_b200 import bamio
    h = b"@HD\tVN:1.6\tSO:unsorted\tGO:query\tSS:template-coordinate\n@SQ\tSN:c\tLN:9\n@PG\tID:bwa\tPN:bwa\n"
    out = bamio.sort_header(h, CO)
    assert _hd(out) == ["VN:1.6", "SO:coordinate"]
    assert dict(f.split(":", 1) for f in _hd(out)) == S.output_header(h, CO)
    assert out.decode().rstrip("\n").split("\n")[-1].startswith("@PG\tID:fgumi_b200\tPN:fgumi_b200\tPP:bwa")
    out = bamio.sort_header(b"@HD\tVN:1.5\tSO:coordinate\tXY:z\n", TC)
    assert _hd(out) == ["VN:1.5", "XY:z", "SO:unsorted", "GO:query", "SS:template-coordinate"]
    assert dict(f.split(":", 1) for f in _hd(out)) == S.output_header(b"@HD\tVN:1.5\tSO:coordinate\tXY:z\n", TC)
    out = bamio.sort_header(b"@SQ\tSN:c\tLN:9\n", CO)
    assert out.split(b"\n")[0] == b"@HD\tSO:coordinate"
    bamio.check_group_sort_order(bamio.sort_header(h, TC), False)


def test_struct_size_of_sort_options(srt):
    from fgumi_b200 import lib as L
    assert L.load().fgb_struct_size(12) == C.sizeof(L.FgbSortOptions) == 24


# ---- the generators and references of tests/test_sort_records_scale_gpu.py -------------------------------------------
CASES = [(TC, b"CB"), (TC, None), (CO, None)]


@pytest.fixture(scope="module")
def bulk():
    """A bulk input as the scale tests build it, at 20 000 records, with a noise lead and an unaligned bodies array."""
    common, rare = SC.bulk_pool(3)
    f = SC.bulk_fields(20000, 3, len(common), len(rare))
    b, off = SC.materialize(common + rare, f, lead=77, skew=1, chunk=100_000)
    return b, off, f


@pytest.fixture(scope="module")
def grid():
    return SC.gather_grid(31)


def test_scale_bulk_input_is_what_it_claims(bulk):
    b, off, f = bulk
    n = len(off) - 1
    assert off[0] == 77 and b.ctypes.data % 4
    recs = SC.records_of(b, off, range(n))
    assert len(set(recs)) == n                                        # byte-unique
    for i in (0, 1, 4567, n - 1):
        r = recs[i]
        assert struct.unpack_from("<ii", r, 0) == (f["tid"][i], f["pos"][i])
        assert struct.unpack_from("<ii", r, 20) == (f["mtid"][i], f["mpos"][i])
        assert r[14] & 0x30 == f["strand"][i]
        assert int.from_bytes(r[9:12], "little") | int.from_bytes(r[28:32], "little") << 24 == i
    common, rare = SC.bulk_pool(3)
    pool = common + rare
    for i in np.flatnonzero(f["idx"] >= len(common))[:8]:            # the rest of each record is its pool record's
        r, p = recs[i], pool[f["idx"][i]]
        assert len(r) == len(p) and r[32:] == p[32:] and r[12:14] == p[12:14] and r[15:20] == p[15:20]
    assert {len(r) for r in rare} >= {65535, 65536, 65537}
    assert max(struct.unpack_from("<H", r, 12)[0] for r in rare) == 1000


def test_scale_serial_bytes_are_not_key_bytes(srt, bulk, grid):
    b, off, _ = bulk
    gb, goff = SC.pack(grid)
    rng = np.random.default_rng(8)
    sample = sorted(rng.choice(len(off) - 1, 2000, replace=False).tolist())
    grid_sample = [i for i, r in enumerate(grid) if i % 4 == 0 or len(r) > 60000]
    for bodies, rec_off, which in ((b, off, sample), (gb, goff, grid_sample)):
        at = rec_off[:-1].astype(np.int64)
        other = bodies.copy()
        for k in SC.SERIAL_BYTES:
            other[at + k] = rng.integers(0, 256, len(at), dtype=np.uint8)
        assert not np.array_equal(other, bodies)
        for order, cell in CASES:
            assert np.array_equal(srt.sort_keys(HEADER, bodies, rec_off, order, cell),
                                  srt.sort_keys(HEADER, other, rec_off, order, cell))
            assert S.keys(SC.records_of(bodies, rec_off, which), HEADER, order, cell) == \
                S.keys(SC.records_of(other, rec_off, which), HEADER, order, cell)


def test_scale_numpy_coordinate_key(srt, bulk):
    tids = SC.TIDS + [-2 ** 31, -2, 3, 2 ** 30]
    pos = SC.POS + [-2 ** 31, -2, 2 ** 31 - 2, 2 ** 30]
    recs = [rec(tid=t, pos=p, flags=fl) for t in tids for p in pos for fl in (0, 0x10, 0x4 | 0x10 | 0x20)]
    b, off = SC.pack_at(recs, 3, 1)
    want = [S.coordinate_key(r) for r in recs]
    assert SC.coordinate_keys(b, off).tolist() == want
    assert srt.sort_keys(HEADER, b, off, CO)[:, 0].tolist() == want
    assert M64 in want and 0 in want and any(k >= 1 << 63 for k in want if k != M64)   # tid < 0, and the wraps
    b, off, _ = bulk
    assert SC.coordinate_keys(b, off).tolist() == [S.coordinate_key(r) for r in SC.records_of(b, off, range(len(off) - 1))]


def test_scale_alignment_combinations(srt, bulk, grid):
    """Every (source offset, output offset, length) mod 4 combination reaches the record gather."""
    every = {(s, o, n) for s in range(4) for o in range(4) for n in range(4)}
    b, off, _ = bulk
    assert SC.alignments(off, SC.sorted_order(SC.coordinate_keys(b, off))) == every
    for cell in (b"CB", None):
        assert SC.alignments(off, SC.sorted_order(srt.sort_keys(HEADER, b, off, TC, cell))) == every
    gb, goff = SC.pack(grid)
    for order, cell in CASES:
        k = S.keys(grid, HEADER, order, cell)
        assert SC.alignments(goff, np.array(sorted(range(len(grid)), key=k.__getitem__))) == every


def test_scale_gather_grid_shapes(grid):
    lens = [len(r) for r in grid]
    assert set(range(32, 401)) <= set(lens)
    assert {65535, 65536, 65537, (1 << 20) + 3} <= set(lens)
    n_cig = [struct.unpack_from("<H", r, 12)[0] for r in grid]
    assert n_cig.count(65535) == 3
    long_mc = [r for r in grid if r.find(b"MCZ") > 0 and len(r) - r.find(b"MCZ") > 100_000]
    assert len(long_mc) == 3 and all(r.count(b"M") > 10_000 for r in long_mc)
    assert len(set(grid)) == len(grid)


def test_scale_references_equal_the_oracle_order(srt):
    """A stable np.argsort of the numpy coordinate keys and a stable np.lexsort of the host key words order records as
    the oracle's stable sort does, and the chunked expected stream is the oracle's stream (ties kept by serials)."""
    recs = SC.stamp_serials(random_records(4000, seed=12))
    b, off = SC.pack_at(recs, 5, 1)
    for order, cell in CASES:
        keys = SC.coordinate_keys(b, off) if order == CO else srt.sort_keys(HEADER, b, off, order, cell)
        perm = SC.sorted_order(keys)
        k = S.keys(recs, HEADER, order, cell)
        assert perm.tolist() == sorted(range(len(recs)), key=k.__getitem__)
        want = bytearray(S.sorted_stream(recs, HEADER, order, cell))
        SC.assert_stream(want, b, off, perm, chunk=5000)
        i = len(recs) // 2
        at = int(SC.stream_offsets(off, perm)[i]) + 4 + 9            # the serial of output record i
        want[at] ^= 1
        with pytest.raises(AssertionError, match="output record %d " % i):
            SC.assert_stream(want, b, off, perm, chunk=5000)


def test_scale_run_plan():
    """run_plan restates the run loop of fgb_sort_records; budget_for gives a first run that ends where asked."""
    def loop(off, budget, words):
        per, n, out, b = 68 + 8 * words, len(off) - 1, [0], 0
        while b < n:
            i = b + 1
            while i < n and 2 * (off[i + 1] - off[b]) + (i + 1 - b) * (per + 4) <= budget:
                i += 1
            out.append(i)
            b = i
        return out
    rng = np.random.default_rng(4)
    off = [9] + (9 + np.cumsum(rng.integers(32, 700, 3000))).tolist()
    for words in (1, 5):
        for budget in (1, 2000, 30000, 10 ** 6, 10 ** 9):
            assert SC.run_plan(np.array(off, np.uint64), budget, words) == loop(off, budget, words)
        assert SC.run_plan(off, SC.budget_for(off, 1234, words), words)[1] == 1234
