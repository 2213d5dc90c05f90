"""`fgumi sort --order queryname` and `queryname::natural` without a GPU: cases restated from the reference's tests
(sort/keys.rs, fgumi-raw-bam sort.rs, commands/sort.rs) against tests/queryname_oracle.py and against the product's
key words (fgb_host_sort_name_key, the code the key kernel runs) and `verify`; the key encoding's order equal to the
oracle comparator's, equality included, on every short string over an edge alphabet and on random names; the
extraction edges, the output header and the C-ABI around the new orders."""
import ctypes as C
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import queryname_oracle as Q       # noqa: E402
from tests.bam_builder import make_record      # noqa: E402
from tests.queryname_cases import ALPHABET, name_records, random_names  # noqa: E402
from tests.sort_cases import pack              # noqa: E402

LEX, NAT = "queryname", "queryname::natural"


@pytest.fixture(scope="module")
def srt():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import sort
    return sort


def key_cmp(srt, ra, rb, order):
    ka, kb = srt.name_key(ra, order), srt.name_key(rb, order)
    return (ka > kb) - (ka < kb)


def check_pair(srt, ra, rb, order, want=None):
    """The oracle and the product's key words agree on the pair (and with `want` when given)."""
    o = Q.compare(ra, rb, order)
    assert key_cmp(srt, ra, rb, order) == o, (ra[32:], rb[32:], order)
    assert key_cmp(srt, rb, ra, order) == -o
    if want is not None:
        assert o == want, (ra[32:], rb[32:], order)


def test_flag_order_values(srt):
    # keys.rs:679-712, 843-866, 872-885, 889-901, 905-912
    for f, want in ((0x0, 0x0), (0x40, 0x4000), (0x80, 0x8000), (0x100, 0x800), (0x800, 0x100), (0x840, 0x4100),
                    (0x140, 0x4800), (0x880, 0x8100), (0x180, 0x8800), (0x63, 0x4000), (0x93, 0x8000),
                    (0x841, 0x4100), (0x181, 0x8800), (0xc0, 0xc000), (113, 0x4000), (177, 0x8000), (2161, 0x4100)):
        assert Q.queryname_flag_order(f) == want
        for order in (LEX, NAT):
            assert srt.name_key(make_record(name=b"rea", flags=f), order)[-1] & 0xFFFF == want


def test_flag_order_sequence(srt):
    # keys.rs:718-754 (all twelve categories in order), 758-815, 820-839 (irrelevant flags)
    seq = [0x0, 0x800, 0x100, 0x40, 0x840, 0x140, 0x80, 0x880, 0x180, 0xc0, 0x8c0, 0x1c0]
    recs = [make_record(name=b"rea", flags=f) for f in seq]
    for order in (LEX, NAT):
        for a, b in zip(recs, recs[1:]):
            check_pair(srt, a, b, order, -1)
        for i, j in itertools.combinations(range(len(recs)), 2):
            check_pair(srt, recs[i], recs[j], order, -1)
    irrelevant = 0x01 | 0x02 | 0x04 | 0x08 | 0x10 | 0x20 | 0x200 | 0x400
    for f in (0x40, 0x880, 0x100):
        for order in (LEX, NAT):
            check_pair(srt, make_record(name=b"x", flags=f), make_record(name=b"x", flags=f | irrelevant), order, 0)


# natural_compare_nul (fgumi-raw-bam sort.rs:282-291)
NUL_CASES = [(b"read1", b"read2", -1), (b"read2", b"read10", -1), (b"01", b"1", 0), (b"a", b"b", -1), (b"", b"", 0),
             (b"SRR1.9", b"SRR1.10", -1)]

# The natural-order cases of keys.rs:922-1376 on which the slice comparator (natural_compare) and the NUL variant the
# sort uses agree.  Left out: the leading-zero tie-breaks (keys.rs:1020-1030, 1198, 1281-1326), where the slice variant
# orders "01" after "1" by length but natural_compare_nul, and so `fgumi sort`, finds the names equal.
SLICE_CASES = [
    (b"abc", b"abd", -1), (b"abd", b"abc", 1), (b"abc", b"abc", 0), (b"ABC", b"abc", -1), (b"z", b"a", 1),
    (b"aaa", b"aab", -1), (b"ZZZ", b"aaa", -1),
    (b"", b"", 0), (b"", b"x", -1), (b"x", b"", 1), (b"", b"0", -1), (b"0", b"", 1), (b"a", b"a", 0), (b"0", b"0", 0),
    (b"abc", b"abcd", -1), (b"abcd", b"abc", 1), (b"read", b"read1", -1), (b"read1", b"read", 1), (b"a1", b"a1b", -1),
    (b"a1b", b"a1", 1),
    (b"0", b"1", -1), (b"1", b"2", -1), (b"9", b"0", 1), (b"5", b"5", 0),
    (b"2", b"10", -1), (b"10", b"2", 1), (b"9", b"10", -1), (b"10", b"9", 1), (b"10", b"10", 0), (b"99", b"100", -1),
    (b"100", b"99", 1), (b"123", b"456", -1), (b"456", b"123", 1), (b"999", b"1000", -1), (b"1000", b"999", 1),
    (b"02", b"1", 1), (b"02", b"10", -1), (b"009", b"10", -1), (b"0100", b"99", 1),
    (b"0", b"a", -1), (b"9", b"a", -1), (b"a", b"0", 1), (b"a", b"9", 1), (b"1", b"A", -1), (b"1", b"Z", -1),
    (b"1", b"z", -1),
    (b"a1b2", b"a1b10", -1), (b"a1b10", b"a1b2", 1), (b"x10y20", b"x10y3", 1), (b"x10y3", b"x10y20", -1),
    (b"abc123def", b"abc123deg", -1), (b"abc123def", b"abc124def", -1), (b"abc124def", b"abc123def", 1),
    (b"file1part2", b"file1part10", -1), (b"file2part1", b"file10part1", -1), (b"v1.2.3", b"v1.2.10", -1),
    (b"v1.2.10", b"v1.10.2", -1),
    (b"A00132:53:HFHJKDSXX:1:1101:12345:67890", b"A00132:53:HFHJKDSXX:1:1102:12345:67890", -1),
    (b"A00132:53:HFHJKDSXX:1:1101:12345:67890", b"A00132:53:HFHJKDSXX:1:1101:12346:67890", -1),
    (b"A00132:53:HFHJKDSXX:1:1101:12345:67890", b"A00132:53:HFHJKDSXX:2:1101:12345:67890", -1),
    (b"A00132:53:HFHJKDSXX:1:1101:12345:67890", b"A00132:54:HFHJKDSXX:1:1101:12345:67890", -1),
    (b"A00132:53:HFHJKDSXX:1:1101:12345:67890", b"A00132:53:HFHJKDSXX:1:1101:12345:67890", 0),
    (b"A00132:53:HFHJKDSXX:1:1101:12345:67890", b"B00132:53:HFHJKDSXX:1:1101:12345:67890", -1),
    (b"INST:1:FLOW:1:1101:1:1", b"INST:1:FLOW:1:2201:1:1", -1),
    (b"SRR099966.1", b"SRR099966.2", -1), (b"SRR099966.9", b"SRR099966.10", -1),
    (b"SRR099966.99", b"SRR099966.100", -1), (b"SRR099966.12345", b"SRR099966.12346", -1),
    (b"SRR099966.12345", b"SRR099966.12345", 0), (b"SRR099966.12345", b"SRR099967.1", -1), (b"SRR1.1", b"SRR2.1", -1),
    (b"SRR9.1", b"SRR10.1", -1),
    (b"mol000001_read0001", b"mol000001_read0002", -1), (b"mol000001_read0009", b"mol000001_read0010", -1),
    (b"mol000001_read0001", b"mol000002_read0001", -1), (b"mol1_read1", b"mol1_read2", -1),
    (b"mol2_read1", b"mol10_read1", -1),
    (b"x99999999999999999999999999999999999999", b"x100000000000000000000000000000000000000", -1),
    (b"prefix99999999999999999999999999suffix", b"prefix99999999999999999999999999suffix", 0),
    (b"x99999999999999999999999999999999999998", b"x99999999999999999999999999999999999999", -1),
    (b"read18446744073709551615", b"read18446744073709551616", -1),
    (b"read99999999999999999999", b"read100000000000000000000", -1),
    (b"a0", b"aa", -1), (b"a9", b"aa", -1), (b"aa", b"a0", 1),
    (b"a1b", b"a1c", -1), (b"a10b", b"a10c", -1), (b"a10b", b"a2c", 1),
    (b"read1", b"read1a", -1), (b"read1a", b"read1", 1), (b"read10", b"read10a", -1), (b"read10a", b"read10", 1),
    (b"r1.1.1", b"r1.1.2", -1), (b"r1.1.9", b"r1.1.10", -1), (b"r1.9.1", b"r1.10.1", -1), (b"r9.1.1", b"r10.1.1", -1),
    (b"a12", b"a9", 1), (b"\xff", b"\xfe", 1), (b"\x80", b"\x7f", 1), (b"0", b"\x80", -1),
]

# Names the reference sorts as a list (keys.rs:1090-1122, 1381-1437), in their natural order
NATURAL_LISTS = [
    [b"r000", b"r001", b"r002", b"r003", b"r004", b"u1", b"x1", b"x2", b"x3", b"x4", b"x5", b"x6"],
    [b"r005", b"r006", b"r007", b"x7", b"x8", b"x9", b"x10", b"x11", b"x12"],
    [b"INST:1:FLOW:1:1101:1:1", b"INST:1:FLOW:1:1101:1:2", b"INST:1:FLOW:1:1101:2:1", b"INST:1:FLOW:1:1102:1:1",
     b"INST:1:FLOW:2:1101:1:1", b"INST:2:FLOW:1:1101:1:1", b"INST:10:FLOW:1:1101:1:1", b"INST:100:FLOW:1:1101:1:1",
     b"INST:100:FLOW:2:2201:9999:1"],
    [b"SRR099966.1", b"SRR099966.2", b"SRR099966.9", b"SRR099966.10", b"SRR099966.99", b"SRR099966.100"],
]


@pytest.mark.parametrize("a,b,want", NUL_CASES + SLICE_CASES)
def test_natural_cases(srt, a, b, want):
    assert Q.natural_compare_nul(a, b) == want
    check_pair(srt, make_record(name=a, flags=0x40), make_record(name=b, flags=0x40), NAT, want)


def test_natural_lists(srt):
    for names in NATURAL_LISTS:
        recs = [make_record(name=nm) for nm in names]
        shuffled = [recs[i] for i in np.random.default_rng(len(names)).permutation(len(recs))]
        assert Q.sort_records(shuffled, NAT) == recs
        keys = sorted(shuffled, key=lambda r: srt.name_key(r, NAT))
        assert keys == recs


def test_leading_zero_names_are_equal_in_the_natural_order(srt):
    # keys.rs:1281-1326 order these by length (slice variant); natural_compare_nul, which the sort uses, finds them
    # equal, so the flag order decides and then the input order
    for a, b in ((b"00", b"0"), (b"000", b"00"), (b"01", b"1"), (b"00100", b"100"), (b"a0b", b"a00b"),
                 (b"a0b", b"a000b"), (b"mol1_read1", b"mol000001_read0001")):
        assert Q.natural_compare_nul(a, b) == 0
        check_pair(srt, make_record(name=a, flags=0x80), make_record(name=b, flags=0x40), NAT, 1)
        check_pair(srt, make_record(name=a, flags=0x40), make_record(name=b, flags=0x40), NAT, 0)
        assert srt.name_key(make_record(name=a), NAT) == srt.name_key(make_record(name=b), NAT)


def test_compare_queryname_raw_cases(srt):
    # fgumi-raw-bam sort.rs:392-425: a byte compare of the names, then the flags
    a, b = make_record(name=b"abc"), make_record(name=b"xyz")
    check_pair(srt, a, b, LEX, -1)
    check_pair(srt, make_record(name=b"rea", flags=0x40), make_record(name=b"rea", flags=0x80), LEX, -1)
    r = make_record(name=b"rea", flags=0x40, ref_id=1, pos=100)
    check_pair(srt, r, r, LEX, 0)
    e = bytearray(33)                                   # l_read_name = 0 on both sides
    check_pair(srt, bytes(e), bytes(e), LEX, 0)


def _exhaustive_names():
    return [bytes(t) for k in range(4) for t in itertools.product(ALPHABET, repeat=k)]


@pytest.mark.parametrize("order", [LEX, NAT])
def test_encoding_is_exact_on_every_short_string(srt, order):
    names = _exhaustive_names()
    keys = [srt.name_key(make_record(name=nm), order) for nm in names]
    cmp = Q.natural_compare_nul if order == NAT else Q.lexicographic_compare
    bad = [(a, b) for (a, ka), (b, kb) in itertools.combinations(zip(names, keys), 2)
           if (ka > kb) - (ka < kb) != cmp(a, b)]
    assert not bad, bad[:5]


@pytest.mark.parametrize("order", [LEX, NAT])
def test_encoding_is_exact_on_random_names(srt, order):
    names = random_names(20000, seed=11)
    flags = np.random.default_rng(12).choice([0x41, 0x81, 0x141, 0x841, 0x0, 0x181], len(names))
    recs = [make_record(name=nm, flags=int(f)) for nm, f in zip(names, flags)]
    keys = [srt.name_key(r, order) for r in recs]
    by_key = sorted(range(len(recs)), key=lambda i: keys[i])
    # consecutive records in key order: the comparator agrees on each, so (both being total preorders) on every pair
    for i, j in zip(by_key, by_key[1:]):
        want = Q.compare(recs[i], recs[j], order)
        assert (keys[i] > keys[j]) - (keys[i] < keys[j]) == want, (names[i], names[j])
    rng = np.random.default_rng(13)
    for i, j in rng.integers(0, len(recs), size=(20000, 2)):
        assert (keys[i] > keys[j]) - (keys[i] < keys[j]) == Q.compare(recs[i], recs[j], order)
    # the ties the names were built to produce are there: equal keys under different bytes
    if order == NAT:
        assert sum(1 for i, j in zip(by_key, by_key[1:]) if keys[i] == keys[j] and names[i] != names[j]) > 0


def test_word_counts(srt):
    from fgumi_b200 import lib as L
    lib = L.load()
    for order, nm, want in ((LEX, b"", 1), (LEX, b"a" * 8, 2), (LEX, b"a" * 9, 3), (LEX, b"a" * 254, 33),
                            (NAT, b"", 1), (NAT, b"a", 2), (NAT, b"abcd", 3), (NAT, b"1a" * 127, 65)):
        r = make_record(name=nm)
        words = np.zeros(65, np.uint64)
        n = C.c_uint32()
        o = srt.options(order, None, 0, 1)
        rb = np.frombuffer(r, np.uint8)
        assert lib.fgb_host_sort_name_key(C.byref(o), rb.ctypes.data, len(r), words.ctypes.data, 65, C.byref(n)) == 0
        assert n.value == want
        # a one-digit run is three bytes: 127 of them and 127 letters fill 508 of the 512 bytes of 64 words
        if nm == b"1a" * 127:
            assert int(words[64]) >> 16 == 508
        assert lib.fgb_host_sort_name_key(C.byref(o), rb.ctypes.data, len(r), words.ctypes.data, want - 1,
                                          C.byref(n)) == L.FGB_ERR_INVALID_ARG and n.value == want
        assert lib.fgb_host_sort_name_key(C.byref(o), rb.ctypes.data, 31, words.ctypes.data, 65,
                                          C.byref(n)) == L.FGB_ERR_LAYOUT
    o = srt.options("coordinate", None, 0, 1)
    rb = np.frombuffer(make_record(name=b"x"), np.uint8)
    assert lib.fgb_host_sort_name_key(C.byref(o), rb.ctypes.data, len(rb), words.ctypes.data, 65,
                                      C.byref(n)) == L.FGB_ERR_INVALID_ARG


def test_extraction_edges(srt):
    base = make_record(name=b"abc", flags=0x40)
    empty = make_record(name=b"", flags=0x40)
    for lrn in (0, 1):
        r = bytearray(base)
        r[8] = lrn
        assert Q.name_and_flags(bytes(r)) == (b"", 0x4000)
        for order in (LEX, NAT):
            check_pair(srt, bytes(r), empty, order, 0)
    past = bytearray(base)
    past[8] = 200                                       # the name runs past the record: empty
    assert Q.name_and_flags(bytes(past))[0] == b""
    for order in (LEX, NAT):
        check_pair(srt, bytes(past), empty, order, 0)
        check_pair(srt, bytes(past), base, order, -1)
    # an embedded NUL: kept by the byte compare, where the name ends for the natural one
    nul, cut = make_record(name=b"ab\0z"), make_record(name=b"ab")
    check_pair(srt, nul, cut, LEX, 1)
    check_pair(srt, nul, cut, NAT, 0)
    check_pair(srt, make_record(name=b"ab\0"), cut, LEX, 1)
    check_pair(srt, make_record(name=b"ab\0\0"), make_record(name=b"ab\0"), LEX, 1)
    check_pair(srt, make_record(name=b"\0", flags=0x40), empty, NAT, 0)


@pytest.mark.parametrize("order", [LEX, NAT])
def test_verify_on_shuffled_and_sorted(srt, order):
    recs = name_records(random_names(1500, seed=21), seed=22, per_name=3)
    b, off = pack(recs)
    got = srt.verify(b"", b, off, order, None, n_threads=3)
    assert got == Q.verify(recs, order) and got[0] > 0
    s = Q.sort_records(recs, order)
    assert srt.verify(b"", *pack(s), order, None, n_threads=3) == (0, None) == Q.verify(s, order)
    # one swap: a violation at the swapped position, found on any thread count
    i = next(k for k in range(1, len(s)) if Q.compare(s[k - 1], s[k], order) < 0)
    s[i - 1], s[i] = s[i], s[i - 1]
    for t in (1, 4, 7):
        assert srt.verify(b"", *pack(s), order, None, n_threads=t) == Q.verify(s, order) == (1, i)


def test_sort_header(srt):
    from fgumi_b200 import bamio
    h = b"@HD\tVN:1.6\tSO:coordinate\tGO:query\tSS:coordinate:x\n@SQ\tSN:c\tLN:9\n@PG\tID:bwa\tPN:bwa\n"
    for order, ss in ((LEX, "lexicographic"), (NAT, "natural")):
        out = bamio.sort_header(h, order)
        hd = out.decode().split("\n")[0]
        assert hd == "@HD\tVN:1.6\tSO:queryname\tSS:" + ss
        assert dict(f.split(":", 1) for f in hd.split("\t")[1:]) == Q.output_header(h, order)
        assert out.decode().split("\n")[-2].startswith("@PG\tID:fgumi_b200\tPN:fgumi_b200\tPP:bwa")
        bamio.check_group_sort_order(out, True)
        with pytest.raises(ValueError):
            bamio.check_group_sort_order(out, False)
        assert bamio.sort_header(b"@SQ\tSN:c\tLN:9\n", order).startswith(b"@HD\tSO:queryname\tSS:" + ss.encode())


def test_abi(srt):
    from fgumi_b200 import lib as L
    lib = L.load()
    assert lib.fgb_struct_size(12) == 24 == C.sizeof(L.FgbSortOptions)
    assert (L.FGB_SORT_QUERYNAME, L.FGB_SORT_QUERYNAME_NATURAL) == (2, 3)
    assert srt.ORDERS["queryname"] == 2 and srt.ORDERS["queryname::natural"] == 3
    b, off = pack([make_record(name=b"x")])
    keys = np.zeros(5, np.uint64)
    bad = C.c_uint64()
    for order in (LEX, NAT):
        o = srt.options(order, None, 0, 1)
        assert lib.fgb_host_sort_keys(C.byref(o), b"", 0, b.ctypes.data, off.ctypes.data, 1, keys.ctypes.data,
                                      C.byref(bad)) == L.FGB_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        srt.options("queryname::lex")
    with pytest.raises(ValueError):
        srt.name_key(make_record(name=b"x"), "coordinate")
    with pytest.raises(L.FgbError):
        srt.name_key(b"\0" * 20, LEX)
