"""fgb_sort_records in queryname order (lexicographic and natural) on the device against tests/queryname_oracle.py:
byte-identical streams on shuffled records with many records per name (equal keys test stability), many runs of
different key widths merged by the host comparator against one run, the edges, one run past a 64 MiB staging buffer,
and bamio.sort_file.  Every output also passes `verify`."""
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import queryname_oracle as Q       # noqa: E402
from tests.bam_builder import make_record      # noqa: E402
from tests.queryname_cases import name_records, random_names  # noqa: E402
from tests.sort_cases import STAGE_BYTES, fit, pack  # noqa: E402

pytestmark = pytest.mark.gpu
ORDERS = ["queryname", "queryname::natural"]
HEADER = b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:1000000\n@PG\tID:bwa\tPN:bwa\n"


@pytest.fixture(scope="module")
def mods():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, sort
    return sort, bamio


def check(mods, out, recs, order):
    sort, bamio = mods
    assert out == Q.sorted_stream(recs, order)
    if out:
        assert sort.verify(HEADER, *bamio.split_stream(out), order, None, n_threads=4) == (0, None)


@pytest.mark.parametrize("order", ORDERS)
def test_sort_matches_the_oracle(mods, order):
    sort = mods[0]
    s = sort.RecordSorter(0, order, n_threads=4)
    for seed, n_names in ((1, 300), (2, 3000)):
        recs = name_records(random_names(n_names, seed), seed)
        out = s.sort(HEADER, *pack(recs))
        check(mods, out, recs, order)
        t = s.last_timing()
        assert t["merge_ms"] == 0 and t["key_kernel_ms"] > 0
    s.close()


@pytest.mark.parametrize("order", ORDERS)
def test_many_runs_equal_one_run(mods, order):
    sort = mods[0]
    # short names first and 254-byte names last, so that runs differ in their key words; the long names share
    # prefixes with each other and with the short ones
    short = name_records([b"read%d" % i for i in range(0, 600, 3)] + [b"r%03d" % i for i in range(40)], seed=3)
    rng = np.random.default_rng(4)
    longs = [b"read" + b"0" * int(rng.integers(0, 3)) + b"%d" % rng.integers(0, 600) + b":" +
             bytes(int(c) for c in rng.choice(np.frombuffer(b"09a:", np.uint8), 200)) for _ in range(60)]
    longs = [nm + b"x" * (254 - len(nm)) for nm in longs]
    recs = short + name_records(longs, seed=5, per_name=4)
    b, off = pack(recs)
    one = sort.RecordSorter(0, order).sort(HEADER, b, off)
    check(mods, one, recs, order)
    for budget in (1, 40000, 300000):
        s = sort.RecordSorter(0, order, device_bytes=budget, n_threads=2)
        assert s.sort(HEADER, b, off) == one
        assert s.last_timing()["merge_ms"] > 0
        s.close()


@pytest.mark.parametrize("order", ORDERS)
def test_edge_cases(mods, order):
    sort = mods[0]
    s = sort.RecordSorter(0, order)
    assert s.sort(HEADER, np.zeros(0, np.uint8), np.zeros(1, np.uint64)) == b""
    r = make_record(name=b"only", flags=0x41)
    assert s.sort(HEADER, *pack([r])) == struct.pack("<I", len(r)) + r
    same = name_records([b"same"] * 50, seed=6)                # every key equal within each flag: input order
    check(mods, s.sort(HEADER, *pack(same)), same, order)
    empty = [make_record(name=b"", flags=f, tlen=i) for i, f in enumerate([0x41, 0x81, 0x0, 0x141] * 40)]
    for k in range(0, len(empty), 7):                           # l_read_name 0 and a name past the record
        e = bytearray(empty[k])
        e[8] = 0 if k % 2 else 200
        empty[k] = bytes(e)
    check(mods, s.sort(HEADER, *pack(empty)), empty, order)
    # names equal only in the natural order: it sorts them by flag, then input order; lexicographic by bytes
    zeros = [b"r1", b"r01", b"r001", b"r0001:7", b"r1:07", b"r0", b"r00", b"r000"]
    recs = name_records(zeros * 5, seed=7)
    out = s.sort(HEADER, *pack(recs))
    check(mods, out, recs, order)
    s.close()


@pytest.mark.parametrize("order", ORDERS)
def test_one_run_past_a_staging_buffer(mods, order):
    sort = mods[0]
    names = random_names(6000, seed=8)
    base = name_records(names, seed=9, per_name=4)
    recs = [fit(r, 3500 + i % 7) for i, r in enumerate(base)]  # 24 000 records, 84 MB: two staging chunks
    b, off = pack(recs)
    assert int(off[-1]) > STAGE_BYTES
    s = sort.RecordSorter(0, order, n_threads=3)
    out = s.sort(HEADER, b, off)
    assert s.last_timing()["merge_ms"] == 0
    check(mods, out, recs, order)
    s.close()


def test_sort_file(mods, tmp_path):
    sort, bamio = mods
    from fgumi_b200 import lib as L
    import ctypes as C
    recs = name_records(random_names(400, seed=10), seed=11)
    payload = bamio.mapped_bam_header(HEADER) + b"".join(struct.pack("<I", len(r)) + r for r in recs)
    lib = L.load()
    comp = np.empty(lib.fgb_bgzf_bound(len(payload)), np.uint8)
    cn = C.c_size_t()
    assert lib.fgb_bgzf_compress(payload, len(payload), 1, 2, 1, comp.ctypes.data, len(comp), C.addressof(cn)) == 0
    src = str(tmp_path / "in.bam")
    comp[:cn.value].tofile(src)
    for order in ORDERS:
        dst = str(tmp_path / ("out_%s.bam" % order.replace(":", "_")))
        tm = bamio.sort_file(src, dst, sort.RecordSorter(0, order), n_threads=2)
        assert tm["input_records"] == len(recs) and "key_kernel_ms" in tm
        text, ob, ooff, _ = bamio.read_bam(dst, 2)
        got = [ob[int(ooff[i]):int(ooff[i + 1])].tobytes() for i in range(len(ooff) - 1)]
        assert got == Q.sort_records(recs, order)
        assert sort.verify(text, ob, ooff, order, None) == (0, None)
        hd = dict(f.split(":", 1) for f in text.decode().split("\n")[0].split("\t")[1:])
        assert hd == Q.output_header(HEADER, order) and hd["VN"] == "1.6"
        pg = [ln for ln in text.decode().split("\n") if ln.startswith("@PG")]
        assert pg[-1].startswith("@PG\tID:fgumi_b200\tPN:fgumi_b200\tPP:bwa")
        bamio.check_group_sort_order(text, True)
