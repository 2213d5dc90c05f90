"""fgb_sort_records on the device against oracle/sort_oracle.py: byte-identical streams for both orders with and
without a cell tag, many runs merged on the host against one run, edge cases, sort then group in memory against the
oracle's sort followed by its group, and bamio.sort_file on a generated BAM."""
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import group_oracle as G     # noqa: E402
from oracle import sort_oracle as S      # noqa: E402
from tests.bam_builder import make_record  # noqa: E402
from tests.sort_cases import HEADER, pack, random_records  # noqa: E402

pytestmark = pytest.mark.gpu
TC, CO = "template-coordinate", "coordinate"
CASES = [(TC, b"CB"), (TC, None), (CO, None)]


@pytest.fixture(scope="module")
def mods():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, group, sort, synth
    return sort, group, synth, bamio


def _shuffled(n, seed):
    recs = random_records(n, seed=seed)
    return [recs[i] for i in np.random.default_rng(seed).permutation(len(recs))]


@pytest.mark.parametrize("order,cell", CASES)
def test_sort_matches_the_oracle(mods, order, cell):
    sort = mods[0]
    s = sort.RecordSorter(0, order, cell, n_threads=4)
    for seed, n in ((1, 5000), (2, 20000)):
        recs = _shuffled(n, seed)
        b, off = pack(recs)
        out = s.sort(HEADER, b, off)
        assert out == S.sorted_stream(recs, HEADER, order, cell)
        ob, ooff = mods[3].split_stream(out)
        assert sort.verify(HEADER, ob, ooff, order, cell) == (0, None)
        t = s.last_timing()
        assert t["merge_ms"] == 0 and t["key_kernel_ms"] > 0
    s.close()


@pytest.mark.parametrize("order,cell", CASES)
def test_many_runs_equal_one_run(mods, order, cell):
    sort = mods[0]
    recs = _shuffled(6000, 3)
    b, off = pack(recs)
    one = sort.RecordSorter(0, order, cell).sort(HEADER, b, off)
    for budget in (1, 40000, 300000):
        s = sort.RecordSorter(0, order, cell, device_bytes=budget, n_threads=2)
        assert s.sort(HEADER, b, off) == one
        t = s.last_timing()
        assert t["merge_ms"] > 0
    assert one == S.sorted_stream(recs, HEADER, order, cell)


def test_edge_cases(mods):
    sort = mods[0]
    for order, cell in CASES:
        s = sort.RecordSorter(0, order, cell)
        assert s.sort(HEADER, np.zeros(0, np.uint8), np.zeros(1, np.uint64)) == b""
        r = random_records(1, seed=9)
        assert s.sort(HEADER, *pack(r)) == struct.pack("<I", len(r[0])) + r[0]
        # every record unmapped without a position: every key word constant except the name hash (or all of them)
        un = [make_record(name=b"u%d" % (i % 7), flags=0x4, ref_id=-1, pos=-1, seq=b"ACGT") for i in range(3000)]
        for k in range(0, 3000, 5):
            un[k] = un[0]
        assert s.sort(HEADER, *pack(un)) == S.sorted_stream(un, HEADER, order, cell)
        same = [un[0]] * 100
        assert s.sort(HEADER, *pack(same)) == S.sorted_stream(same, HEADER, order, cell)


def test_errors(mods):
    sort = mods[0]
    from fgumi_b200 import lib as L
    s = sort.RecordSorter(0, TC)
    recs = random_records(10, seed=4)
    recs[6] = recs[6][:20]
    with pytest.raises(L.FgbError) as e:
        s.sort(HEADER, *pack(recs))
    assert e.value.status == L.FGB_ERR_LAYOUT and "record 6" in str(e.value)
    ok = random_records(50, seed=4)
    assert s.sort(HEADER, *pack(ok)) == S.sorted_stream(ok, HEADER, TC, b"CB")


def test_sort_then_group_in_memory(mods):
    sort, group, synth, bamio = mods
    from oracle import umi_oracle as U
    hdr, b, off = synth.mapped_templates(60, molecules=4, mean_family=3.0, seed=21, unmapped_mate_rate=0.3,
                                         secondary_rate=0.1, cross_contig_rate=0.2, reverse_rate=0.4)
    recs = [b[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]
    recs = [recs[i] for i in np.random.default_rng(2).permutation(len(recs))]
    sb, soff = pack(recs)
    stream = sort.RecordSorter(0, TC).sort(hdr, sb, soff)
    want_sorted = S.sort_records(recs, hdr, TC)
    assert stream == b"".join(struct.pack("<I", len(r)) + r for r in want_sorted)
    gb, goff = bamio.split_stream(stream)
    keep, groups = group.group_by_position(gb, goff, hdr)
    kb, koff = group.compact(gb, goff, keep)
    g = group.ReadGrouper(0, "adjacency", 1)
    g.add_groups(kb, koff, groups)
    got = g.flush()
    cfg = G.Config(strategy=U.ADJACENCY, edits=1)
    want, _ = G.group_stream(want_sorted, hdr, cfg)
    assert got == want


def test_sort_file(mods, tmp_path):
    sort, group, synth, bamio = mods
    from fgumi_b200 import lib as L
    import ctypes as C
    hdr, b, off = synth.mapped_templates(40, molecules=3, seed=5, unmapped_mate_rate=0.3, secondary_rate=0.1,
                                         cross_contig_rate=0.2)
    recs = [b[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]
    recs = [recs[i] for i in np.random.default_rng(8).permutation(len(recs))]
    payload = bamio.mapped_bam_header(hdr) + b"".join(struct.pack("<I", len(r)) + r for r in recs)
    lib = L.load()
    comp = np.empty(lib.fgb_bgzf_bound(len(payload)), np.uint8)
    cn = C.c_size_t()
    assert lib.fgb_bgzf_compress(payload, len(payload), 1, 2, 1, comp.ctypes.data, len(comp), C.addressof(cn)) == 0
    src = str(tmp_path / "in.bam")
    comp[:cn.value].tofile(src)
    for order in (TC, CO):
        dst = str(tmp_path / ("out_%s.bam" % order))
        tm = bamio.sort_file(src, dst, sort.RecordSorter(0, order), n_threads=2)
        assert tm["input_records"] == len(recs) and "key_kernel_ms" in tm
        text, ob, ooff, _ = bamio.read_bam(dst, 2)
        got = [ob[int(ooff[i]):int(ooff[i + 1])].tobytes() for i in range(len(ooff) - 1)]
        assert got == S.sort_records(recs, hdr, order)
        hd = dict(f.split(":", 1) for f in text.decode().split("\n")[0].split("\t")[1:])
        assert hd == S.output_header(hdr, order) and hd["VN"] == "1.6"
        pg = [ln for ln in text.decode().split("\n") if ln.startswith("@PG")]
        assert pg[-1].startswith("@PG\tID:fgumi_b200\tPN:fgumi_b200\tPP:bwa")
        if order == TC:
            bamio.check_group_sort_order(text, False)
