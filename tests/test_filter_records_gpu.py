"""`fgumi filter --ref` on the device against tests/filter_oracle.py: the kept stream, the rejects stream and the
counters byte-identical to the oracle for simplex and duplex records on both strands, with and without tag reversal,
in template and single-read mode, on 1 and 6 host threads, over several calls on one handle, with 65 535-base reads,
with a device budget small enough for several runs and with staging buffers small enough that uploads and downloads
cross many chunks; the reference's alignment-tag known answers through the device; every call-failing error once,
emitting nothing, and the first of two errors of different kinds; and bamio.filter_file end to end, whole and in
QNAME-cut batches, on a BAM built from tests/bam_builder.py records and a written FASTA."""
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import filter_oracle as O      # noqa: E402
from tests import filter_streams as S     # noqa: E402
from tests.bam_builder import make_record   # noqa: E402

pytestmark = pytest.mark.gpu

CONFIGS = [
    dict(max_no_call_fraction=0.5, max_base_error_rate=(0.3,)),
    dict(min_reads=(3, 2, 1), max_no_call_fraction=0.6, max_base_error_rate=(0.3,), min_mean_base_quality=20.0,
         require_ss_agreement=True, min_base_quality=5),
    dict(max_no_call_fraction=40.0, max_read_error_rate=(0.5,), max_base_error_rate=(0.5,)),
]


@pytest.fixture(scope="module")
def mods():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import bamio, filter as F
    return F, bamio


@pytest.fixture(scope="module")
def world(mods, tmp_path_factory):
    F, _ = mods
    contigs = S.genome(7)
    path = tmp_path_factory.mktemp("ref") / "ref.fa"
    path.write_bytes(S.fasta(contigs, crlf=True))
    ref = F.Reference(str(path))
    yield contigs, ref, O.parse_fasta(path.read_bytes())
    ref.close()


def product_kw(cfg_kw):   # the oracle's option names -> RecordFilter's
    kw = dict(cfg_kw)
    if "require_ss_agreement" in kw:
        kw["require_single_strand_agreement"] = kw.pop("require_ss_agreement")
    return kw


def run(F, ref, hdr, recs, cfg_kw, tmpl, rev, threads=1, device_bytes=0, use_ref=True):
    rf = F.RecordFilter(filter_by_template=tmpl, reverse_per_base_tags=rev, track_rejects=True, n_threads=threads,
                        device_bytes=device_bytes, **product_kw(cfg_kw))
    try:
        b, off = S.pack(recs)
        return rf.filter(hdr, b, off, ref if use_ref else None), rf.last_timing()
    finally:
        rf.close()


def oracle(recs, hdr, cfg_kw, tmpl, rev, genome):
    return O.filter_records(recs, hdr, O.Config(filter_by_template=tmpl, reverse_per_base_tags=rev, **cfg_kw), genome)


@pytest.mark.parametrize("ci", range(len(CONFIGS)))
@pytest.mark.parametrize("tmpl", [True, False])
@pytest.mark.parametrize("rev", [False, True])
def test_streams_match_oracle(mods, world, ci, tmpl, rev):
    F, _ = mods
    contigs, ref, genome = world
    hdr = S.header(contigs)
    recs = S.records(100 + ci, contigs, n_templates=400)
    want = oracle(recs, hdr, CONFIGS[ci], tmpl, rev, genome)
    for threads in (1, 6):
        (kept, rej, st), tm = run(F, ref, hdr, recs, CONFIGS[ci], tmpl, rev, threads)
        assert st == want[2]
        assert kept == want[0]
        assert rej == want[1]
    assert want[2]["passed"] and want[2]["failed"]
    assert tm["pass1_ms"] > 0 and tm["pass2_ms"] > 0


def test_several_calls_and_runs(mods, world):
    F, _ = mods
    contigs, ref, genome = world
    hdr = S.header(contigs)
    rf = F.RecordFilter(track_rejects=True, reverse_per_base_tags=True, device_bytes=300_000, **CONFIGS[0])
    try:
        for seed in range(3):   # several calls on one handle; a budget of a few hundred templates per run
            recs = S.records(200 + seed, contigs, n_templates=600)
            want = oracle(recs, hdr, CONFIGS[0], True, True, genome)
            b, off = S.pack(recs)
            kept, rej, st = rf.filter(hdr, b, off, ref)
            assert (kept, rej, st) == want
        # without rejects tracking the rejects stream is empty and the kept one unchanged
        rf2 = F.RecordFilter(track_rejects=False, reverse_per_base_tags=True, **CONFIGS[0])
        kept2, rej2, st2 = rf2.filter(hdr, b, off, ref)
        rf2.close()
        assert kept2 == want[0] and rej2 == b"" and st2 == want[2]
    finally:
        rf.close()


def test_long_reads_and_many_records(mods, world):
    F, _ = mods
    contigs = S.genome(11, n_contigs=2, length=200_000)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "long.fa")
        with open(p, "wb") as f:
            f.write(S.fasta(contigs))
        ref = F.Reference(p)
        genome = O.parse_fasta(S.fasta(contigs))
        hdr = S.header(contigs)
        recs = S.records(5, contigs, n_templates=40, long_every=8)
        assert max(len(r) for r in recs) > 3 * 65535
        for tmpl in (True, False):
            want = oracle(recs, hdr, CONFIGS[2], tmpl, True, genome)
            (got, _) = run(F, ref, hdr, recs, CONFIGS[2], tmpl, True)
            assert got == want
        # many short records: several grid waves, against the oracle on the same input
        recs = S.records(6, contigs, n_templates=12000, length=60)
        want = oracle(recs, hdr, CONFIGS[0], True, False, genome)
        (got, _) = run(F, ref, hdr, recs, CONFIGS[0], True, False, threads=6)
        assert got == want
        ref.close()


def test_staging_chunks(mods, world, monkeypatch):
    """4 KiB staging buffers: every upload (records, offsets, template tables) and both downloads cross many chunks,
    so the alternating buffers and their events are reused."""
    F, _ = mods
    contigs, ref, genome = world
    hdr = S.header(contigs)
    monkeypatch.setenv("FGB_FILTER_STAGE_BYTES", "4096")
    recs = S.records(31, contigs, n_templates=500)
    want = oracle(recs, hdr, CONFIGS[0], True, True, genome)
    assert sum(map(len, recs)) > 50 * 4096 and len(want[0]) > 10 * 4096 and len(want[1]) > 10 * 4096
    for threads in (1, 6):
        (got, _) = run(F, ref, hdr, recs, CONFIGS[0], True, True, threads)
        assert got == want


@pytest.mark.parametrize("case", __import__("tests.test_filter_oracle_kat", fromlist=["CASES"]).CASES,
                         ids=lambda c: c[0])
def test_alignment_tag_known_answers(mods, case, tmp_path):
    """The reference's alignment_tags.rs cases through the device: NM / UQ / MD as the reference's tests expect."""
    F, _ = mods
    _, seq, quals, cigar, nm, uq, md = case
    path = tmp_path / "chr1.fa"
    path.write_bytes(b">chr1\nACGTACGTACGTACGT\n")
    ref = F.Reference(str(path))
    rec = bytes(make_record(name=b"q", ref_id=0, pos=0, cigar=cigar, seq=seq, quals=bytes(quals),
                            tags=[(b"cd", "Bs", [9] * len(seq))]))
    (kept, rej, st), _ = run(F, ref, b"@SQ\tSN:chr1\tLN:16\n", [rec], dict(max_no_call_fraction=1.0,
                                                                        max_base_error_rate=(1.0,)), False, False)
    ref.close()
    out = (kept or rej)[4:]
    t = O.R._aux_tags(O.R.Rec(out).aux())
    assert (t[b"NM"][1], t[b"UQ"][1], t[b"MD"][1]) == (nm, uq, md)


def test_unmapped_only_without_reference(mods, world):
    F, _ = mods
    contigs, _, _ = world
    hdr = S.header(contigs)
    recs = [r for r in S.records(9, contigs, n_templates=400) if struct.unpack_from("<H", r, 14)[0] & 0x4]
    assert len(recs) > 5
    want = oracle(recs, hdr, CONFIGS[2], False, False, None)
    (got, _) = run(F, None, hdr, recs, CONFIGS[2], False, False, use_ref=False)
    assert got == want


def _err_cases(contigs):
    hdr = S.header(contigs, extra=(b"chrMissing",))
    good = S.records(3, contigs, n_templates=20)
    mapped = lambda **kw: bytes(make_record(name=b"bad", flags=0, seq=b"ACGTACGTAC", **kw))
    n_hdr = len(contigs) + 1
    return hdr, good, [
        ("no reference", mapped(ref_id=0, pos=10), False),
        ("ref_id outside the header", mapped(ref_id=n_hdr, pos=10), True),
        ("contig missing from the FASTA", mapped(ref_id=n_hdr - 1, pos=10), True),
        ("past the contig's end", mapped(ref_id=0, pos=len(contigs[0][1]) - 5), True),
        ("negative position", mapped(ref_id=0, pos=-3), True),
        ("CIGAR longer than the read", mapped(ref_id=0, pos=10, cigar="8M4I"), True),
        ("truncated", mapped(ref_id=0, pos=10)[:-4], True),
        ("shorter than 32 bytes", b"\0" * 20, True),
        ("two primary R1s", None, True),
        ("one base past the contig's end", mapped(ref_id=0, pos=len(contigs[0][1]) - 9), True),
    ]


@pytest.mark.parametrize("later", ["truncated", "contig", "cigar"])
def test_first_of_two_errors(mods, world, later):
    """A second primary R1 (found while ordering templates) before a record cut short (found by the host's record
    checks) or a record aligned to a missing contig or with a bad CIGAR (found on the device): the duplicate is named."""
    F, _ = mods
    contigs, ref, genome = world
    hdr, good, _ = _err_cases(contigs)
    r1 = bytes(make_record(name=b"dup", flags=0x41, ref_id=0, pos=5, seq=b"ACGTACGTAC"))
    bad = {"truncated": bytes(make_record(name=b"bad", ref_id=0, pos=10, seq=b"ACGTACGTAC"))[:-4],
           "contig": bytes(make_record(name=b"bad", ref_id=len(contigs), pos=10, seq=b"ACGTACGTAC")),
           "cigar": bytes(make_record(name=b"bad", ref_id=0, pos=10, cigar="8M4I", seq=b"ACGTACGTAC"))}[later]
    recs = good[:6] + [r1, r1] + good[6:12] + [bad] + good[12:]
    rf = F.RecordFilter(track_rejects=True, **CONFIGS[0])
    try:
        b, off = S.pack(recs)
        with pytest.raises(Exception):
            rf.filter(hdr, b, off, ref)
        assert rf.bad_record == 7
        with pytest.raises(O.FilterError) as oe:
            O.filter_records(recs, hdr, O.Config(**CONFIGS[0]), genome)
        assert oe.value.record == 7
    finally:
        rf.close()


@pytest.mark.parametrize("k", range(10))
def test_errors_fail_the_call(mods, world, k):
    F, _ = mods
    contigs, ref, genome = world
    hdr, good, cases = _err_cases(contigs)
    what, bad, use_ref = cases[k]
    if not use_ref:   # every record before the bad one is unmapped, so the missing reference is first met there
        good = [r for r in S.records(4, contigs, n_templates=600) if struct.unpack_from("<H", r, 14)[0] & 0x4]
        assert len(good) > 10
    if bad is None:   # a second primary R1 in one template
        r1 = bytes(make_record(name=b"dup", flags=0x41, ref_id=0, pos=5, seq=b"ACGTACGTAC"))
        recs = good[:10] + [r1, r1] + good[10:]
        at = 11
    else:
        recs = good[:10] + [bad] + good[10:] + [bad]
        at = 10
    rf = F.RecordFilter(track_rejects=True, **CONFIGS[0])
    try:
        b, off = S.pack(recs)
        with pytest.raises(Exception) as ei:
            rf.filter(hdr, b, off, ref if use_ref else None)
        assert rf.bad_record == at, (what, str(ei.value))
        with pytest.raises(O.FilterError) as oe:
            O.filter_records(recs, hdr, O.Config(**CONFIGS[0]), genome if use_ref else None)
        assert oe.value.record == at
        # the next call on the handle is unaffected
        b, off = S.pack(good)
        assert rf.filter(hdr, b, off, ref) == O.filter_records(good, hdr, O.Config(**CONFIGS[0]), genome)
        assert rf.bad_record is None
    finally:
        rf.close()


@pytest.mark.parametrize("batch_records", [1_000_000, 37])
def test_filter_file(mods, world, tmp_path, batch_records):
    F, bamio = mods
    contigs, ref, genome = world
    hdr = S.header(contigs)
    recs = S.records(21, contigs, n_templates=300)
    import fgumi_b200.lib as L
    lib = L.load()
    payload = bamio.mapped_bam_header(hdr) + b"".join(struct.pack("<I", len(r)) + r for r in recs)
    cap = lib.fgb_bgzf_bound(len(payload))
    comp = np.empty(cap, np.uint8)
    import ctypes as C
    cn = C.c_size_t()
    assert lib.fgb_bgzf_compress(payload, len(payload), 1, 1, 1, comp.ctypes.data, cap, C.addressof(cn)) == 0
    inp = tmp_path / "in.bam"
    comp[:cn.value].tofile(str(inp))
    rf = F.RecordFilter(track_rejects=True, **CONFIGS[0])
    bamio.filter_file(str(inp), str(tmp_path / "out.bam"), rf, ref, rejects=str(tmp_path / "rej.bam"),
                      stats=str(tmp_path / "stats.txt"), batch_records=batch_records)
    rf.close()
    want = oracle(recs, hdr, CONFIGS[0], True, False, genome)
    for path, stream in (("out.bam", want[0]), ("rej.bam", want[1])):
        text, bodies, off, _ = bamio.read_bam(str(tmp_path / path))
        assert text.count(b"@PG") == 1 and b"fgumi_b200 filter" in text
        got = b"".join(struct.pack("<I", int(off[i + 1] - off[i])) + bodies[int(off[i]):int(off[i + 1])].tobytes()
                       for i in range(len(off) - 1))
        assert got == stream
    st = want[2]
    assert (tmp_path / "stats.txt").read_text() == (
        f"total_reads\t{st['total']}\npassed_reads\t{st['passed']}\nfailed_reads\t{st['failed']}\n"
        f"pass_rate\t{st['passed'] / st['total']:.4f}\n")
