"""`fgumi filter --ref` on the device (fgb_filter_records) against tests/filter_oracle.py at the shapes its warp-per-record
walk meets in real inputs, the kept stream, the rejects stream and the counters byte for byte:

- the reference's tag lookup (a repeated tag read from its first entry, aD / bD found by name before their value is
  sized) on the hand-built records of tests/test_filter_shapes.py;
- the MD walk on that file's deterministic records, whose NM / UQ / MD are pinned there as literals;
- NM / UQ / MD edits for every existing integer type, MD as Z and H at the regenerated and another length, each tag
  at the start, middle or end of the aux data or repeated, records without aux data, unmapped records with every
  subset of the three, and regenerated values on the boundaries of append_int_tag's types;
- masking with every B element type of per-base tags shorter than, as long as and longer than the read, ac / bc as
  Z and B:C, and tag reversal of arrays of 1-, 2- and 4-byte elements and strings of many lengths;
- a 4.3 GB reference built in memory, with test contigs straddling genome offsets 2^31 and 2^32 and one past 2^32;
- outputs far larger than their inputs with one template per run, a 64-record template and a template larger than
  the device budget by itself."""
import ctypes as C
import os
import random
import resource
import struct
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import filter_oracle as O          # noqa: E402
from tests import filter_streams as S         # noqa: E402
from tests import test_filter_shapes as T     # noqa: E402
from tests.bam_builder import make_record     # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import filter as F
    return F


@pytest.fixture(scope="module")
def ref(F, tmp_path_factory):
    path = tmp_path_factory.mktemp("ref") / "shapes.fa"
    path.write_bytes(S.fasta(T.CONTIGS, width=80))
    r = F.Reference(str(path))
    yield r
    r.close()


def product_kw(cfg_kw):
    kw = dict(cfg_kw)
    if "require_ss_agreement" in kw:
        kw["require_single_strand_agreement"] = kw.pop("require_ss_agreement")
    return kw


def run(F, ref, hdr, recs, cfg_kw, tmpl=False, rev=False, device_bytes=0):
    rf = F.RecordFilter(filter_by_template=tmpl, reverse_per_base_tags=rev, track_rejects=True,
                        device_bytes=device_bytes, **product_kw(cfg_kw))
    try:
        b, off = S.pack(recs)
        return rf.filter(hdr, b, off, ref)
    finally:
        rf.close()


def check(F, ref, recs, cfg_kw, tmpl=False, rev=False, hdr=T.HEADER, genome=T.GENOME, device_bytes=0, names=None):
    """The device against the oracle; a differing record is named by its case."""
    want = O.filter_records(recs, hdr, O.Config(filter_by_template=tmpl, reverse_per_base_tags=rev, **cfg_kw), genome)
    got = run(F, ref, hdr, recs, cfg_kw, tmpl, rev, device_bytes)
    if got != want and names is not None:
        split = lambda s: [s[p + 4:p + 4 + struct.unpack_from("<I", s, p)[0]] for p in _starts(s)]
        for g, w in zip(split(got[0]) + split(got[1]), split(want[0]) + split(want[1])):
            assert g == w, names.get(O.R.Rec(bytes(w)).name, O.R.Rec(bytes(w)).name)
    assert got == want
    return want


def _starts(s):
    p, out = 0, []
    while p < len(s):
        out.append(p)
        p += 4 + struct.unpack_from("<I", s, p)[0]
    return out


# ---- the reference's tag lookup -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mapped", [False, True])
def test_lookup_rule_cases(F, ref, mapped):
    recs = [T.lookup_record(c, *((0, 0, 0) if mapped else ())) for c in T.LOOKUP_CASES]
    want = check(F, ref, recs, T.LOOKUP_CFG, names={b"k_" + c[0].encode(): c[0] for c in T.LOOKUP_CASES})
    assert want[2]["bases_masked"] == sum(c[3] for c in T.LOOKUP_CASES)
    assert want[2]["passed"] == sum(c[4] for c in T.LOOKUP_CASES)


# ---- the MD walk ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rev", [False, True])
def test_md_walk_cases(F, ref, rev):
    recs = T.md_records()
    if rev:   # the same records on the reverse strand with per-base tags to reverse
        recs = [make_record(name=b"r%03d" % k, flags=0x10, ref_id=c[1], pos=c[2], cigar=c[3],
                            seq=bytes(O.R.Rec(r).sequence()), tags=[(b"cd", "BS", [i % 100 for i in range(O.R.Rec(r).l_seq)])])
                for k, (c, r) in enumerate(zip(T.MD_CASES, recs))]
    names = {b"%s%03d" % (b"r" if rev else b"md", k): c[0] for k, c in enumerate(T.MD_CASES)}
    want = check(F, ref, recs, T.OPEN, rev=rev, names=names)
    assert want[2]["passed"] == len(recs)


@pytest.mark.parametrize("c", [0, 2])
def test_read_ending_on_the_contig_end(F, ref, c):
    """A read ending on the last base of an inner contig and of the last contig passes; one base longer fails the
    call on that record."""
    ctg = T.CONTIGS[c][1]
    ok = make_record(name=b"end", ref_id=c, pos=len(ctg) - 20, cigar="20M", seq=ctg[-20:].upper())
    check(F, ref, [ok], T.OPEN)
    bad = make_record(name=b"past", ref_id=c, pos=len(ctg) - 20, cigar="21M", seq=ctg[-20:].upper() + b"A")
    rf = F.RecordFilter(track_rejects=True, filter_by_template=False, **T.OPEN)
    try:
        b, off = S.pack([ok, bad])
        with pytest.raises(Exception, match="past the end"):
            rf.filter(T.HEADER, b, off, ref)
        assert rf.bad_record == 1
    finally:
        rf.close()


# ---- tag edits ------------------------------------------------------------------------------------------------------
INT_TYPES = ["c", "C", "s", "S", "i", "I"]
FILLER = [(b"RG", "Z", b"grp1"), (b"XA", "i", 7)]


def _base(name, tags, cigar="20M", mis=(4,), flags=0, pos=3, quals=None):
    return make_record(name=name, flags=flags, ref_id=0, pos=pos, cigar=cigar, quals=quals,
                       seq=T.along(T.CHR_A, pos, cigar, mis), tags=tags)


def _regenerated_md(cigar="20M", mis=(4,), pos=3):
    r = bytearray(_base(b"x", [], cigar, mis, pos=pos))
    O.regenerate(r, 0, T.SQ, T.GENOME)
    return O.R._aux_tags(O.R.Rec(bytes(r)).aux())[b"MD"][1]


def _placed(entry, where):
    return {"start": [entry] + FILLER, "middle": FILLER[:1] + [entry] + FILLER[1:], "end": FILLER + [entry]}[where]


def tag_edit_records():
    md = _regenerated_md()
    out, names = [], {}

    def add(label, **kw):
        name = b"t%04d" % len(out)
        names[name] = label
        out.append(_base(name, **kw))

    for where in ("start", "middle", "end"):
        for tag in (b"NM", b"UQ"):
            for ty in INT_TYPES:
                add("%s:%s at %s" % (tag.decode(), ty, where), tags=_placed((tag, ty, 100), where))
        for ty, v in (("Z", md), ("Z", md + b"0"), ("H", b"F" * len(md)), ("H", b"F" * (len(md) - 1)), ("Z", b"")):
            add("MD:%s len %d at %s" % (ty, len(v), where), tags=_placed((b"MD", ty, v), where))
    add("none", tags=FILLER)
    add("no aux data", tags=[])
    rng = random.Random(5)
    for k in range(40):   # all three, in random order and types, among other tags
        tags = [(b"NM", rng.choice(INT_TYPES), rng.randint(0, 100)), (b"UQ", rng.choice(INT_TYPES), rng.randint(0, 100)),
                (b"MD", rng.choice("ZH"), rng.choice([md, b"1", b"F" * len(md)]))] + FILLER
        rng.shuffle(tags)
        add("mixed %d" % k, tags=tags)
    for tag, a, b in ((b"NM", ("i", 3), ("C", 4)), (b"NM", ("C", 3), ("i", 4)), (b"UQ", ("i", 3), ("i", 4)),
                      (b"UQ", ("S", 3), ("c", 4)), (b"MD", ("Z", md), ("Z", b"9")), (b"MD", ("Z", b"9"), ("Z", md))):
        add("%s twice %s %s" % (tag.decode(), a[0], b[0]), tags=[(tag, *a)] + FILLER[:1] + [(tag, *b)])
    # unmapped records with each subset of the three tags
    for mask in range(8):
        tags = [t for k, t in enumerate([(b"NM", "C", 3), (b"UQ", "i", 40), (b"MD", "Z", b"20")]) if mask >> k & 1]
        for where in ("start", "end"):
            tg = tags + FILLER if where == "start" else FILLER + tags
            name = b"t%04d" % len(out)
            names[name] = "unmapped %d %s" % (mask, where)
            out.append(make_record(name=name, flags=0x4, ref_id=-1, pos=-1, cigar="", seq=b"ACGTACGTAC", tags=tg))
    return out, names


def test_tag_edits(F, ref):
    recs, names = tag_edit_records()
    check(F, ref, recs, T.OPEN, names=names)


def boundary_records():
    """Regenerated NM and UQ on both sides of append_int_tag's c / C / S / i boundaries, with the tags absent and
    present as C and i."""
    out, names = [], {}
    cases = []
    for v in (127, 128, 255, 256, 65535, 65536):
        cases.append(("NM %d" % v, dict(cigar="10M%dD10M" % v, mis=())))
    for v in (127, 128, 255, 256, 65535, 65536):
        q = [255] * (v // 255) + ([v % 255] if v % 255 else [])
        n = len(q)
        quals = bytes(q) + bytes([30] * 10)
        cases.append(("UQ %d" % v, dict(cigar="%dM" % (n + 10), mis=tuple(range(n)), quals=quals)))
    cases.append(("65535 0xFF mismatches", dict(cigar="65535M", mis=tuple(range(65535)), quals=b"\xff" * 65535)))
    for label, kw in cases:
        for existing in ([], [(b"NM", "C", 1), (b"UQ", "C", 1)], [(b"NM", "i", 1), (b"UQ", "i", 1)]):
            name = b"b%04d" % len(out)
            names[name] = "%s with %s" % (label, [e[1] for e in existing])
            out.append(_base(name, tags=existing + FILLER, **kw))
    return out, names


def test_regenerated_values_on_type_boundaries(F, ref):
    recs, names = boundary_records()
    want = check(F, ref, recs, T.OPEN, names=names)
    types = set()
    for p in _starts(want[0]):
        t = O.R._aux_tags(O.R.Rec(want[0][p + 4:p + 4 + struct.unpack_from("<I", want[0], p)[0]]).aux())
        types |= {t[b"NM"][0], t[b"UQ"][0]}
    assert {"c", "C", "S", "i"} <= types


# ---- masking and reversal -----------------------------------------------------------------------------------------
B_TYPES = ["Bc", "BC", "Bs", "BS", "Bi", "BI", "Bf"]


def _vals(rng, ty, n, hi):
    if ty == "Bf":
        return [rng.random() * hi for _ in range(n)]
    lo = -3 if ty in ("Bc", "Bs", "Bi") else 0
    return [rng.randint(lo, hi) for _ in range(n)]


def masking_records(seed=3, L=40):
    rng = random.Random(seed)
    out, names = [], {}
    strs = [b"ACGTacgtRYN", b"ACGTN"]

    def add(label, flags, tags):
        name = b"m%04d" % len(out)
        names[name] = label
        seq = bytearray(T.along(T.CHR_A, 3, "%dM" % L, (rng.randrange(L),)))
        seq[rng.randrange(L)] = ord("N")
        out.append(make_record(name=name, flags=flags, ref_id=0, pos=3, cigar="%dM" % L, seq=bytes(seq),
                               quals=bytes(rng.randint(2, 40) for _ in range(L)), tags=tags))

    for ty in B_TYPES:
        for n in (L - 7, L, L + 9):
            for flags in (0, 0x10):
                add("simplex %s %d" % (ty, n), flags, [(b"cd", ty, _vals(rng, ty, n, 6)), (b"ce", ty, _vals(rng, ty, n, 2)),
                                                      (b"cD", "C", 6)])
                tags = [(b"aD", "C", 5), (b"bD", "C", 4)]
                for t in (b"ad", b"bd", b"ae", b"be"):
                    tt = rng.choice([ty, "Bs"]) if t[1:] == b"e" else ty
                    tags.append((t, tt, _vals(rng, tt, n, 5 if t[1:] == b"d" else 1)))
                for t in (b"ac", b"bc"):
                    s = bytes(rng.choice(rng.choice(strs)) for _ in range(rng.choice((L - 5, L, L + 5))))
                    tags.append((t, "Z", s) if rng.random() < 0.5 else (t, "BC", list(s)))
                rng.shuffle(tags)
                add("duplex %s %d" % (ty, n), flags, tags)
    return out, names


@pytest.mark.parametrize("ss", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_masking_shapes(F, ref, ss, rev):
    recs, names = masking_records()
    cfg = dict(min_reads=(2, 1, 0), max_read_error_rate=(0.5,), max_base_error_rate=(0.3,), min_base_quality=5,
               max_no_call_fraction=0.9, require_ss_agreement=ss)
    want = check(F, ref, recs, cfg, rev=rev, names=names)
    assert want[2]["passed"] and want[2]["failed"] and want[2]["bases_masked"]


def reversal_records(L=50):
    rng = random.Random(9)
    out, names = [], {}
    for ty in B_TYPES:
        for n in (0, 1, 2, 31, 32, 33, 64, 65, 200):
            name = b"v%04d" % len(out)
            names[name] = "%s x %d" % (ty, n)
            zs = bytes(rng.choice(b"ACGTacgtRYNn") for _ in range(n))
            tags = [(b"cd", ty, _vals(rng, ty, n, 9)), (b"bd", ty, _vals(rng, ty, n, 9)), (b"aq", "Z", zs[:n]),
                    (b"ac", "Z", zs), (b"bc", "Z", zs[::-1]), (b"bq", "BC", list(zs))]
            out.append(make_record(name=name, flags=0x10, ref_id=0, pos=3, cigar="%dM" % L,
                                   seq=T.along(T.CHR_A, 3, "%dM" % L), tags=tags))
    return out, names


def test_tag_reversal_shapes(F, ref):
    recs, names = reversal_records()
    cfg = dict(T.OPEN, min_reads=(1,))
    check(F, ref, recs, cfg, rev=True, names=names)


# ---- a human-size reference ---------------------------------------------------------------------------------------
TWO31, TWO32 = 1 << 31, 1 << 32


def _free_device_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def test_reference_past_4_gib(F):
    """A 4.3 GB reference image built in memory: contig t31 straddles genome offset 2^31, t32 straddles 2^32 and
    t32b lies wholly past it; reads at both ends of each and across both boundaries."""
    total = TWO32 + 4000
    need = total + (2 << 30)
    free = _free_device_bytes()
    if free < need:
        pytest.skip("the device has %d bytes free; this test needs %d" % (free, need))
    t0 = time.perf_counter()
    rng = random.Random(41)
    tests = {n: bytes(rng.choice(b"ACGTacgt") for _ in range(ln)) for n, ln in ((b"t31", 1200), (b"t32", 1200),
                                                                               (b"t32b", 1000))}
    layout = [(b"fill1", TWO31 - 600), (b"t31", 1200), (b"fill2", TWO32 - 600 - (TWO31 + 600)), (b"t32", 1200),
              (b"t32b", 1000), (b"tail", 100)]
    size = sum(len(n) + 2 + ln + 1 for n, ln in layout)
    img = np.empty(size, np.uint8)
    p, g = 0, 0
    starts = {}
    for name, ln in layout:
        head = b">" + name + b"\n"
        img[p:p + len(head)] = np.frombuffer(head, np.uint8)
        p += len(head)
        body = tests.get(name)
        if body is not None:
            img[p:p + ln] = np.frombuffer(body, np.uint8)
        else:
            img[p:p + ln] = ord("N") if name != b"tail" else ord("A")
        starts[name] = g
        p += ln
        g += ln
        img[p] = ord("\n")
        p += 1
    assert p == size and starts[b"t31"] < TWO31 < starts[b"t31"] + 1200
    assert starts[b"t32"] < TWO32 < starts[b"t32"] + 1200 and starts[b"t32b"] > TWO32
    lib = F._l.load()
    h = C.c_void_p()
    free0 = _free_device_bytes()
    st = lib.fgb_reference_create(0, img.ctypes.data, size, C.byref(h))
    del img
    assert st == 0
    ref_dev = free0 - _free_device_bytes()
    ref = F.Reference.__new__(F.Reference)
    ref._lib, ref._h, ref.device = lib, h, 0
    try:
        assert ref.contigs() == [(n.decode(), ln) for n, ln in layout]
        hdr = b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n, ln) for n, ln in layout)
        sq = [n for n, _ in layout]
        recs = []
        for name, body in tests.items():
            c = sq.index(name)
            cross = {b"t31": TWO31, b"t32": TWO32}.get(name, starts[name] + 500) - starts[name]
            for cigar, span in (("60M", 60), ("20M2D20M1I19M", 61)):
                for pos in (0, len(body) - span, cross - 30, cross - 1, cross - span + 1):
                    seq = bytearray(T.along(body, pos, cigar))
                    for k in rng.sample(range(len(seq)), 3):
                        seq[k] = rng.choice(b"ACGT")
                    recs.append(make_record(name=b"g%03d" % len(recs), ref_id=c, pos=pos, cigar=cigar, seq=bytes(seq),
                                            tags=[(b"MD", "Z", b"60"), (b"NM", "C", 0)]))
        want = O.filter_records(recs, hdr, O.Config(filter_by_template=False, **T.OPEN), tests)
        got = run(F, ref, hdr, recs, T.OPEN)
        assert got == want
        assert want[2]["passed"] == len(recs)
    finally:
        ref.close()
    print("\n4.3 GB reference: peak host RSS %.2f GB, reference on the device %.2f GB, %.1f s" % (
        resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6, ref_dev / 1e9, time.perf_counter() - t0))


# ---- large outputs and large templates ----------------------------------------------------------------------------
def test_outputs_far_past_the_run_budget(F, ref):
    """100 000-base deletions: each record's MD is ~1000 times its input, and with one template per run the kept and
    rejects buffers grow run after run."""
    recs = []
    for k in range(24):
        for r1 in (True, False):
            recs.append(make_record(name=b"d%03d" % k, flags=0x41 if r1 else 0x81, ref_id=0, pos=7 + k,
                                    cigar="10M100000D10M", seq=T.along(T.CHR_A, 7 + k, "10M100000D10M", (k % 20,)),
                                    tags=[(b"cd", "Bs", [5] * 20), (b"cD", "C", 0 if k % 3 == 0 else 5)]))
    cfg = dict(T.OPEN, min_reads=(1,))
    want = check(F, ref, recs, cfg, tmpl=True, device_bytes=1)
    assert len(want[0]) > 30 * 100_000 and len(want[1]) > 10 * 100_000


def test_large_templates(F, ref):
    rng = random.Random(12)

    def rec(name, flags, L=150):
        pos = rng.randrange(0, len(T.CHR_A) - L - 10)
        cigar = rng.choice(["%dM" % L, "%dM3D%dM" % (L // 2, L - L // 2), "%dM2I%dM" % (L // 2, L - L // 2 - 2)])
        seq = T.along(T.CHR_A, pos, cigar, tuple(rng.sample(range(L), 2)))
        cd = [rng.randint(0, 6) for _ in range(L)]
        return make_record(name=name, flags=flags | (0x10 if rng.random() < 0.5 else 0), ref_id=0, pos=pos,
                           cigar=cigar, seq=seq, tags=[(b"cd", "Bs", cd), (b"cD", "C", max(cd))])

    big = [rec(b"big", 0x41), rec(b"big", 0x81)]
    big += [rec(b"big", rng.choice([0x100 | 0x41, 0x100 | 0x81, 0x800 | 0x41, 0x800 | 0x81])) for _ in range(62)]
    small = lambda k: [rec(b"s%03d" % k, 0x41), rec(b"s%03d" % k, 0x81)]
    recs = small(0) + small(1) + big + small(2)
    huge = [rec(b"huge", 0x41, 20000), rec(b"huge", 0x81, 20000)]
    cfg = dict(min_reads=(1,), max_base_error_rate=(0.3,), max_read_error_rate=(1.0,), max_no_call_fraction=0.5)
    for device_bytes in (0, 4096):   # 4096: the 64-record template runs alone
        check(F, ref, recs, cfg, tmpl=True, rev=True, device_bytes=device_bytes)
    # a template larger than the budget by itself, between two small ones
    check(F, ref, small(3) + huge + small(4), cfg, tmpl=True, device_bytes=30000)
