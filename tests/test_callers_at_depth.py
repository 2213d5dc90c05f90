"""The record-level callers (fgb_caller_*) on deep families and long reads, against the Python record oracle.

The other caller tests use families of at most 8 reads of 40-150 bases.  Real libraries have families of tens to
thousands of reads of 150-301 bases, and the callers change form at thresholds those small families never reach:
- device record assembly (K5) writes cD / cM as 'c' up to 127 and 'C' from 128 to 255;
- a unit deeper than 255 reads sends the whole simplex batch to host assembly from 16-bit columns ('S' tags);
- the filter epilogue (K4) masks a base only when errors / depth is strictly above the rate; its per-depth table is
  exercised here at depths 10, 20 and 130 with e / d equal to the rate;
- the filter's statuses are written per submit chunk;
- duplex molecules with more than 255 pooled source reads leave the fused epilogue for the scalar recount;
- the row builder and the overlap pre-pass see rows longer than 256 bases, odd lengths and deep overlapping pairs.
Every test compares every output byte, the record count and the caller statistics with the oracle, and asserts
that the path it is meant to cover was taken."""
import os
import re
import struct
import sys
from functools import lru_cache

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import record_oracle as R          # noqa: E402
from tests import oracle_lib as O              # noqa: E402
from tests.bam_builder import make_record, parse_records   # noqa: E402
from tests.test_record_oracle_kat import vote_fn   # noqa: E402

P, F1, F2, REV, MREV = R.PAIRED, R.FIRST_SEGMENT, R.LAST_SEGMENT, R.REVERSE, R.MATE_REVERSE
ACGT = np.frombuffer(b"ACGT", np.uint8)
IUPAC = np.frombuffer(b"RYKMSWBDHV", np.uint8)
COMP = bytes.maketrans(b"ACGTNRYKMSWBDHV", b"TGCANYRMKSWVHDB")

# Family depths (reads per unit: per read type for paired families).  They straddle every threshold: the 'c' / 'C'
# boundary of cD / cM (127 / 128), the one-byte limit (255 / 256), and the deep-kernel classes of the vote (24 / 25).
LADDER_NARROW = (1, 2, 4, 5, 23, 24, 25, 64, 127, 128, 129, 255)
LADDER_DEEP = (256, 300, 513, 1500)
LENS = (150, 151, 250, 301)
TIE_DEPTHS = (10, 20, 130)             # e / d == 0.1 == max_base_error_rate at the tie columns
TIE_COLS = (10, 11, 12, 13, 14)        # read-orientation columns every read covers, trimmed or clipped
TIE_RATE = 0.1
PAD = 320                              # template bases on either side of the insert (reads run past short inserts)
LONG_UMI = b"U" * 248                  # "fgumi:" + UMI = 254 bytes, the longest read name a record may have


# ------------------------------------------------------------------------------------------------------------------
# workload
# ------------------------------------------------------------------------------------------------------------------
def _revcomp(s: bytes) -> bytes:
    return s.translate(COMP)[::-1]


def _read(rng, ref_seq: bytes, rev: bool, dissent=None, error_rate=0.01, tail=True):
    """One read's stored (reference-orientation) SEQ and QUAL from its true reference-orientation bases.  Noise is
    applied in read orientation: ~1 % substitutions, now and then an N or an IUPAC code, and a low-quality tail that
    `trim` cuts and `min_input_base_quality` masks.  `dissent` = read-orientation columns that get a confident
    wrong base; the tie columns are otherwise kept clean and confident."""
    ro = np.frombuffer(_revcomp(ref_seq) if rev else ref_seq, np.uint8).copy()
    n = len(ro)
    q = rng.integers(18, 41, size=n)
    m = rng.random(n) < error_rate
    ro[m] = ACGT[rng.integers(0, 4, size=int(m.sum()))]
    if rng.random() < 0.15:
        ro[rng.integers(20, n)] = ord("N")
    if rng.random() < 0.05:
        ro[rng.integers(20, n)] = IUPAC[rng.integers(0, len(IUPAC))]
    if tail and rng.random() < 0.3:
        k = int(rng.integers(1, 60))
        q[n - k:] = rng.integers(2, 9, size=k)
    clean = np.frombuffer(_revcomp(ref_seq) if rev else ref_seq, np.uint8)
    for c in TIE_COLS:
        ro[c] = clean[c]
        q[c] = 35
    for c in dissent or ():
        ro[c] = ACGT[(int(np.flatnonzero(ACGT == clean[c])[0]) + 1) % 4]
    q = q.astype(np.uint8)
    if rev:
        return _revcomp(ro.tobytes()), q[::-1].tobytes()
    return ro.tobytes(), q.tobytes()


def _tags(rng, umi, rx):
    t = [(b"MI", "Z", umi)]
    if rng.random() < 0.9:
        r = bytearray(rx)
        if rng.random() < 0.15:                                  # a UMI read with an error: the RX consensus votes
            i = int(rng.integers(0, len(r)))
            if r[i] != ord("-"):
                r[i] = ACGT[rng.integers(0, 4)]
        t.append((b"RX", "Z", bytes(r)))
    if rng.random() < 0.4:
        t.append((b"CB", "Z", b"CELL%d" % int(rng.integers(0, 3))))
    return t


def _cig(l, clip, rev):
    """All-M, or a 5-base soft clip at the read's 5' end (the start of a forward read, the end of a reverse one)."""
    if not clip:
        return "%dM" % l, 0
    return ("%dM5S" % (l - 5), 0) if rev else ("5S%dM" % (l - 5), 5)


def _pair(rng, name, tmpl, insert, l1, l2, r1_rev, clip, tags, d1=None, d2=None):
    """An FR pair of one molecule: the forward mate starts at template 0, the reverse one ends at `insert`.  Inserts
    shorter than a read make the reads run past their mates (the mate-overlap clip); inserts shorter than l1 + l2
    make them overlap (the overlapping-bases pre-pass).  r1_rev puts R1 on the reverse strand."""
    lf, lr = (l2, l1) if r1_rev else (l1, l2)
    sf, qf = _read(rng, tmpl[PAD:PAD + lf], False, d2 if r1_rev else d1)
    sr, qr = _read(rng, tmpl[PAD + insert - lr:PAD + insert], True, d1 if r1_rev else d2)
    cf, of = _cig(lf, clip, False)
    cr, _ = _cig(lr, clip, True)
    pf, pr = 1000 + of, 1000 + insert - lr
    ef, er = pf + lf - of, pr + lr - (5 if clip else 0)
    tl = max(ef, er) - min(pf, pr)
    tf, tr = (tl, -tl) if pf <= pr else (-tl, tl)
    fwd = make_record(name=name, flags=P | MREV | (F2 if r1_rev else F1), pos=pf, mate_ref_id=0,
                      mate_pos=pr, tlen=tf, seq=sf, quals=qf, cigar=cf, tags=tags + [(b"MC", "Z", cr.encode())])
    rev = make_record(name=name, flags=P | REV | (F1 if r1_rev else F2), pos=pr, mate_ref_id=0,
                      mate_pos=pf, tlen=tr, seq=sr, quals=qr, cigar=cr, tags=tags + [(b"MC", "Z", cf.encode())])
    return [rev, fwd] if r1_rev else [fwd, rev]


def simplex_family(rng, g, depth, kind="pair", tie=False, umi=None):
    """One MI group: `depth` fragments, or `depth` pairs (so R1 and R2 units each have `depth` reads).  Read lengths
    are mixed within the family; strand, soft clip and insert size are per family.  tie=True: at TIE_COLS exactly
    depth / 10 reads of each unit carry a confident wrong base, so errors / depth == 0.1 there."""
    tmpl = ACGT[rng.integers(0, 4, size=2 * PAD + 700)].tobytes()
    umi = umi if umi is not None else b"%d" % g
    rx_len = int(rng.integers(5, 9))
    rx = ACGT[rng.integers(0, 4, size=rx_len)].tobytes() + b"-" + ACGT[rng.integers(0, 4, size=rx_len)].tobytes()
    insert = int(rng.choice([120, 160, 240, 330, 480, 640]))
    r1_rev = rng.random() < 0.4
    clip = rng.random() < 0.25
    k = depth // 10 if tie else 0
    recs = []
    for d in range(depth):
        lens = LENS[int(rng.integers(0, 4))], LENS[int(rng.integers(0, 4))]
        dis = TIE_COLS if d < k else None
        tags = _tags(rng, umi, rx)
        name = b"g%d_%d" % (g, d)
        if kind == "frag":
            l = lens[0]
            s, q = _read(rng, tmpl[PAD:PAD + l] if not r1_rev else tmpl[PAD + insert - l:PAD + insert], r1_rev, dis)
            c, o = _cig(l, clip, r1_rev)
            pos = 1000 + o if not r1_rev else 1000 + insert - l
            recs.append(make_record(name=name, flags=REV if r1_rev else 0, pos=pos, seq=s, quals=q, cigar=c, tags=tags))
        else:
            recs += _pair(rng, name, tmpl, insert, lens[0], lens[1], r1_rev, clip, tags, dis, dis)
    return recs


def simplex_workload(seed, ladder, copies=1, ties=True, frag_depths=(1, 5, 24, 128, 255)):
    rng = np.random.default_rng(seed)
    groups, g = [], 0
    for c in range(copies):
        for depth in ladder:
            umi = LONG_UMI[:-1] + b"%d" % c if depth == 64 and c < 2 else None
            groups.append(simplex_family(rng, g, depth, "pair", umi=umi)); g += 1
            if depth in frag_depths:
                groups.append(simplex_family(rng, g, depth, "frag")); g += 1
    if ties:
        for depth in TIE_DEPTHS:
            groups.append(simplex_family(rng, g, depth, "pair", tie=True)); g += 1
    order = rng.permutation(len(groups))                  # deep families between shallow ones
    return [groups[i] for i in order]


def duplex_molecule(rng, g, n_ab, n_ba):
    """One duplex molecule: n_ab pairs of the A strand (R1 forward) and n_ba of the B strand (R1 reverse), so the
    AB-R1 / BA-R2 pool holds n_ab + n_ba reads."""
    tmpl = ACGT[rng.integers(0, 4, size=2 * PAD + 700)].tobytes()
    insert = int(rng.choice([200, 330, 480, 640]))
    recs = []
    for strand, n in (("A", n_ab), ("B", n_ba)):
        rx = b"AACGT-GGTCA" if strand == "A" else b"GGTCA-AACGT"
        for d in range(n):
            tags = [(b"MI", "Z", b"%d/%s" % (g, strand.encode())), (b"RX", "Z", rx)]
            if rng.random() < 0.3:
                tags.append((b"CB", "Z", b"CELL"))
            lens = LENS[int(rng.integers(0, 4))], LENS[int(rng.integers(0, 4))]
            recs += _pair(rng, b"m%d%s%d" % (g, strand.encode(), d), tmpl, insert, lens[0], lens[1], strand == "B",
                          False, tags)
    return recs


# (AB pairs, BA pairs): strand depths across 127 / 128 and 255 / 256, pooled AB + BA reads across 255
DUPLEX_LADDER = ((1, 0), (1, 1), (2, 1), (5, 4), (24, 2), (3, 25), (64, 64), (127, 129), (128, 127), (200, 60),
                 (255, 1), (256, 0), (300, 300), (40, 260), (6, 6))


def duplex_workload(seed):
    rng = np.random.default_rng(seed)
    groups = [duplex_molecule(rng, g, a, b) for g, (a, b) in enumerate(DUPLEX_LADDER)]
    order = rng.permutation(len(groups))
    return [groups[i] for i in order]


CODEC_LADDER = (1, 2, 5, 24, 25, 64, 128, 255, 256, 300)


def codec_workload(seed):
    """CODEC molecules: `n` overlapping pairs, R1 one strand and R2 the other, 250-301 bp reads (150 bp now and then),
    inserts from fully overlapped to a 50-base overlap.  Every R2 of some molecules carries the same changes at 3 or 30
    read positions, so the two strand consensuses disagree there (the disagreement gates)."""
    rng = np.random.default_rng(seed)
    groups = []
    for g, n in enumerate(CODEC_LADDER):
        tmpl = ACGT[rng.integers(0, 4, size=2 * PAD + 700)].tobytes()
        insert = int(rng.choice([240, 301, 420, 500]))
        r1_rev = rng.random() < 0.4
        strand_diff = sorted(rng.choice(np.arange(20, 140), size=(0, 3, 30)[g % 3], replace=False).tolist())
        recs = []
        for d in range(n):
            l1 = int(rng.choice([250, 251, 301, 301, 150]))
            l2 = int(rng.choice([250, 251, 301, 301, 150]))
            tags = [(b"MI", "Z", b"%d" % g), (b"RX", "Z", b"ACGTA-CCGTT")]
            if rng.random() < 0.3:
                tags.append((b"CB", "Z", b"CELL%d" % (g % 2)))
            recs += _pair(rng, b"c%d_%d" % (g, d), tmpl, insert, l1, l2, r1_rev, False, tags, d2=strand_diff)
        groups.append(recs)
    order = rng.permutation(len(groups))
    return [groups[i] for i in order]


# ------------------------------------------------------------------------------------------------------------------
# oracle side and record helpers
# ------------------------------------------------------------------------------------------------------------------
def split_stream(data: bytes):
    out, p = [], 0
    while p < len(data):
        (n,) = struct.unpack_from("<I", data, p)
        out.append(data[p + 4:p + 4 + n])
        p += 4 + n
    return out


def tag_types(data: bytes, tag: bytes):
    """The BAM type characters of an integer tag over every record of a stream."""
    return {R._aux_tags(R.Rec(r).aux())[tag][0] for r in split_stream(data) if tag in R._aux_tags(R.Rec(r).aux())}


def tie_positions(data: bytes):
    """Positions of a stream's records where errors / depth == TIE_RATE exactly, per depth (from the cd / ce arrays)."""
    seen = {}
    for rec in parse_records(data):
        for d, e in zip(rec["tags"].get(b"cd", []), rec["tags"].get(b"ce", [])):
            if d > 0 and e / d == TIE_RATE:
                seen[d] = seen.get(d, 0) + 1
    return seen


def vanilla_oracle(groups, per_base=True, overlap=False, trim=False):
    oracle = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(
        min_reads=1, min_consensus_base_quality=2, produce_per_base_tags=per_base, trim=trim,
        min_input_base_quality=10, cell_tag=b"CB"), vote_fn, O.builder_call)
    ov = R.OverlappingOracle() if overlap else None
    want, count = bytearray(), 0
    for g in groups:
        recs = g
        if ov is not None:
            recs = [bytearray(r) for r in g]
            ov.apply(recs)
            recs = [bytes(r) for r in recs]
        d, n = oracle.consensus_reads(recs)
        want += d
        count += n
    return bytes(want), count, oracle, ov


@lru_cache(maxsize=None)
def simplex_groups(kind):
    if kind == "narrow":
        return simplex_workload(11, LADDER_NARROW, copies=4)
    if kind == "plus256":
        return simplex_workload(11, LADDER_NARROW, copies=4) + [simplex_family(np.random.default_rng(13), 999, 256)]
    return simplex_workload(12, LADDER_NARROW + LADDER_DEEP)


@lru_cache(maxsize=None)
def simplex_expected(kind, per_base=True, overlap=False, trim=False):
    want, count, oracle, ov = vanilla_oracle(simplex_groups(kind), per_base, overlap, trim)
    return want, count, oracle.stats, (ov.stats() if ov is not None else None)


def assert_same_stream(got: bytes, want: bytes):
    if got != want:
        a, b = parse_records(got), parse_records(want)
        assert len(a) == len(b), (len(a), len(b))
        for i, (x, y) in enumerate(zip(a, b)):
            assert x == y, (i, {k: v for k, v in x.items() if x[k] != y.get(k)}, {k: v for k, v in y.items() if y[k] != x.get(k)})
    assert got == want


def assert_simplex_stats(gstats, s):
    assert gstats["total_reads"] == s.total_reads and gstats["consensus_reads"] == s.consensus_reads
    assert gstats["filtered_reads"] == s.filtered_reads
    for k in ("InsufficientReads", "SecondaryOrSupplementary", "ZeroLengthAfterTrimming", "MinorityAlignment",
              "OrphanConsensus"):
        assert gstats[k] == s.rejections.get(k, 0), k


def run_caller(make, groups, capfd=None):
    """Run one caller over the groups; returns (output, statistics, C-level stderr)."""
    c = make()
    c.add_groups(groups)
    out = c.flush()
    st = c.statistics()
    c.close()
    err = capfd.readouterr().err if capfd is not None else ""
    return out, st, err


def n_chunks(trace: str) -> int:
    return len(set(re.findall(r"^\s+chunk (\d+)\s", trace, re.M)))


def simplex_caller(fg, per_base=True, n_threads=1, trim=False, **kw):
    opt = fg.VanillaUmiConsensusOptions(min_reads=1, min_consensus_base_quality=2, produce_per_base_tags=per_base,
                                        trim=trim, min_input_base_quality=10)
    return fg.VanillaUmiConsensusCaller("fgumi", "A", opt, device=0, cell_tag=b"CB", n_threads=n_threads, **kw)


def cd_values(data: bytes):
    return {r["tags"][b"cD"] for r in parse_records(data)}


# ------------------------------------------------------------------------------------------------------------------
# simplex: device assembly, host assembly, filter, chunks, overlap pre-pass
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("threads,per_base,trim", [(1, True, False), (8, True, True), (1, False, True), (8, False, False)])
def test_simplex_device_assembly_at_depth(threads, per_base, trim, monkeypatch, capfd):
    """Every unit has at most 255 reads and no filter is set: records are assembled on the device (K5), with cD / cM
    typed 'c' up to 127 and 'C' from 128."""
    import fgumi_b200 as fg
    groups = simplex_groups("narrow")
    want, count, s, _ = simplex_expected("narrow", per_base, trim=trim)
    monkeypatch.setenv("FGB_CALLER_TRACE", "1")
    capfd.readouterr()
    got, st, err = run_caller(lambda: simplex_caller(fg, per_base, threads, trim), groups, capfd)
    assert "records assembled on the device" in err, err[-2000:]
    assert got.count == count
    assert_same_stream(got.data, want)
    assert_simplex_stats(st, s)
    assert tag_types(got.data, b"cD") == {"c", "C"} and tag_types(got.data, b"cM") == {"c", "C"}
    assert {1, 127, 128, 129, 255} <= cd_values(got.data)


@pytest.mark.gpu
def test_simplex_host_assembly_with_a_256_read_family(monkeypatch, capfd):
    """The same groups plus one 256-read family: the batch is assembled on the host from 16-bit columns, and the
    deep unit's cD is typed 'S' while the rest keep 'c' / 'C'."""
    import fgumi_b200 as fg
    groups = simplex_groups("plus256")
    want, count, s, _ = simplex_expected("plus256")
    monkeypatch.setenv("FGB_CALLER_TRACE", "1")
    capfd.readouterr()
    got, st, err = run_caller(lambda: simplex_caller(fg, True, 4), groups, capfd)
    assert "fgb_caller flush" in err and "records assembled on the device" not in err, err[-2000:]
    assert got.count == count
    assert_same_stream(got.data, want)
    assert_simplex_stats(st, s)
    assert tag_types(got.data, b"cD") == {"c", "C", "S"}
    assert {127, 128, 255, 256} <= cd_values(got.data)


def filtered_expected(kind, nc):
    """Oracle caller -> oracle filter, and the tie positions (errors / depth == max_base_error_rate) of the unfiltered
    stream, where a strict `>` keeps the base and `>=` would mask it."""
    unfiltered, _, _, _ = simplex_expected(kind)
    flt = R.SimplexFilterOracle(R.FilterThresholds(2, 0.05, TIE_RATE), 10, None, nc)
    data, kept = flt.filter_stream(unfiltered)
    return data, kept, flt, tie_positions(unfiltered)


def filtered_caller(fg, nc, n_threads=1):
    f = fg.ConsensusFilter(min_reads=2, max_read_error_rate=0.05, max_base_error_rate=TIE_RATE, min_base_quality=10,
                           max_no_call_fraction=nc)
    return simplex_caller(fg, True, n_threads, filter=f)


def assert_filter_stats(st, flt):
    assert st["filter_records"] == flt.total and st["filter_passed"] == flt.passed
    assert st["filter_bases_masked"] == flt.bases_masked
    assert 0 < flt.passed < flt.total


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["narrow", "deep"])
@pytest.mark.parametrize("nc", [0.3, 40.0])            # no-call limit as a fraction, and as a count (>= 1.0)
def test_simplex_filter_at_depth(kind, nc, monkeypatch, capfd):
    """The filter epilogue (K4) on units of at most 255 reads (host assembly from 8-bit columns) and on deeper units
    (16-bit columns), with e / d == max_base_error_rate at depths 10, 20 and 130."""
    import fgumi_b200 as fg
    groups = simplex_groups(kind)
    want, kept, flt, ties = filtered_expected(kind, nc)
    assert {10, 20, 130} <= set(ties)
    monkeypatch.setenv("FGB_CALLER_TRACE", "1")
    capfd.readouterr()
    got, st, err = run_caller(lambda: filtered_caller(fg, nc, 3), groups, capfd)
    assert "fgb_caller flush" in err and "records assembled on the device" not in err
    assert got.count == kept
    assert_same_stream(got.data, want)
    assert_filter_stats(st, flt)
    if kind == "deep":
        assert "S" in tag_types(got.data, b"cD")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["device", "filter"])
def test_multi_chunk_submit_at_depth(case, monkeypatch, capfd):
    """The same batch cut into 1 MB submit chunks gives the bytes of the one-chunk run and of the oracle: record
    assembly per chunk, and filter statuses written at each chunk's units."""
    import fgumi_b200 as fg
    kind = "narrow" if case == "device" else "deep"
    groups = simplex_groups(kind)
    if case == "device":
        want, count, s, _ = simplex_expected(kind)
        make = lambda: simplex_caller(fg, True, 4)
    else:
        want, count, flt, _ = filtered_expected(kind, 0.3)
        make = lambda: filtered_caller(fg, 0.3, 4)
    monkeypatch.setenv("FGB_CALLER_TRACE", "1")
    monkeypatch.setenv("FGB_SUBMIT_TRACE", "1")
    monkeypatch.delenv("FGB_SUBMIT_CHUNK_MB", raising=False)
    capfd.readouterr()
    one, st1, err1 = run_caller(make, groups, capfd)
    monkeypatch.setenv("FGB_SUBMIT_CHUNK_MB", "1")            # read when the caller's engine is created
    many, st2, err2 = run_caller(make, groups, capfd)
    assert n_chunks(err1) == 1 and n_chunks(err2) > 1, (n_chunks(err1), n_chunks(err2))
    assert ("records assembled on the device" in err2) == (case == "device")
    assert many.count == one.count == count
    assert many.data == one.data
    assert_same_stream(many.data, want)
    assert st1 == st2
    if case == "device":
        assert_simplex_stats(st2, s)
    else:
        assert_filter_stats(st2, flt)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,track_rejects", [("narrow", False), ("deep", False), ("deep", True)])
def test_overlap_prepass_at_depth(kind, track_rejects):
    """consensus_call_overlapping_bases on deep families of overlapping 150-301 bp pairs: the device pre-pass (K0o)
    with device assembly (narrow) and with host assembly (deep), and the host pre-pass (track_rejects), against the
    oracle's pre-pass followed by the oracle caller."""
    import fgumi_b200 as fg
    groups = simplex_groups(kind)
    want, count, s, ov = simplex_expected(kind, overlap=True)
    got, st, _ = run_caller(lambda: simplex_caller(fg, True, 4, consensus_call_overlapping_bases=True,
                                                   track_rejects=track_rejects), groups)
    assert got.count == count
    assert_same_stream(got.data, want)
    assert_simplex_stats(st, s)
    assert (st["overlapping_bases"], st["overlap_bases_agreeing"], st["overlap_bases_disagreeing"],
            st["overlap_bases_corrected"]) == ov
    assert ov[0] > 100000 and ov[2] > 0 and ov[3] > 0
    assert want != simplex_expected(kind)[0]                  # the pre-pass changes the output


# ------------------------------------------------------------------------------------------------------------------
# duplex and CODEC
# ------------------------------------------------------------------------------------------------------------------
DUPLEX_FILTER = dict(min_reads=(10, 5, 2), max_read_error_rate=(0.05, 0.05, 0.1), max_base_error_rate=(0.2, 0.1, 0.3),
                     min_base_quality=20, max_no_call_fraction=0.3)


@lru_cache(maxsize=None)
def duplex_expected(min_reads, filtered):
    from tests.test_caller_parity import duplex_job_fn
    oracle = R.DuplexCallerOracle("fgumi", "A", min_reads=min_reads, per_base=True, cell_tag=b"CB", vote_fn=vote_fn,
                                  builder_fn=O.builder_call, duplex_job_fn=duplex_job_fn)
    want, count = bytearray(), 0
    for g in duplex_workload(21):
        d, n = oracle.consensus_reads(g)
        want += d
        count += n
    unfiltered = bytes(want)
    flt = None
    if filtered:
        T, f = R.FilterThresholds, DUPLEX_FILTER
        flt = R.DuplexFilterOracle(*[T(f["min_reads"][i], f["max_read_error_rate"][i], f["max_base_error_rate"][i])
                                     for i in range(3)], f["min_base_quality"], None, f["max_no_call_fraction"], False)
        want, count = flt.filter_stream(unfiltered)
    return bytes(want), count, oracle, flt, unfiltered


@pytest.mark.gpu
@pytest.mark.parametrize("min_reads", [(1, 1, 0), (3, 2, 1)])
@pytest.mark.parametrize("filtered", [False, True])
def test_duplex_caller_at_depth(min_reads, filtered):
    """Duplex molecules with strand depths up to 300 and more than 255 pooled source reads (the scalar error recount)
    and 150-301 bp reads, with and without the duplex filter."""
    import fgumi_b200 as fg
    groups = duplex_workload(21)
    want, count, oracle, flt, unfiltered = duplex_expected(min_reads, filtered)
    recs = parse_records(unfiltered)
    assert any(r["tags"].get(b"aD", 0) > 0 and r["tags"].get(b"bD", 0) > 0 and r["tags"][b"cD"] > 255 for r in recs)
    assert any(max(r["tags"].get(b"aD", 0), r["tags"].get(b"bD", 0)) > 255 for r in recs)
    assert {"c", "C", "S"} <= tag_types(unfiltered, b"aD") | tag_types(unfiltered, b"bD")
    f = fg.DuplexConsensusFilter(**DUPLEX_FILTER) if filtered else None
    got, st, _ = run_caller(lambda: fg.DuplexConsensusCaller("fgumi", "A", min_reads=min_reads, produce_per_base_tags=True,
                                                            device=0, cell_tag=b"CB", n_threads=4, filter=f), groups)
    assert got.count == count
    assert_same_stream(got.data, want)
    s = oracle.stats
    assert st["total_reads"] == s.total_reads and st["consensus_reads"] == s.consensus_reads
    assert st["filtered_reads"] == s.filtered_reads
    for k in ("InsufficientReads", "PotentialCollision", "MinorityAlignment"):
        assert st[k] == s.rejections.get(k, 0), k
    if filtered:
        assert st["filter_records"] == flt.total and st["filter_passed"] == flt.passed
        assert st["filter_bases_masked"] == flt.bases_masked
        assert 0 < flt.passed < flt.total
    assert count >= 8


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [
    dict(),
    dict(max_dis=20, max_rate=0.05, per_base=True),
    dict(min_reads_per_strand=25, outer_qual=7, outer_len=10, ss_qual=4, per_base=True),
])
def test_codec_caller_at_depth(kw):
    """CODEC molecules with strands of up to 300 reads of 150-301 bp: long padded combine jobs and large depth sums."""
    import fgumi_b200 as fg
    from tests.test_codec_oracle_kat import codec_job_fn
    groups = codec_workload(31)
    oracle = R.CodecCallerOracle("codec", "RG1", vote_fn=vote_fn, builder_fn=O.builder_call, codec_job_fn=codec_job_fn,
                                 cell_tag=b"CB", **kw)
    want, count = bytearray(), 0
    for g in groups:
        d, n = oracle.consensus_reads(g)
        want += d
        count += n
    got, st, _ = run_caller(lambda: fg.CodecConsensusCaller(
        "codec", "RG1", min_reads_per_strand=kw.get("min_reads_per_strand", 1), single_strand_qual=kw.get("ss_qual"),
        outer_bases_qual=kw.get("outer_qual"), outer_bases_length=kw.get("outer_len", 5),
        max_duplex_disagreements=kw.get("max_dis"), max_duplex_disagreement_rate=kw.get("max_rate", 1.0),
        produce_per_base_tags=kw.get("per_base", False), device=0, cell_tag=b"CB", n_threads=4), groups)
    assert got.count == count
    assert_same_stream(got.data, bytes(want))
    assert st["total_reads"] == oracle.total_input_reads
    assert st["consensus_reads"] == oracle.consensus_reads_generated
    assert st["filtered_reads"] == oracle.reads_filtered
    for k in ("FragmentRead", "InsufficientReads", "MinorityAlignment", "InsufficientOverlap", "IndelErrorBetweenStrands"):
        assert st[k] == oracle.rejections.get(k, 0), k
    assert st["duplex_bases"] == oracle.duplex_bases and st["duplex_disagreements"] == oracle.duplex_disagreements
    assert count >= 3 and max(cd_values(bytes(want))) > 255 and oracle.duplex_disagreements > 0


# ------------------------------------------------------------------------------------------------------------------
# CPU: the product's host code at depth on the mock engine
# ------------------------------------------------------------------------------------------------------------------
MOCK_LADDER = (1, 2, 5, 24, 25, 127, 128, 129, 255, 256, 300, 513)
MOCK_DUPLEX_LADDER = ((1, 1), (2, 1), (5, 4), (127, 129), (128, 127), (200, 60), (256, 0), (300, 280))


def test_callers_at_depth_on_a_mock_engine(tmp_path):
    """The host side of the simplex and duplex callers at depth -- host record assembly, the integer tag widths
    ('c' / 'C' / 'S') and the record-size formula, the filter stages -- compiled with ASan + UBSan and run on the CPU
    with tests/native/mock_engine.cpp standing in for the GPU; the bytes must equal the oracle pipeline's."""
    import shutil
    import subprocess
    import fgumi_b200 as fg
    from tests.test_caller_planning import _oracle_stream
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    libdir = os.path.join(ROOT, "fgumi_b200")
    fg.lib.load()
    exe = tmp_path / "caller_e2e"
    nat = os.path.join(ROOT, "tests", "native")
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=address,undefined",
                        "-fno-sanitize-recover=all", "-o", str(exe), os.path.join(nat, "caller_e2e.cpp"),
                        os.path.join(nat, "mock_engine.cpp"), os.path.join(libdir, "csrc", "host", "caller_host.cpp"),
                        os.path.join(libdir, "csrc", "host_tables.cpp"), os.path.join(ROOT, "oracle", "fgumi_oracle.cpp"),
                        os.path.join(ROOT, "oracle", "oracle_capi.cpp"),
                        "-L" + libdir, "-lfgumi_b200", "-Wl,-rpath," + libdir, "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rng = np.random.default_rng(41)
    cases = [(0, simplex_workload(41, MOCK_LADDER, frag_depths=(5, 128, 256))),
             (1, [duplex_molecule(rng, g, a, b) for g, (a, b) in enumerate(MOCK_DUPLEX_LADDER)])]
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1")
    for mode, groups in cases:
        path = tmp_path / ("groups%d.bin" % mode)
        with open(path, "wb") as f:
            f.write(struct.pack("<II", mode, len(groups)))
            for g in groups:
                f.write(struct.pack("<I", len(g)))
                for rec in g:
                    f.write(struct.pack("<I", len(rec)) + bytes(rec))
        for variant in (0, 1):
            want = _oracle_stream(mode, variant, groups)
            ints = tag_types(want, b"cD") | tag_types(want, b"cM") | tag_types(want, b"aD") | tag_types(want, b"bD")
            assert {"c", "C", "S"} <= ints, (mode, variant, ints)
            for threads in (1, 4):
                outp = tmp_path / ("out_%d_%d_%d.bin" % (mode, variant, threads))
                r = subprocess.run([str(exe), str(path), str(threads), str(variant), str(outp)], capture_output=True,
                                   text=True, timeout=900, env=env)
                assert r.returncode == 0 and r.stdout.startswith("ok count"), (mode, variant, threads, r.stdout[-300:],
                                                                               r.stderr[-3000:])
                assert_same_stream(open(outp, "rb").read(), want)
