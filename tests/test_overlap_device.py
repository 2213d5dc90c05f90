"""The device overlapping-bases pre-pass (K0o, unpack_kernels.cuh overlap_kernel) against the host pre-pass and the
record oracle.

With a GPU the simplex caller does not rewrite the mates' overlap on the host: it plans runs from the headers and
CIGARs, K0o applies them on the uploaded records, and the host predicts the row lengths K0o will leave behind
(plan_read_len_eff evaluates the rule at each row's tail).  The reference runs the pre-pass on every MI group before
the caller looks at it (simplex.rs:395-398), so rejected pairs are co-called and counted too.  Three parts:
A. groups the rules reject, holding overlapping pairs, at every place in a batch (first, last, middle, alone, and a
   group whose last record is a rejected mate), through add_group, add_groups on 1 and 4 threads, two flushes on one
   caller, and the zero-copy path; bytes and every statistic against the oracle and against the host pre-pass
   (track_rejects=True);
B. row tails decided by co-called bases (ties, masked differences, lifted agreements, N mates, several positions,
   odd offsets, I / D / N runs, one-base overlaps, quality sums at the cap), each case counted on the oracle;
C. all nine strategies through fgb_submit_ex(FGB_IN_RECORDS): records + runs against records the host pre-pass
   rewrote, vote columns and counters, with runs on records that yield no row at both ends of the blob."""
import ctypes as C
import os
import sys
from functools import lru_cache

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import record_oracle as R              # noqa: E402
from tests import oracle_lib as O                  # noqa: E402
from tests.bam_builder import make_record, encode_op   # noqa: E402
from tests.test_record_oracle_kat import vote_fn   # noqa: E402

P, F1, F2, REV, MREV = R.PAIRED, R.FIRST_SEGMENT, R.LAST_SEGMENT, R.REVERSE, R.MATE_REVERSE
M, I, D, N_ = 0, 1, 2, 3
ACGT = np.frombuffer(b"ACGT", np.uint8)
OVERLAP_STATS = ("overlapping_bases", "overlap_bases_agreeing", "overlap_bases_disagreeing", "overlap_bases_corrected")
REJECTIONS = ("InsufficientReads", "SecondaryOrSupplementary", "ZeroLengthAfterTrimming", "MinorityAlignment",
              "OrphanConsensus")


# ------------------------------------------------------------------------------------------------------------------
# workload builder
# ------------------------------------------------------------------------------------------------------------------
def _cigar_str(cig):
    return "".join("%d%s" % (n, "MIDNSHP=X"[k]) for k, n in cig)


def _ref_len(cig):
    return sum(n for k, n in cig if k in (M, D, N_, 7, 8))


def fr_pair(name, mi, s1, cig1, seq1, q1, s2, cig2, seq2, q2):
    """An FR pair: R1 forward from 1-based s1, R2 reverse from s2 (stored in reference orientation), mate fields and
    MC tags filled in as an aligner would.  With s1 <= s2 and R1 ending no later than R2, neither mate reads past the
    other, so the mate-overlap clip leaves both rows whole and both oriented tails lie in the overlap."""
    e1, e2 = s1 + _ref_len(cig1) - 1, s2 + _ref_len(cig2) - 1
    tl = max(e1, e2) - min(s1, s2) + 1
    tf = tl if s1 <= s2 else -tl
    tags = [(b"MI", "Z", mi)]
    r1 = make_record(name=name, flags=P | F1 | MREV, pos=s1 - 1, cigar=[encode_op(k, n) for k, n in cig1],
                     mate_ref_id=0, mate_pos=s2 - 1, tlen=tf, seq=bytes(seq1), quals=bytes(q1),
                     tags=tags + [(b"MC", "Z", _cigar_str(cig2).encode())])
    r2 = make_record(name=name, flags=P | F2 | REV, pos=s2 - 1, cigar=[encode_op(k, n) for k, n in cig2],
                     mate_ref_id=0, mate_pos=s1 - 1, tlen=-tf, seq=bytes(seq2), quals=bytes(q2),
                     tags=tags + [(b"MC", "Z", _cigar_str(cig1).encode())])
    return bytes(r1), bytes(r2)


def _blocks(rec):
    """Aligned (M / = / X) blocks of a record: (1-based ref start, read offset, length)."""
    v = R.Rec(rec)
    ref, read, out = v.pos + 1, 0, []
    for op in v.cigar_ops():
        k, n = op & 0xF, op >> 4
        if k in (0, 7, 8):
            out.append((ref, read, n))
            ref += n
            read += n
        else:
            ref += n if k in (2, 3) else 0
            read += n if k in (1, 4) else 0
    return out


def plan_runs(r1, r2):
    """The runs of a pair: stretches where both mates have aligned bases on the same reference positions, as
    (o1, o2, len) in R1 order -- what overlap.h plan_pair hands the device."""
    runs = []
    for ra, qa, na in _blocks(r1):
        for rb, qb, nb in _blocks(r2):
            lo, hi = max(ra, rb), min(ra + na, rb + nb)
            if lo < hi:
                runs.append((qa + lo - ra, qb + lo - rb, hi - lo))
    return sorted(runs)


def _pair_from_template(rng, L=50, d=None, cig1=None, cig2=None, qlo=20, qhi=41):
    """An overlapping pair read off a random template: R1 from 100, R2 from 100 + d, both L bases, few errors."""
    d = int(rng.integers(5, 26)) if d is None else d
    cig1 = cig1 or [(M, L)]
    cig2 = cig2 or [(M, L)]
    tmpl = ACGT[rng.integers(0, 4, size=400)]
    def read(start, cig):
        seq, ref, out = tmpl, start, []
        for k, n in cig:
            if k == M:
                out += list(seq[ref:ref + n]); ref += n
            elif k == I:
                out += list(ACGT[rng.integers(0, 4, size=n)])
            else:
                ref += n
        s = np.array(out, np.uint8)
        m = rng.random(len(s)) < 0.02
        s[m] = ACGT[rng.integers(0, 4, size=int(m.sum()))]
        return s, rng.integers(qlo, qhi, size=len(s)).astype(np.uint8)
    s1, q1 = read(100, cig1)
    s2, q2 = read(100 + d, cig2)
    return s1, q1, s2, q2, 101, 101 + d, cig1, cig2


def ordinary_pair(rng, name, mi):
    s1, q1, s2, q2, p1, p2, c1, c2 = _pair_from_template(rng)
    return list(fr_pair(name, mi, p1, c1, s1, q1, p2, c2, s2, q2))


def group(rng, kind, g, min_reads):
    """One MI group of a kind:
    ord       min_reads + 1 ordinary pairs (one consensus R1 and R2);
    single    one overlapping pair, below min_reads (2 or 3);
    zero      min_reads + 1 pairs; the last one's R2 yields no row (all N, or every base below the input quality
              limit even after the co-call) while its R1 survives; that R2 is the group's last record;
    minority  min_reads + 1 pairs; the last pair's mates both carry an alignment the others do not (minority)."""
    mi = b"g%d" % g
    n = 1 if kind == "single" else min_reads + 1
    recs = []
    for k in range(n):
        recs += ordinary_pair(rng, b"g%d_%d" % (g, k), mi)
    name = b"g%d_%d" % (g, n - 1)
    if kind == "zero":
        s1, q1, s2, q2, p1, p2, c1, c2 = _pair_from_template(rng)
        if g % 2:
            s2[:] = ord("N")
        else:                                # agreeing overlap: 2..4 + 1..4 stays below 10 after the sum
            ov = 50 - (p2 - p1)
            q1[50 - ov:] = rng.integers(2, 5, size=ov)
            s2[:ov] = s1[50 - ov:]
            q2[:] = rng.integers(1, 5, size=50)
        recs[-2:] = fr_pair(name, mi, p1, c1, s1, q1, p2, c2, s2, q2)
    elif kind == "minority":
        s1, q1, s2, q2, p1, p2, c1, c2 = _pair_from_template(rng, cig1=[(M, 20), (D, 2), (M, 30)],
                                                             cig2=[(M, 25), (I, 3), (M, 22)])
        recs[-2:] = fr_pair(name, mi, p1, c1, s1, q1, p2, c2, s2, q2)
    return recs


LAYOUTS = {
    "first": ("single", "ord", "ord"),
    "last": ("ord", "ord", "single"),
    "middle": ("ord", "single", "ord"),
    "only": ("single", "single", "single"),
    "last_mate_zero": ("ord", "minority", "zero"),
    "last_mate_minority": ("zero", "ord", "minority"),
}


@lru_cache(maxsize=None)
def layout_groups(layout, min_reads, threaded):
    """The groups of one batch.  `threaded` puts 70 more groups in the middle (ordinary ones; rejected ones for the
    layout of only rejected groups), enough for add_groups to cut the batch between 2+ threads."""
    rng = np.random.default_rng(17 + 10 * sorted(LAYOUTS).index(layout) + min_reads)
    kinds = list(LAYOUTS[layout])
    if threaded:
        fill = "single" if layout == "only" else "ord"
        kinds = kinds[:1] + [fill] * 70 + kinds[1:]
    return tuple(tuple(group(rng, k, g, min_reads)) for g, k in enumerate(kinds))


def oracle_run(groups, min_reads, min_q=10, overlap=True):
    """Oracle pre-pass (every group) followed by the oracle caller: (bytes, count, caller stats, overlap stats)."""
    opt = R.VanillaOptions(min_reads=min_reads, min_consensus_base_quality=2, min_input_base_quality=min_q)
    oracle = R.VanillaCallerOracle("fgumi", "A", opt, vote_fn, O.builder_call)
    ov = R.OverlappingOracle()
    out, count = bytearray(), 0
    for g in groups:
        recs = [bytearray(r) for r in g]
        if overlap:
            ov.apply(recs)
        d, n = oracle.consensus_reads([bytes(r) for r in recs])
        out += d
        count += n
    return bytes(out), count, oracle.stats, ov.stats()


def stat_view(s, ov, times=1):
    """The product's statistic names for an oracle run, `times` flushes of it."""
    d = {"total_reads": s.total_reads, "consensus_reads": s.consensus_reads, "filtered_reads": s.filtered_reads}
    d.update({k: s.rejections.get(k, 0) for k in REJECTIONS})
    d.update(dict(zip(OVERLAP_STATS, ov)))
    return {k: v * times for k, v in d.items()}


# ---- part B: row tails ------------------------------------------------------------------------------------------
TAIL_CASES = ("tie", "lowdiff", "lift", "n_tail", "n_mate", "sum93")
OPS = ("M", "M", "I", "D", "N", "ID", "DN")


def _op_cigar(rng, L, op):
    """L read bases with `op` (I, D or N; one or two of them) inside the read's last 30 bases."""
    if op == "M":
        return [(M, L)]
    cuts = sorted(int(x) for x in rng.choice(np.arange(max(3, L - 28), L - 3, 2 * len(op)), size=len(op),
                                             replace=False))
    cig, at = [], 0
    for k, (c, o) in enumerate(zip(cuts, op)):
        cig.append((M, c - at))
        nxt = cuts[k + 1] if k + 1 < len(cuts) else L
        n = int(rng.integers(1, 4)) if o != "N" else int(rng.integers(5, 40))
        if o == "I":
            n = max(1, min(n, nxt - c - 1))
        cig.append(({"I": I, "D": D, "N": N_}[o], n))
        at = c + (n if o == "I" else 0)
    cig.append((M, L - at))
    assert all(n > 0 for _, n in cig) and sum(n for k, n in cig if k in (M, I)) == L
    return cig


def _plant(rng, case, min_q, c_t, q_t, c_m, q_m):
    """Set the tail mate's base / quality (c_t, q_t) and the other mate's (c_m, q_m) at one overlap position."""
    other = lambda b: ACGT[(int(np.flatnonzero(ACGT == b)[0]) + int(rng.integers(1, 4))) % 4]
    if case == "tie":                    # disagreement, equal qualities: N on both sides
        c_m = other(c_t)
        q_t = q_m = int(rng.integers(min_q, 60))
    elif case == "lowdiff":              # disagreement whose difference stays below the input limit
        c_m = other(c_t)
        lo = int(rng.integers(0, 60))
        hi = lo + int(rng.integers(2, max(3, min_q)))
        q_t, q_m = (lo, hi) if rng.random() < 0.5 else (hi, lo)
    elif case == "lift":                 # agreement of two masked qualities whose sum reaches the limit
        c_m = c_t
        q_t = int(rng.integers(1, max(2, min_q)))
        q_m = int(rng.integers(max(1, min_q - q_t), min_q))
    elif case == "n_tail":               # the tail mate has N: the position is skipped
        c_t = ord("N")
    elif case == "n_mate":               # the other mate has N: skipped, a masked tail stays masked
        c_m = ord("N")
        q_t = int(rng.integers(0, max(1, min_q)))
    elif case == "sum93":                # agreement at / past the cap
        c_m = c_t
        q_t = int(rng.integers(30, 94))
        q_m = int(rng.integers(max(0, 93 - q_t), 94))
    return c_t, q_t, c_m, q_m


def tail_pair(rng, g, min_q):
    """An FR pair with planted tail positions: returns (records, [(side, case) planted], runs)."""
    L1, L2 = int(rng.choice([31, 40, 51, 64])), int(rng.choice([31, 40, 51, 64]))
    op1, op2 = OPS[int(rng.integers(0, len(OPS)))], OPS[int(rng.integers(0, len(OPS)))]
    cig1, cig2 = _op_cigar(rng, L1, op1), _op_cigar(rng, L2, op2)
    ov = 1 if rng.random() < 0.08 else int(rng.integers(2, min(_ref_len(cig1), _ref_len(cig2)) + 1))
    s1 = 101
    e1 = s1 + _ref_len(cig1) - 1
    s2 = e1 - ov + 1
    qlo = min_q + 1
    seq1 = ACGT[rng.integers(0, 4, size=L1)].copy()
    seq2 = ACGT[rng.integers(0, 4, size=L2)].copy()
    q1 = rng.integers(qlo, qlo + 25, size=L1).astype(np.uint8)
    q2 = rng.integers(qlo, qlo + 25, size=L2).astype(np.uint8)
    r1, r2 = fr_pair(b"t%d" % g, b"t%d" % g, s1, cig1, seq1, q1, s2, cig2, seq2, q2)
    runs = plan_runs(r1, r2)
    m1 = {o1 + k: o2 + k for o1, o2, n in runs for k in range(n)}
    m2 = {v: k for k, v in m1.items()}
    for i1, i2 in m1.items():            # agreeing overlap unless planted
        seq2[i2] = seq1[i1]
    planted, used = [], set()
    for side in ("r1", "r2"):
        if rng.random() < 0.15:
            continue
        depth = int(rng.choice([1, 1, 2, 3, 4]))
        for j in range(depth):
            it = L1 - 1 - j if side == "r1" else j          # oriented tail: R1's 3' end, R2's record start
            mm = m1 if side == "r1" else m2
            if it not in mm:
                break
            im = mm[it]
            key = (it, im) if side == "r1" else (im, it)     # (R1 offset, R2 offset): a position is planted once
            if key in used:
                break
            used.add(key)
            case = TAIL_CASES[int(rng.integers(0, len(TAIL_CASES)))]
            st, qt, sm, qm = (seq1, q1, seq2, q2) if side == "r1" else (seq2, q2, seq1, q1)
            st[it], qt[it], sm[im], qm[im] = _plant(rng, case, min_q, st[it], qt[it], sm[im], qm[im])
            planted.append((side, case, j))
    recs = fr_pair(b"t%d" % g, b"t%d" % g, s1, cig1, seq1, q1, s2, cig2, seq2, q2)
    return list(recs), planted, runs


def final_len(rec, min_q):
    r = R.Rec(rec)
    sr = R.create_source_read(r, 0, R.num_bases_extending_past_mate(r), R.VanillaOptions(min_input_base_quality=min_q))
    return 0 if sr is None else len(sr.bases)


@lru_cache(maxsize=None)
def tail_workload(min_q, n=260):
    rng = np.random.default_rng(100 + min_q)
    return tuple(tail_pair(rng, g, min_q) for g in range(n))


def tail_census(min_q):
    """Per case, how often the workload reaches it (on the oracle), and how often the pre-pass makes a row longer or
    shorter than it would be without it."""
    c = {k: 0 for k in ("longer", "shorter", "one_base", "odd_start", "odd_end", "runs2", "runs3", "several",
                        "r1_tie_stripped", "r2_tie_stripped", "lowdiff_masked", "lift_kept", "n_skipped",
                        "sum93_capped")}
    for recs, planted, runs in tail_workload(min_q):
        after = [bytearray(r) for r in recs]
        R.OverlappingOracle().apply(after)
        for k in range(2):
            a, b = final_len(recs[k], min_q), final_len(bytes(after[k]), min_q)
            c["longer"] += b > a
            c["shorter"] += b < a
        v0, v1 = [R.Rec(r) for r in recs], [R.Rec(bytes(r)) for r in after]
        c["one_base"] += sum(n for _, _, n in runs) == 1
        c["odd_start"] += any(o1 % 2 or o2 % 2 for o1, o2, _ in runs)
        c["odd_end"] += any((o1 + n) % 2 or (o2 + n) % 2 for o1, o2, n in runs)
        c["runs2"] += len(runs) == 2
        c["runs3"] += len(runs) >= 3
        c["several"] += any(j > 0 for _, _, j in planted)
        for side, case, j in planted:
            k = 0 if side == "r1" else 1
            L = v0[k].l_seq
            i = L - 1 - j if side == "r1" else j
            b0, b1 = v0[k].sequence()[i], v1[k].sequence()[i]
            qa, qb = v0[k].quals()[i], v1[k].quals()[i]
            fl = final_len(bytes(after[k]), min_q)
            oriented = L - 1 - i if side == "r2" else i      # position in read orientation
            if case == "tie" and b1 == ord("N") and b0 != ord("N") and fl <= oriented:
                c["r1_tie_stripped" if side == "r1" else "r2_tie_stripped"] += 1
            elif case == "lowdiff" and b1 != ord("N") and qb < min_q and fl <= oriented:
                c["lowdiff_masked"] += 1
            elif case == "lift" and qa < min_q <= qb and fl > oriented:
                c["lift_kept"] += 1
            elif case in ("n_tail", "n_mate") and qa == qb and b0 == b1 and fl <= oriented:
                c["n_skipped"] += 1
            elif case == "sum93" and qb == 93:
                c["sum93_capped"] += 1
    return c


TAIL_MINIMA = {"longer": 40, "shorter": 60, "one_base": 8, "odd_start": 60, "odd_end": 60, "runs2": 30, "runs3": 8,
               "several": 60, "r1_tie_stripped": 10, "r2_tie_stripped": 10, "lowdiff_masked": 10, "lift_kept": 10,
               "n_skipped": 10, "sum93_capped": 20}


# ---- part C: fgb_submit_ex(FGB_IN_RECORDS) -------------------------------------------------------------------------
RUN_DTYPE = np.dtype([("seq1_off", "<u8"), ("seq2_off", "<u8"), ("l_seq1", "<u4"), ("l_seq2", "<u4"),
                      ("o1", "<u4"), ("o2", "<u4"), ("len", "<u4"), ("flags", "<u4")])
assert RUN_DTYPE.itemsize == 40
PRE = POST = 93                          # the highest phreds the engine accepts


def abi_pairs(seed=5, n=90):
    """Pairs for the ABI differential: simple CIGARs, I / D / N (multi-run pairs), a deletion of 3 read bases in
    R1 so two runs of R1 meet inside one packed byte, one-base overlaps.  Qualities span 0..93."""
    rng = np.random.default_rng(seed)
    pairs = []
    for g in range(n):
        kind = g % 5
        L1, L2 = int(rng.integers(20, 70)), int(rng.integers(20, 70))
        if kind == 0:
            c1, c2 = [(M, L1)], [(M, L2)]
        elif kind == 1:
            c1, c2 = _op_cigar(rng, L1, "ID"), _op_cigar(rng, L2, "N")
        elif kind == 2:                  # R1 offsets ..a-1 | a.. with a odd: the two runs share a packed byte
            a = L1 - 2 * int(rng.integers(3, 8)) - 1
            c1, c2 = [(M, a), (D, int(rng.integers(1, 4))), (M, L1 - a)], [(M, L2)]
        elif kind == 3:
            c1, c2 = _op_cigar(rng, L1, "D"), _op_cigar(rng, L2, "I")
        else:
            c1, c2 = [(M, L1)], [(M, L2)]
        ov = 1 if kind == 4 else int(rng.integers(2, min(_ref_len(c1), _ref_len(c2)) + 1))
        s2 = 101 + _ref_len(c1) - ov
        seq1, seq2 = ACGT[rng.integers(0, 4, size=L1)].copy(), ACGT[rng.integers(0, 4, size=L2)].copy()
        q1, q2 = rng.integers(0, 94, size=L1).astype(np.uint8), rng.integers(0, 94, size=L2).astype(np.uint8)
        r1, r2 = fr_pair(b"c%d" % g, b"c%d" % g, 101, c1, seq1, q1, s2, c2, seq2, q2)
        runs = plan_runs(r1, r2)
        for o1, o2, k in runs:           # mostly agreeing, with disagreements and N on either side
            for t in range(k):
                u = rng.random()
                if u < 0.6:
                    seq2[o2 + t] = seq1[o1 + t]
                elif u < 0.65:
                    seq1[o1 + t] = ord("N")
                elif u < 0.7:
                    seq2[o2 + t] = ord("N")
        pairs.append(fr_pair(b"c%d" % g, b"c%d" % g, 101, c1, seq1, q1, s2, c2, seq2, q2))
    return pairs


def _seq_off(rec):
    v = R.Rec(rec)
    return v.seq_offset(), v.l_seq


def abi_batch(pairs, with_rows):
    """The blob of every pair's records, the runs of every pair (offsets into the blob), and one single-read unit per
    record of the pairs in `with_rows` (full-length rows)."""
    blob, offs = b"", []
    for r1, r2 in pairs:
        offs.append((len(blob), len(blob) + len(r1)))
        blob += r1 + r2
    runs = []
    for (r1, r2), (a1, a2) in zip(pairs, offs):
        (so1, l1), (so2, l2) = _seq_off(r1), _seq_off(r2)
        for k, (o1, o2, n) in enumerate(plan_runs(r1, r2)):
            runs.append((a1 + so1, a2 + so2, l1, l2, o1, o2, n, 1 if k else 0))
    rows, raws = [], []
    for i in with_rows:
        for rec, a in zip(pairs[i], offs[i]):
            so, L = _seq_off(rec)
            rows.append(L)
            raws.append((a + so, L, 1 if R.Rec(rec).flags & REV else 0))
    return blob, np.array(runs, RUN_DTYPE), rows, raws


def submit_records(fg, eng, blob, rows, raws, min_q, runs=None, agree=0, disagree=0):
    """fgb_submit_ex(FGB_IN_RECORDS) of one-read units; returns (base, qual, depth, errors) and the overlap counters."""
    lib = fg.lib.load()
    layout = fg.pack_source_reads([[(b"\0" * n, b"\0" * n)] for n in rows], 1)
    fg.plan_tiles(layout)
    rr = np.zeros(len(raws) + 1, dtype=fg.RAW_READ_DTYPE)
    for k, x in enumerate(raws):
        rr[k] = x
    out = fg.HostColumns.alloc(layout.n_out)
    data = np.frombuffer(blob, np.uint8).copy()
    b = fg.lib.FgbBatch(layout.n_units, layout.n_reads, layout.n_bytes, layout.n_out, len(layout.tiles), None, None,
                        layout.reads.ctypes.data, layout.units.ctypes.data, layout.tiles.ctypes.data)
    c = fg.lib.FgbColumns(out.base.ctypes.data, out.qual.ctypes.data, out.depth.ctypes.data, out.errors.ctypes.data)
    rc = fg.lib.FgbRecordColumns(len(data), data.ctypes.data, rr.ctypes.data, min_q)
    o = fg.lib.FgbSubmitOptions()
    o.input_format, o.output_format = fg.lib.FGB_IN_RECORDS, fg.lib.FGB_OUT_U16
    o.records = C.cast(C.pointer(rc), C.c_void_p)
    stats = np.zeros(4, np.uint64)
    if runs is not None and len(runs):
        o.overlap_runs, o.n_overlap_runs = runs.ctypes.data, len(runs)
        o.overlap_stats = stats.ctypes.data
        o.overlap_agreement, o.overlap_disagreement = agree, disagree
    eng._check(lib.fgb_submit_ex(eng._h, C.byref(b), C.byref(c), C.byref(o)), "fgb_submit_ex")
    eng.wait()
    assert bytes(data) == blob                           # the host blob is never written
    return (out.base, out.qual, out.depth, out.errors), tuple(int(x) for x in stats), layout


def host_rewritten(fg, pairs, agree, disagree):
    """The pairs after the product's host pre-pass (fgb_overlap_apply_group) with one strategy, and its counters."""
    out, tot = [], np.zeros(4, np.int64)
    for r1, r2 in pairs:
        got, st = fg.apply_overlapping_consensus([r1, r2], agree, disagree)
        out.append(tuple(got))
        tot += st
    return out, tuple(int(x) for x in tot)


def quality_map(pre=PRE, post=POST):
    """Output quality of a one-read unit for every input quality 0..93 (CPU oracle, no consensus-quality floor)."""
    import fgumi_b200 as fg
    b = fg.pack_source_reads([[(b"A", bytes([q]))] for q in range(94)], 1)
    _, oq, _, _, _ = O.simplex_batch(b, pre, post, 1, 0)
    return [int(oq[int(b.units["out_off"][q])]) for q in range(94)]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the builder against the oracles
# ------------------------------------------------------------------------------------------------------------------
def test_builder_kinds_reach_their_rejections():
    """Each group kind is rejected the way it is meant to be, the pre-pass counts overlap in every kind, and in the
    'zero' kind the group's last record is the mate that yields no row."""
    rng = np.random.default_rng(3)
    for min_reads in (2, 3):
        for kind, reason in (("single", "InsufficientReads"), ("zero", "ZeroLengthAfterTrimming"),
                             ("minority", "MinorityAlignment")):
            for g in range(4):
                recs = group(rng, kind, g, min_reads)
                data, n, s, ov = oracle_run([recs], min_reads)
                assert s.rejections.get(reason, 0) >= 1, (kind, min_reads, s.rejections)
                if kind == "single":
                    assert n == 0 and data == b""
                else:
                    assert n == 2, (kind, min_reads, n)
                if kind != "zero" or g % 2 == 0:
                    assert ov[0] > 0, (kind, g)
                if kind == "zero":
                    after = [bytearray(r) for r in recs]
                    R.OverlappingOracle().apply(after)
                    assert final_len(bytes(after[-1]), 10) == 0 and final_len(bytes(after[-2]), 10) > 0
                    assert R.Rec(recs[-1]).flags & F2
        data, n, s, ov = oracle_run([group(rng, "ord", 9, min_reads)], min_reads)
        assert n == 2 and s.filtered_reads == 0 and ov[0] > 0


def test_builder_runs_match_the_oracle_pre_pass():
    """plan_runs (the runs the tests hand the device) covers exactly the positions the oracle co-calls."""
    pairs = abi_pairs(seed=7, n=60) + [tuple(p[0]) for p in tail_workload(10)[:60]]
    for r1, r2 in pairs:
        runs = plan_runs(r1, r2)
        s1, s2 = R.Rec(r1).sequence(), R.Rec(r2).sequence()
        called = sum(1 for o1, o2, n in runs for t in range(n) if s1[o1 + t] != ord("N") and s2[o2 + t] != ord("N"))
        o = R.OverlappingOracle()
        o.call(bytearray(r1), bytearray(r2))
        assert o.overlapping_bases == called
        assert all(runs[k][0] + runs[k][2] <= runs[k + 1][0] for k in range(len(runs) - 1))


@pytest.mark.parametrize("min_q", [10, 30])
def test_tail_workload_reaches_every_case(min_q):
    """Every tail case of part B is reached, the minimum number of times, on the oracle."""
    c = tail_census(min_q)
    short = {k: (c[k], v) for k, v in TAIL_MINIMA.items() if c[k] < v}
    assert not short, short


def test_quality_map_of_a_one_read_unit():
    """Part C compares vote columns, so a quality the pre-pass changed must change the output.  No error rates the
    engine accepts make a one-read unit's output quality one-to-one on 2..93 (the pre- and post-UMI error terms
    squeeze the top of the scale); at 93 / 93 it is the identity on 2..65, and part C checks the rest of the
    range through its counters and the one-to-one part through the vote."""
    f = quality_map()
    assert f[2:66] == list(range(2, 66))
    assert len(set(f[2:])) < 92                       # the top collides: see above
    for pre, post in ((45, 40), (90, 90)):
        g = quality_map(pre, post)
        assert sum(a == b for a, b in zip(g[2:66], range(2, 66))) < 64


@pytest.mark.parametrize("agree,disagree", [(a, d) for a in range(3) for d in range(3)])
def test_abi_pairs_host_pre_pass_matches_the_oracle(fg, agree, disagree):
    pairs = abi_pairs()
    got, st = host_rewritten(fg, pairs, agree, disagree)
    o = R.OverlappingOracle(agree, disagree)
    for (r1, r2), (g1, g2) in zip(pairs, got):
        a, b = bytearray(r1), bytearray(r2)
        o.call(a, b)
        assert (bytes(a), bytes(b)) == (g1, g2)
    assert st == o.stats() and st[0] > 1000 and st[2] > 100


# ------------------------------------------------------------------------------------------------------------------
# GPU part A: rejected groups with overlapping pairs at every batch position
# ------------------------------------------------------------------------------------------------------------------
def _caller(fg, min_reads, n_threads, track_rejects=False, min_q=10):
    opt = fg.VanillaUmiConsensusOptions(min_reads=min_reads, min_consensus_base_quality=2, min_input_base_quality=min_q)
    return fg.VanillaUmiConsensusCaller("fgumi", "A", opt, device=0, consensus_call_overlapping_bases=True,
                                        n_threads=n_threads, track_rejects=track_rejects)


def _two_flushes(c, groups, entry):
    outs = []
    for _ in range(2):
        if entry == "add_group":
            for g in groups:
                c.add_group(list(g))
        else:
            c.add_groups([list(g) for g in groups])
        outs.append(c.flush())
    st = c.statistics()
    c.close()
    return outs, st


@pytest.mark.gpu
@pytest.mark.parametrize("min_reads", [2, 3])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_rejected_groups_at_every_batch_position(fg, layout, min_reads):
    for entry, threads in (("add_group", 1), ("add_groups", 1), ("add_groups", 4)):
        groups = layout_groups(layout, min_reads, threads > 1)
        want, count, s, ov = oracle_run(groups, min_reads)
        assert ov[0] > 0
        outs, st = _two_flushes(_caller(fg, min_reads, threads), groups, entry)
        for out in outs:
            assert out.count == count and out.data == want, (layout, entry, threads)
        assert {k: st[k] for k in stat_view(s, ov)} == stat_view(s, ov, 2), (layout, entry, threads)
        host_outs, host_st = _two_flushes(_caller(fg, min_reads, threads, track_rejects=True), groups, entry)
        assert [(o.data, o.count) for o in host_outs] == [(o.data, o.count) for o in outs]
        assert host_st == st


@pytest.mark.gpu
@pytest.mark.parametrize("min_reads", [1, 2])
def test_rejected_groups_zero_copy(fg, min_reads):
    """The same layouts from the caller's own page-locked blob (options.zero_copy_records), which must stay as it
    was: the pre-pass is applied to the device copy only."""
    import torch
    from fgumi_b200 import benchlegs
    lib = fg.lib.load()
    for layout in sorted(LAYOUTS):
        for threads in (1, 4):
            groups = layout_groups(layout, max(min_reads, 2), threads > 1)
            want, count, s, ov = oracle_run(groups, min_reads)
            recs = [r for g in groups for r in g]
            blob = b"".join(recs)
            pinned = torch.empty(len(blob) + 64, dtype=torch.uint8).pin_memory()
            pinned.numpy()[:len(blob)] = np.frombuffer(blob, np.uint8)
            off = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.uint64)
            grp = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.uint64)
            c = benchlegs._Caller(lib, 0, threads, overlap=True, zero_copy=True, min_reads=min_reads)
            try:
                for _ in range(2):
                    ptr, n, cnt = c.process(pinned.data_ptr(), off.ctypes.data, grp.ctypes.data, len(groups))
                    assert cnt == count and (C.string_at(ptr, n) if n else b"") == want, (layout, threads)
                st = dict(zip(fg.lib.STAT_NAMES, c.stats()))
            finally:
                c.close()
            assert {k: st[k] for k in stat_view(s, ov)} == stat_view(s, ov, 2), (layout, threads)
            assert pinned.numpy()[:len(blob)].tobytes() == blob


# ------------------------------------------------------------------------------------------------------------------
# GPU part B: row tails decided by the co-called bases
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("min_q", [10, 30])
def test_row_tails_decided_by_co_called_bases(fg, min_q):
    groups = [tuple(p[0]) for p in tail_workload(min_q)]
    want, count, s, ov = oracle_run(groups, 1, min_q)
    c = tail_census(min_q)
    assert all(c[k] >= v for k, v in TAIL_MINIMA.items()), c
    for threads in (1, 4):
        outs, st = _two_flushes(_caller(fg, 1, threads, min_q=min_q), groups, "add_groups")
        for out in outs:
            assert out.count == count and out.data == want, threads
        assert {k: st[k] for k in stat_view(s, ov)} == stat_view(s, ov, 2)
        host_outs, host_st = _two_flushes(_caller(fg, 1, threads, track_rejects=True, min_q=min_q), groups,
                                          "add_groups")
        assert [(o.data, o.count) for o in host_outs] == [(o.data, o.count) for o in outs] and host_st == st
    assert want != oracle_run(groups, 1, min_q, overlap=False)[0]


# ------------------------------------------------------------------------------------------------------------------
# GPU part C: all nine strategies through fgb_submit_ex(FGB_IN_RECORDS)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_records_quality_map_control(fg):
    """A control batch without runs: each one-read unit's output quality is the CPU oracle's map of its input."""
    f = quality_map()
    quals = np.arange(94, dtype=np.uint8)
    rec = make_record(name=b"ctl", flags=0, pos=100, seq=bytes(ACGT[np.arange(94) % 4]), quals=quals.tobytes())
    so, L = _seq_off(rec)
    pad = make_record(name=b"pad", pos=1, seq=b"ACGT" * 10)
    blob = bytes(pad) + bytes(rec) + bytes(pad)
    eng = fg.Engine(0, PRE, POST, 1, 0)
    try:
        (ob, oq, od, oe), _, _ = submit_records(fg, eng, blob, [L], [(len(pad) + so, L, 0)], 0)
    finally:
        eng.close()
    assert list(oq[:94]) == f and bytes(ob[:94]) == bytes(ACGT[np.arange(94) % 4])


@pytest.mark.gpu
@pytest.mark.parametrize("min_q", [0, 20])
def test_records_runs_all_strategies_by_differential(fg, min_q):
    """(a) original records + runs with strategy s; (b) records rewritten by fgb_overlap_apply_group(s), no runs.
    The first and last pairs of the blob get runs but no rows."""
    pairs = abi_pairs()
    with_rows = list(range(1, len(pairs) - 1))
    eng = fg.Engine(0, PRE, POST, 1, 0)
    try:
        for agree in range(3):
            for disagree in range(3):
                blob, runs, rows, raws = abi_batch(pairs, with_rows)
                assert runs["flags"].any() and len(runs) > len(pairs)
                cols_a, st_a, _ = submit_records(fg, eng, blob, rows, raws, min_q, runs, agree, disagree)
                rewritten, st_host = host_rewritten(fg, pairs, agree, disagree)
                blob_b, _, _, raws_b = abi_batch(rewritten, with_rows)
                assert raws_b == raws
                cols_b, st_b, _ = submit_records(fg, eng, blob_b, rows, raws, min_q)
                for x, y in zip(cols_a, cols_b):
                    assert np.array_equal(x, y), (agree, disagree, min_q)
                assert st_a == st_host and st_b == (0, 0, 0, 0), (agree, disagree)
                assert host_rewritten(fg, [pairs[0], pairs[-1]], agree, disagree)[1][0] > 0   # the rowless ends count
                cols_0, _, _ = submit_records(fg, eng, blob, rows, raws, min_q)             # and the runs matter
                assert sum(int(np.count_nonzero(x != y)) for x, y in zip(cols_a[:2], cols_0[:2])) > 100, (agree, disagree)
    finally:
        eng.close()
