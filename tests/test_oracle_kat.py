"""Pins the CPU oracle against every known-answer test the reference holds for the hot path
(SURVEY.md §8c).  Each test names the reference test it reproduces
(fgumi 0.2.0: crates/fgumi-consensus/src/<file>:<line>).  CPU only.
"""
import ctypes as C
import math

import numpy as np
import pytest

from tests import oracle_lib as O
from fgumi_b200.engine import pack_source_reads

LN = math.log


@pytest.fixture(scope="module")
def L():
    return O.load()


# ------------------------------------------------------------------ phred.rs:356-701
def test_phred_to_ln_error(L):  # phred.rs:357-369
    for q, p in ((10, 0.1), (20, 0.01), (30, 0.001)):
        assert abs(L.orc_phred_to_ln_error_prob(q) - LN(p)) < 1e-10


def test_phred_round_trip(L):  # phred.rs:372-379
    for q in (2, 10, 20, 30, 40, 50, 60):
        assert L.orc_ln_prob_to_phred(L.orc_phred_to_ln_error_prob(q)) == q


def test_ln_sum_exp(L):  # phred.rs:382-394
    assert abs(L.orc_ln_sum_exp(LN(0.1), LN(0.2)) - LN(0.3)) < 1e-10
    v = np.array([LN(0.1), LN(0.2), LN(0.3)])
    assert abs(L.orc_ln_sum_exp_array(v.ctypes.data, 3) - LN(0.6)) < 1e-10


def test_error_two_trials_grid(L):  # phred.rs:397-432 (fgbio 100x100 grid, tol 1e-4)
    r = L.orc_ln_error_prob_two_trials(LN(0.1), LN(0.1))
    assert abs(math.exp(r) - (0.2 - (4.0 / 3.0) * 0.01)) < 1e-10
    for i in range(1, 101):
        for j in range(1, 101):
            p1, p2 = 1.0 / i, 1.0 / j
            exp = p1 * (1 - p2) + (1 - p1) * p2 + p1 * p2 * (2.0 / 3.0)
            act = math.exp(L.orc_ln_error_prob_two_trials(LN(p1), LN(p2)))
            assert abs(act - exp) < 1e-4, (i, j)


def test_ln_sum_exp_fgbio(L):  # phred.rs:436-456
    f = L.orc_ln_sum_exp
    ninf = float("-inf")
    assert abs(math.exp(f(10.0, 10.0)) - 2 * math.exp(10)) < 1e-5 * math.exp(10)
    assert abs(math.exp(f(10.0, 20.0)) - (math.exp(10) + math.exp(20))) < 1e-5 * math.exp(20)
    assert abs(math.exp(f(20.0, 10.0)) - (math.exp(10) + math.exp(20))) < 1e-5 * math.exp(20)
    assert abs(math.exp(f(10.0, ninf)) - math.exp(10)) < 1e-5
    assert abs(math.exp(f(ninf, 10.0)) - math.exp(10)) < 1e-5
    assert abs(f(-718.3947756282423, -8.404216861178751) - (-8.404216861178751)) < 1e-5


def test_ln_a_minus_b_fgbio(L):  # phred.rs:459-477
    f = L.orc_ln_a_minus_b
    q10, q20 = L.orc_phred_to_ln_error_prob(10), L.orc_phred_to_ln_error_prob(20)
    assert f(10.0, 10.0) == float("-inf")
    assert f(q10, q10) == float("-inf")
    assert abs(math.exp(f(q10, q20)) - 0.09) < 1e-5
    assert abs(f(LN(10.0), float("-inf")) - LN(10.0)) < 1e-5


def test_ln_one_minus_exp_fgbio(L):  # phred.rs:480-500, :632-648
    f = L.orc_ln_one_minus_exp
    assert abs(math.exp(f(LN(0.1))) - 0.9) < 1e-5
    assert abs(math.exp(f(LN(0.01))) - 0.99) < 1e-5
    assert abs(math.exp(f(LN(0.90))) - 0.1) < 1e-5
    assert abs(math.exp(f(LN(0.99))) - 0.01) < 1e-5
    assert abs(math.exp(f(float("-inf"))) - 1.0) < 1e-5
    assert f(0.0) == float("-inf") and f(1.0) == float("-inf")
    assert abs(f(LN(0.5)) - LN(0.5)) < 1e-10


def test_phred_conversions_fgbio(L):  # phred.rs:503-530, :588-599
    f = L.orc_ln_prob_to_phred
    assert f(float("-inf")) == 93
    assert f(LN(0.1)) == 10
    assert f(LN(0.5)) == 3
    assert f(0.0) == 2
    assert f(LN(0.9)) == 2
    assert f(LN(1e-15)) == 93


def test_log1pexp_regions(L):  # phred.rs:533-550, :673-689
    f = L.orc_log1pexp
    assert abs(f(-50.0) - math.exp(-50.0)) < 1e-10
    assert abs(f(-37.0) - math.log1p(math.exp(-37.0))) < 1e-10
    assert abs(f(0.0) - LN(2.0)) < 1e-10
    assert abs(f(10.0) - LN(1 + math.exp(10.0))) < 1e-10
    assert abs(f(25.0) - (25.0 + math.exp(-25.0))) < 1e-10
    assert abs(f(40.0) - 40.0) < 1e-10 and abs(f(100.0) - 100.0) < 1e-10
    assert 0.0 < f(-37.0) < 1e-15
    assert abs(f(18.0) - LN(1 + math.exp(18.0))) < 1e-10
    assert abs(f(33.3) - (33.3 + math.exp(-33.3))) < 1e-10


def test_phred_boundaries(L):  # phred.rs:561-585
    assert abs(L.orc_phred_to_ln_error_prob(0)) < 1e-10
    assert abs(math.exp(L.orc_phred_to_ln_error_prob(2)) - 10 ** -0.2) < 1e-6
    assert abs(math.exp(L.orc_phred_to_ln_error_prob(93)) - 10 ** -9.3) < 1e-15
    assert L.orc_phred_to_ln_correct_prob(0) == float("-inf")
    c93 = L.orc_phred_to_ln_correct_prob(93)
    assert c93 < 0 and abs(c93) < 1e-9


def test_two_trials_quick_approximation(L):  # phred.rs:651-670
    big, small = LN(0.5), LN(1e-6)
    assert abs(L.orc_ln_error_prob_two_trials(big, small) - big) < 0.01
    assert abs(L.orc_ln_error_prob_two_trials(small, big) - big) < 0.01


def test_ln_sum_exp_array_edges(L):  # phred.rs:602-620
    assert L.orc_ln_sum_exp_array(None, 0) == float("-inf")
    v = np.array([LN(0.5)])
    assert abs(L.orc_ln_sum_exp_array(v.ctypes.data, 1) - LN(0.5)) < 1e-10
    v = np.array([LN(0.2), LN(0.3)])
    assert abs(L.orc_ln_sum_exp_array(v.ctypes.data, 2) - L.orc_ln_sum_exp(LN(0.2), LN(0.3))) < 1e-10
    v = np.array([float("-inf"), float("-inf")])
    assert L.orc_ln_sum_exp_array(v.ctypes.data, 2) == float("-inf")


# ------------------------------------------------------------------ base_builder.rs:488-788
def test_single_base_perfect():  # base_builder.rs:492-504
    b, q, obs, _ = O.builder_call(45, 40, b"A" * 10, [40] * 10)
    assert b == "A" and q >= 40 and obs.sum() == 10


def test_mixed_bases():  # :507-521
    b, _, obs, _ = O.builder_call(45, 40, b"A" * 8 + b"C" * 2, [30] * 10)
    assert b == "A" and obs.sum() == 10


def test_no_observations():  # :524-531
    b, q, obs, _ = O.builder_call(45, 40, b"", [])
    assert (b, q) == ("N", 2) and obs.sum() == 0


def test_ignore_n_and_case():  # :534-557
    b, _, obs, _ = O.builder_call(45, 40, b"ANA", [40] * 3)
    assert b == "A" and obs.sum() == 2
    b, _, obs, _ = O.builder_call(45, 40, b"aAa", [40] * 3)
    assert b == "A" and obs.sum() == 3


def test_observations_for_base():  # :577-590
    _, _, obs, _ = O.builder_call(45, 40, b"AACG", [40] * 4)
    assert list(obs) == [2, 1, 1, 0]


def test_quality_variation():  # :593-605
    assert O.builder_call(45, 40, b"AAAAAC", [40] * 5 + [10])[0] == "A"


def test_equal_likelihood_no_call():  # :623-638
    assert O.builder_call(93, 93, b"", [])[:2] == ("N", 2)
    assert O.builder_call(93, 93, b"AC", [20, 20])[:2] == ("N", 2)


def test_massive_pileup():  # :642-669
    b, q, obs, _ = O.builder_call(50, 50, b"C" * 1000, [20] * 1000)
    assert (b, q) == ("C", 50) and list(obs) == [0, 1000, 0, 0]
    b, q, obs, _ = O.builder_call(50, 50, b"C" * 1000 + b"T" * 10, [20] * 1010)
    assert (b, q) == ("C", 50) and obs.sum() == 1010 and obs[3] == 10


def test_conflicting_evidence():  # :673-682
    b, q, _, _ = O.builder_call(50, 50, b"AC", [30, 28])
    assert b == "A" and q <= 5
    assert q == 4   # SURVEY Appendix B value


def test_single_observation_q20():  # :686-702
    assert O.builder_call(50, 50, b"A", [20])[:2] == ("A", 20)
    assert O.builder_call(50, 50, b"C", [20])[:2] == ("C", 20)


def test_kahan_order_independence():  # :707-739
    r1 = O.builder_call(45, 40, b"AAAAACCCC", [10, 20, 30, 40, 50, 15, 25, 35, 45])
    r2 = O.builder_call(45, 40, b"ACACACACA", [10, 15, 20, 25, 30, 35, 40, 45, 50])
    assert r1[:2] == r2[:2] and r1[0] == "A"


def test_extreme_quality_range():  # :743-759
    assert O.builder_call(45, 40, b"A" * 100 + b"C" * 10, [2] * 100 + [93] * 10)[0] == "C"


def test_scale_base_qualities_post_umi():  # :766-788, exact values from SURVEY Appendix B
    for qin, qexp in zip((20, 15, 10, 5), (9, 8, 7, 4)):
        _, q, _, _ = O.builder_call(93, 10, b"A", [qin])
        assert q <= qin and q == qexp


def test_appendix_b_vectors():
    """SURVEY.md Appendix B (params 45/40)."""
    assert O.builder_call(45, 40, b"A", [37])[:2] == ("A", 34)
    assert O.builder_call(45, 40, b"AA", [37, 37])[:2] == ("A", 45)
    for n in (3, 4, 8):
        assert O.builder_call(45, 40, b"A" * n, [37] * n)[:2] == ("A", 45)
    assert O.builder_call(45, 40, b"AAAAAAAC", [37] * 8)[:2] == ("A", 45)
    assert O.builder_call(45, 40, b"AAAC", [30] * 4)[:2] == ("A", 44)
    _, _, _, ll = O.builder_call(45, 40, b"A" * 8, [37] * 8)
    assert abs((ll[0] - ll[1]) - 73.69368101330362) < 1e-9
    sq = O.tables(45, 40)[3]
    assert list(sq[:46]) == [2, 2, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 13, 14, 15, 16, 17, 18,
                             19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 33, 34, 35,
                             35, 36, 36, 37, 37, 38, 38, 38]


# ------------------------------------------------------------------ vanilla_caller.rs (column level)
def _simplex(units, pre=45, post=40, min_reads=1, min_cons_q=0):
    batch = pack_source_reads(units, min_reads)
    ob, oq, od, oe, cl = O.simplex_batch(batch, pre, post, min_reads, min_cons_q)
    res = []
    for i, sl in enumerate(batch.unit_slices()):
        assert cl[i] == batch.units["cons_len"][i]
        res.append((bytes(ob[sl]), list(oq[sl]), list(od[sl]), list(oe[sl])))
    return res


def test_single_input_lut_bounds():  # vanilla_caller.rs:2036-2059
    sq = O.tables(45, 40)[3]
    assert len(sq) == 94 and sq[0] <= 2 and sq[60] <= 42


def test_consensus_from_two_reads():  # vanilla_caller.rs:2083-2112
    (b, q, d, e), = _simplex([[(b"GATTACA", bytes([10] * 7))] * 2])
    assert b == b"GATTACA" and all(x > 10 for x in q) and d == [2] * 7 and e == [0] * 7


def test_two_reads_exact_quality():  # vanilla_caller.rs:3462-3517: closed form = 23, +-1
    p = 10 ** (10 / -10.0)
    ok, err = 1 - p, p / 3
    num = ok ** 2
    expected = math.floor(-10 * math.log10(1 - num / (num + 3 * err ** 2)))
    assert expected == 23
    (b, q, _, _), = _simplex([[(b"GATTACA", bytes([10] * 7))] * 2], pre=93, post=93)
    assert b == b"GATTACA" and all(abs(x - expected) <= 1 for x in q)
    assert q == [23] * 7


def test_one_disagreement_lowers_quality():  # vanilla_caller.rs:2117-2152
    q10 = bytes([10] * 7)
    (b, q, d, e), = _simplex([[(b"GATTACA", q10), (b"GATTACA", q10), (b"GATTTCA", q10)]], pre=93)
    assert b == b"GATTACA"
    assert q[4] < q[0] and e[4] == 1 and e[0] == 0 and d == [3] * 7


def test_consensus_length_is_min_reads_th_longest():  # vanilla_caller.rs:2157-2222
    reads = [(b"A" * n, bytes([30] * n)) for n in (10, 8, 6)]
    for m, exp in ((1, 10), (2, 8), (3, 6)):
        (b, q, d, e), = _simplex([reads], min_reads=m)
        assert len(b) == exp
    (b, q, d, e), = _simplex([reads], min_reads=1)
    assert d == [3] * 6 + [2] * 2 + [1] * 2


def test_low_quality_single_read_masked():  # vanilla_caller.rs:2227-2254 (after host masking)
    # host prep turns q < min_input_q into ('N', 2): a single read of those -> (N, 2), depth 0
    (b, q, d, e), = _simplex([[(b"NNNN", bytes([2] * 4))]], min_cons_q=2)
    assert b == b"NNNN" and q == [2] * 4 and d == [0] * 4 and e == [0] * 4


def test_per_read_and_per_base_tags():  # vanilla_caller.rs:2396-2464
    q30 = bytes([30] * 10)
    r4 = bytearray(b"A" * 10)
    r4[5] = ord("C")
    (b, q, d, e), = _simplex([[(b"A" * 10, q30)] * 3 + [(bytes(r4), q30)]], min_cons_q=40)
    assert b == b"A" * 10
    assert max(d) == 4 and min(d) == 4
    assert abs(sum(e) / sum(d) - 0.025) < 0.01
    assert e == [0] * 5 + [1] + [0] * 4


def test_errors_relative_to_consensus():  # vanilla_caller.rs:2473-2515
    q20 = bytes([20] * 8)
    (b, q, d, e), = _simplex([[(b"GATNACAG", q20), (b"GATGACAG", q20), (b"GATGACAG", q20),
                               (b"GATTACAG", q20)]], min_cons_q=0)
    assert b[3:4] == b"G" and len(d) == 8 and d[3] == 3 and e[3] == 1


def test_tie_position_counts_all_as_errors():  # base_builder.rs:433-436 + vanilla_caller.rs:1341
    q30 = bytes([30] * 5)
    (b, q, d, e), = _simplex([[(b"AAAAA", q30), (b"AANAA", q30), (b"AACAA", q30)]], min_cons_q=0)
    # A@30 vs C@30 is an exact tie -> (N, 2); errors = depth - obs['N'] = depth
    assert d == [3, 3, 2, 3, 3] and e == [0, 0, 2, 0, 0] and b == b"AANAA" and q[2] == 2


def test_consensus_ns_when_all_inputs_masked():  # vanilla_caller.rs:2522-2569
    # host masking (min_input_base_quality 30) turns the three Q20 reads into N/Q2 rows
    n7, q2 = b"N" * 7, bytes([2] * 7)
    (b, q, d, e), = _simplex([[(n7, q2), (n7, q2), (n7, q2), (b"CTAATGT", bytes([30] * 7))]],
                             pre=93, post=93, min_reads=1, min_cons_q=40)
    assert b == b"N" * 7 and q == [2] * 7 and d == [1] * 7


def test_all_n_position_depth_zero():  # vanilla_caller.rs:1345-1346: depth 0 < min_reads -> (N, 0)
    q30 = bytes([30] * 3)
    (b, q, d, e), = _simplex([[(b"ANA", q30), (b"ANA", q30)]], min_reads=1, min_cons_q=2)
    assert b == b"ANA" and q[1] == 0 and d[1] == 0


def test_depth_below_min_reads_gives_q0():  # vanilla_caller.rs:1345-1346
    q30 = bytes([30] * 4)
    (b, q, d, e), = _simplex([[(b"ACGT", q30), (b"AC", q30[:2])]], min_reads=2)
    assert len(b) == 2   # consensus_len = 2nd longest
    (b, q, d, e), = _simplex([[(b"ACGT", q30), (b"ANGT", q30)]], min_reads=2)
    assert b[1:2] == b"N" and q[1] == 0 and d[1] == 1


# ------------------------------------------------------------------ duplex_caller.rs:2494-2575
def _duplex(a_bases, a_quals, b_bases, b_quals, source=None):
    L = O.load()
    n = len(a_bases)
    ab = np.frombuffer(a_bases, np.uint8).copy(); bb = np.frombuffer(b_bases, np.uint8).copy()
    aq = np.array(a_quals, np.uint8); bq = np.array(b_quals, np.uint8)
    z = np.zeros(n, np.uint16)
    ob = np.zeros(n, np.uint8); oq = np.zeros(n, np.uint8); oe = np.zeros(n, np.uint16)
    L.orc_duplex_combine(ab.ctypes.data, aq.ctypes.data, z.ctypes.data, z.ctypes.data,
                         bb.ctypes.data, bq.ctypes.data, z.ctypes.data, z.ctypes.data, n, None,
                         None, -1, ob.ctypes.data, oq.ctypes.data, oe.ctypes.data)
    return bytes(ob), list(oq), list(oe)


def test_duplex_agreement_sums_quals():  # duplex_caller.rs:2494-2519
    b, q, _ = _duplex(b"ACGT", [20, 30, 40, 50], b"ACGT", [20, 30, 40, 50])
    assert b == b"ACGT" and q == [40, 60, 80, 93]


def test_duplex_disagreement_takes_higher():  # :2522-2547
    b, q, _ = _duplex(b"ACGT", [30] * 4, b"TGCA", [10, 15, 20, 25])
    assert b == b"ACGT" and q == [20, 15, 10, 5]


def test_duplex_equal_qual_disagreement():  # :2550-2575
    b, q, _ = _duplex(b"ACGT", [30] * 4, b"TGCA", [30] * 4)
    assert b == b"NNNN" and q == [2, 2, 2, 2]


def test_duplex_n_propagation():  # duplex_caller.rs:930-935
    b, q, _ = _duplex(b"ANGT", [30] * 4, b"ACNT", [30] * 4)
    assert b == b"ANNT" and q == [60, 2, 2, 60]


# ------------------------------------------------------------------ codec_caller.rs combine
def _codec(ab, aq, ad, ae, bb, bq, bd, be):
    L = O.load()
    n = len(ab)
    arr8 = lambda x: np.frombuffer(x, np.uint8).copy() if isinstance(x, (bytes, bytearray)) else np.array(x, np.uint8)
    arr16 = lambda x: np.array(x, np.uint16)
    A = [arr8(ab), arr8(aq), arr16(ad), arr16(ae), arr8(bb), arr8(bq), arr16(bd), arr16(be)]
    ob = np.zeros(n, np.uint8); oq = np.zeros(n, np.uint8)
    od = np.zeros(n, np.uint16); oe = np.zeros(n, np.uint16)
    nb, nd = C.c_uint64(), C.c_uint64()
    L.orc_codec_combine(*[x.ctypes.data for x in A], n, ob.ctypes.data, oq.ctypes.data,
                        od.ctypes.data, oe.ctypes.data, C.addressof(nb), C.addressof(nd))
    return bytes(ob), list(oq), list(od), list(oe), nb.value, nd.value


def test_codec_combine_rules():  # codec_caller.rs:1068-1149
    # pos0 agree, pos1 A wins, pos2 B wins, pos3 equal-qual disagreement, pos4 A only (B pad 'n'),
    # pos5 B only with Q2 -> N, pos6 both padding, pos7 uppercase N in A masks
    b, q, d, e, nb, nd = _codec(b"AACAAnnN", [30, 30, 10, 20, 25, 0, 0, 2], [3, 3, 3, 3, 3, 0, 0, 3],
                                [0, 1, 0, 0, 1, 0, 0, 0],
                                b"ACGTnTnA", [40, 10, 30, 20, 0, 2, 0, 30], [2, 2, 2, 2, 0, 2, 0, 2],
                                [0, 0, 1, 0, 0, 0, 0, 0])
    assert b == b"AAGNANNN"
    assert q == [70, 20, 20, 2, 25, 2, 2, 2]
    assert d == [5, 5, 5, 5, 3, 2, 0, 2]
    assert e == [0, 1 + 2, 1 + 3, 0 + 2, 1, 0, 0, 0]
    assert nb == 4 and nd == 3


# ------------------------------------------------------------------ more of duplex_caller.rs
def _duplex_cols(ab, aq, ad, ae, bb, bq, bd, be, n_source=-1):
    """duplex_combine with explicit depth / error columns (approximate error branch by default)."""
    L = O.load()
    n = min(len(ab), len(bb))
    A = [np.frombuffer(ab, np.uint8).copy(), np.array(aq, np.uint8), np.array(ad, np.uint16), np.array(ae, np.uint16)]
    B = [np.frombuffer(bb, np.uint8).copy(), np.array(bq, np.uint8), np.array(bd, np.uint16), np.array(be, np.uint16)]
    ob = np.zeros(n, np.uint8); oq = np.zeros(n, np.uint8); oe = np.zeros(n, np.uint16)
    L.orc_duplex_combine(*[x.ctypes.data for x in A], *[x.ctypes.data for x in B], n, None, None, n_source,
                         ob.ctypes.data, oq.ctypes.data, oe.ctypes.data)
    return bytes(ob), list(oq), list(oe)


def _duplex_arms(ab, aq, ad, ae, bb, bq, bd, be):
    """duplex_consensus(Some/None, Some/None, None): status, bases, quals, errors."""
    L = O.load()
    la, lb = len(ab), len(bb)
    A = [np.frombuffer(ab, np.uint8).copy(), np.array(aq, np.uint8), np.array(ad, np.uint16), np.array(ae, np.uint16)]
    B = [np.frombuffer(bb, np.uint8).copy(), np.array(bq, np.uint8), np.array(bd, np.uint16), np.array(be, np.uint16)]
    cap = max(la, lb, 1)
    ob = np.zeros(cap, np.uint8); oq = np.zeros(cap, np.uint8); oe = np.zeros(cap, np.uint16)
    n = C.c_size_t()
    st = L.orc_duplex_job(*[x.ctypes.data for x in A], la, *[x.ctypes.data for x in B], lb, None, None, 0,
                          ob.ctypes.data, oq.ctypes.data, oe.ctypes.data, C.addressof(n))
    return st, bytes(ob[:n.value]), list(oq[:n.value]), list(oe[:n.value])


def test_duplex_n_bases_and_mixed():                 # :2659-2686, :2968-3001
    b, q, _ = _duplex(b"ANAA", [20] * 4, b"AANA", [20] * 4)
    assert b == b"ANNA" and q[1] == 2 and q[2] == 2
    b, q, _ = _duplex(b"ANGT", [30] * 4, b"TNCG", [25] * 4)
    assert b == b"ANGT" and q == [5, 2, 5, 5]


def test_duplex_quality_capping_and_threshold():     # :2714-2766, :3003-3031
    assert _duplex(b"AAA", [50, 60, 93], b"AAA", [50, 60, 93])[1] == [93, 93, 93]
    b, q, _ = _duplex(b"ACGT", [5, 4, 3, 10], b"TGCA", [3, 2, 2, 8])     # differences of 2, 2, 1, 2 all mask
    assert b == b"NNNN" and q == [2, 2, 2, 2]
    b, q, _ = _duplex(b"AAAA", [25] * 4, b"TTTT", [25] * 4)
    assert b == b"NNNN" and q == [2, 2, 2, 2]
    assert _duplex(b"AAAA", [45] * 4, b"AAAA", [20] * 4)[1] == [65] * 4  # :2768-2808 deep vs shallow strand


def test_duplex_consensus_arms():                    # :4300-4337, :4702-4731, :5112-5173
    # (a strand that is None never reaches the combine here: the host emits the survivor directly;
    #  what the arms function decides is the "no coverage inside the truncated region" rule, :852-882)
    st, b, q, e = _duplex_arms(b"ACGTAC", [30] * 6, [5] * 6, [0] * 6, b"ACGT", [25] * 4, [4] * 4, [0] * 4)
    assert st == 0 and len(b) == 4 and len(q) == 4                       # both: truncated to the shorter strand
    st, b, q, e = _duplex_arms(b"ACGTAC", [30] * 6, [0, 0, 0, 0, 5, 5], [0] * 6, b"TGCA", [25] * 4, [4] * 4, [0] * 4)
    assert st == 2 and b == b"TGCA"                                      # AB has no depth in [0,4): BA only
    st, b, q, e = _duplex_arms(b"AC", [30, 30], [0, 0], [0, 0], b"AC", [30, 30], [5, 5], [0, 0])
    assert st == 2 and b == b"AC" and q == [30, 30]
    st, b, q, e = _duplex_arms(b"ACGT", [30, 31, 32, 33], [5] * 4, [0, 1, 0, 1], b"TTTT", [9] * 4, [0] * 4, [0] * 4)
    assert st == 1 and (b, q, e) == (b"ACGT", [30, 31, 32, 33], [0, 1, 0, 1])   # AB only: passes through whole
    st, b, q, e = _duplex_arms(b"AC", [30, 30], [0, 0], [0, 0], b"AC", [30, 30], [0, 0], [0, 0])
    assert st == 3 and b == b""                                          # neither strand has coverage: None
    st, b, q, e = _duplex_arms(b"NA", [30, 30], [5, 5], [0, 0], b"AN", [30, 30], [5, 5], [0, 0])
    assert st == 0 and b == b"NN"                                        # N in either strand masks


def test_duplex_more_ss_pair_cases():                # :2688-2712, :2768-2803, :3003-3027, :3150-3176
    # length mismatch: the duplex read is as long as the shorter strand
    st, b, q, e = _duplex_arms(b"AAAA", [20] * 4, [3] * 4, [0] * 4, b"AAA", [20] * 3, [2] * 3, [0] * 3)
    assert st == 0 and b == b"AAA" and q == [40, 40, 40]
    # deep coverage on one strand does not change the quality rule: 45 + 20
    b, q, _ = _duplex(b"AAAA", [45] * 4, b"AAAA", [20] * 4)
    assert b == b"AAAA" and q == [65] * 4
    # equal qualities on disagreeing strands: no call, quality 2
    b, q, _ = _duplex(b"AAAA", [25] * 4, b"TTTT", [25] * 4)
    assert b == b"NNNN" and q == [2] * 4
    # an N strand masks the other one, whichever side it is on
    b, q, _ = _duplex(b"NNNN", [2] * 4, b"TTTT", [30] * 4)
    assert b == b"NNNN" and q == [2] * 4
    b, q, _ = _duplex(b"AAAA", [30] * 4, b"NNNN", [2] * 4)
    assert b == b"NNNN" and q == [2] * 4


def test_duplex_error_approximation():               # :4339-4406, :5015-5078
    _, _, e = _duplex_cols(b"ACGT", [30] * 4, [5] * 4, [1, 0, 2, 0], b"ACGT", [25] * 4, [4] * 4, [0, 1, 0, 2])
    assert e == [1, 1, 2, 2]                                             # agreement: errors add
    b, _, e = _duplex_cols(b"AT", [30, 40], [5, 5], [1, 2], b"AC", [25, 30], [4, 4], [0, 1])
    assert b == b"AT" and e[1] == 5                                      # a wins: a_err + (b_depth - b_err)


def test_cap_quality_and_is_error_semantics():       # :4481-4501
    # cap_quality through the combine: sums clamp at 93, differences at 2
    assert _duplex(b"A", [93], b"A", [93])[1] == [93] and _duplex(b"A", [3], b"C", [2])[1] == [2]
    # is_error: N on either side is not an error (exact recount against source rows)
    L = O.load()
    ab = np.frombuffer(b"AN", np.uint8).copy(); q = np.array([30, 30], np.uint8)
    d = np.array([2, 2], np.uint16); z = np.zeros(2, np.uint16)
    rows = [np.frombuffer(b"TN", np.uint8).copy(), np.frombuffer(b"AA", np.uint8).copy()]
    ptrs = (C.c_void_p * 2)(*[r.ctypes.data for r in rows]); lens = (C.c_size_t * 2)(2, 2)
    ob = np.zeros(2, np.uint8); oq = np.zeros(2, np.uint8); oe = np.zeros(2, np.uint16)
    L.orc_duplex_combine(ab.ctypes.data, q.ctypes.data, d.ctypes.data, z.ctypes.data, ab.ctypes.data, q.ctypes.data,
                         d.ctypes.data, z.ctypes.data, 2, ptrs, lens, 2, ob.ctypes.data, oq.ctypes.data, oe.ctypes.data)
    assert list(oe) == [1, 0]        # 'T' vs consensus 'A' counts; source 'N' does not; consensus N counts nothing
