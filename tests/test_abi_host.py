"""CPU-only checks of the product's host side: the C-ABI library loads and exports every symbol
include/fgumi_b200.h declares, the host-built tables are bit-identical to the oracle's, the tile
planner honours the layout rules, and compute entry points fail loudly without a GPU (no CPU
fallback).  No compute call is made here."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import __graft_entry__ as graft
from tests import oracle_lib as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fg():
    graft.build()
    import fgumi_b200
    return fgumi_b200


def test_header_symbols_exported_abi_v4(fg):
    """The library exports exactly the header's symbols, and reports ABI version 4 (the version without the one-shot
    fgb_duplex_submit / fgb_codec_submit)."""
    hdr = open(os.path.join(ROOT, "include", "fgumi_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(fgb_[a-z_0-9]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = fg.lib.load()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert declared == set(fg.lib.SYMBOLS)
    assert lib.fgb_abi_version() == 4


def test_struct_sizes_match_header(fg):
    l = fg.lib
    assert C.sizeof(l.FgbUnit) == 16 and C.sizeof(l.FgbTile) == 32
    assert C.sizeof(l.FgbParams) == 8
    assert C.sizeof(l.FgbDuplexJob) == 16 and C.sizeof(l.FgbCodecJob) == 32
    assert C.sizeof(l.FgbCodecParams) == 24
    lib = l.load()
    for i, t in enumerate((l.FgbCallerOptions, l.FgbFilterParams, l.FgbSubmitOptions, l.FgbRawColumns,
                           None, l.FgbBatch, l.FgbCodecParams, l.FgbParams, l.FgbDuplexFilterParams,
                           l.FgbRecordColumns)):
        if t is not None:
            assert lib.fgb_struct_size(i) == C.sizeof(t), (i, t)
    assert lib.fgb_struct_size(4) == 16 and lib.fgb_struct_size(99) == 0


@pytest.mark.parametrize("pre,post", [(45, 40), (50, 50), (93, 93), (93, 10), (30, 20), (10, 45)])
def test_host_tables_bit_identical_to_oracle(fg, pre, post):
    lib = fg.lib.load()
    c = np.zeros(94); e = np.zeros(94); lp = C.c_double(); sq = np.zeros(94, np.uint8)
    qt = np.zeros(256, np.uint8); fq = C.c_uint32()
    st = lib.fgb_host_tables(pre, post, c.ctypes.data, e.ctypes.data, C.addressof(lp),
                             sq.ctypes.data, qt.ctypes.data, C.addressof(fq))
    assert st == 0
    oc, oe, olp, osq = O.tables(pre, post)
    assert c.tobytes() == oc.tobytes() and e.tobytes() == oe.tobytes()
    assert lp.value == olp and np.array_equal(sq, osq)
    assert fq.value == O.load().orc_ln_prob_to_phred(olp)
    # the SWAR proof table: n identical observations at quality >= qt[n] are PROVEN to come out
    # of the reference's call() as (base, phred(ln_pre))
    for n in (1, 2, 3, 4, 8, 100, 254, 255):
        if qt[n] <= 93:
            for q in {int(qt[n]), min(93, int(qt[n]) + 1), 93}:
                b, qq, _, ll = O.builder_call(pre, post, b"A" * n, [q] * n)
                assert (b, qq) == ("A", fq.value), (n, q)
    assert qt[0] == 255


def test_fast_path_threshold_defaults(fg):
    lib = fg.lib.load()
    qt = np.zeros(256, np.uint8)
    lib.fgb_host_tables(45, 40, None, None, None, None, qt.ctypes.data, None)
    assert qt[0] == 255 and qt[1] == 255      # one observation can never dominate
    assert qt[2] <= 40                        # two Q37+ observations are enough (SURVEY App. B)
    assert qt[8] <= 10           # depth 8: every unmasked base (q >= 10) qualifies
    assert qt[3] <= 31


def _proof(fg, pre, post):
    lib = fg.lib.load()
    dfix = np.zeros(96, np.int32); g2 = C.c_int32(); nmax = C.c_uint32()
    assert lib.fgb_host_proof_tables(pre, post, dfix.ctypes.data, C.addressof(g2), C.addressof(nmax)) == 0
    return dfix, g2.value, nmax.value


@pytest.mark.parametrize("pre,post", [(45, 40), (50, 50), (30, 20), (60, 60), (93, 93), (20, 45)])
def test_dominant_winner_proof_against_oracle(fg, pre, post):
    """Whenever the integer proof fires, the oracle's literal f64 call() must return
    (winner, phred(ln_pre)).  Random pileups near the decision boundary."""
    dfix, g2fix, nmax2 = _proof(fg, pre, post)
    fq = O.load().orc_ln_prob_to_phred(O.tables(pre, post)[2])
    rng = np.random.default_rng(pre * 100 + post)
    fired = 0
    INT_MIN = np.iinfo(np.int32).min
    assert dfix[0] == INT_MIN          # quality 0 has correct[0] = -inf: never usable
    for trial in range(6000):
        n = int(rng.integers(1, 14))
        if n > nmax2:
            continue
        nalt = int(rng.integers(0, max(1, n // 2) + 1))
        qs = rng.integers(1, 60, size=n)
        bs = np.array([ord("G")] * (n - nalt) + list(rng.choice([65, 67, 84], size=nalt)), np.uint8)
        perm = rng.permutation(n)
        bs, qs = bs[perm], qs[perm]
        S = {65: 0, 67: 0, 71: 0, 84: 0}
        cnt = {65: 0, 67: 0, 71: 0, 84: 0}
        for b, q in zip(bs, qs):
            S[int(b)] += int(dfix[min(int(q), 93)]); cnt[int(b)] += 1
        order = sorted(S.items(), key=lambda kv: -kv[1])
        gap = order[0][1] - order[1][1]
        if gap >= g2fix + 2 * n + 1:
            fired += 1
            b, q, obs, _ = O.builder_call(pre, post, bs.tobytes(), [int(x) for x in qs])
            assert (ord(b), q) == (order[0][0], fq), (trial, bs, qs, gap, g2fix)
    if nmax2 >= 13:
        assert fired > 200


@pytest.mark.parametrize("pre,post", [(45, 40), (30, 30), (93, 93), (20, 45), (60, 10), (45, 93)])
def test_unanimous_step_table_against_oracle(fg, pre, post):
    """The step table of the shallow kernel (quality of a unanimous pileup by its fixed-point likelihood gap): wherever
    the kernel's acceptance rule lets the table answer, the oracle's literal add / call sequence gives that quality."""
    lib = fg.lib.load()
    bp = np.zeros(128, np.int32); qv = np.zeros(128, np.uint8)
    n, guard = C.c_uint32(), C.c_int32()
    assert lib.fgb_host_unanimous_steps(pre, post, bp.ctypes.data, qv.ctypes.data, C.addressof(n), C.addressof(guard)) == 0
    n, guard = n.value, guard.value
    assert 0 < n < 127 and guard >= 64
    assert np.all(np.diff(bp[:n].astype(np.int64)) > 0) and np.all(np.diff(qv[:n].astype(np.int64)) > 0)
    assert np.all(bp[n:] == np.iinfo(np.int32).max)
    dfix, g2fix, nmax2 = _proof(fg, pre, post)
    rng = np.random.default_rng(1000 * pre + post)
    answered = 0
    trials = 0
    for depth in (1, 2, 3, 4):
        for _ in range(2500):
            # low and middling qualities: the gaps the table exists for (below the fast path's 23 nats)
            qs = rng.integers(1, 50, size=depth)
            g = int(sum(int(dfix[q]) for q in qs))
            e = 2 * depth + 1
            if g <= e + 64 or g + e >= 23 * 65536:
                continue
            trials += depth > 1      # one observation of quality q sits right at the start of "its" step: those go literal
            lo, hi = g - e - guard, g + e + guard
            k = int(np.searchsorted(bp[:n], lo, side="right")) - 1
            if k < 0 or bp[k + 1] <= hi:
                continue                       # the kernel would evaluate this one literally
            answered += depth > 1
            b, q, obs, _ = O.builder_call(pre, post, b"G" * depth, [int(x) for x in qs])
            assert (b, q) == ("G", int(qv[k])), (depth, qs, g, k, bp[k], bp[k + 1])
    assert answered > 0.8 * trials > 0


def test_create_without_gpu_fails_loudly(fg):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(fg.lib.FgbError) as ei:
        fg.Engine(device=0)
    assert ei.value.status == fg.lib.FGB_ERR_NO_DEVICE


def _plan(fg, units, min_reads=1):
    b = fg.pack_source_reads(units, min_reads)
    return b, fg.plan_tiles(b)


def test_planner_small_and_empty(fg):
    b, tiles = _plan(fg, [])
    assert len(tiles) == 0
    rows = [(b"ACGT" * 10, bytes([30] * 40))] * 3
    b, tiles = _plan(fg, [rows, rows])
    assert len(tiles) == 1
    t = tiles[0]
    assert t["n_units"] == 2 and t["n_reads"] == 6 and t["byte_begin"] == 0
    assert t["byte_len"] % 16 == 0 and t["byte_len"] >= 6 * 40
    assert t["flags"] >> 8 == 5           # uniform tile: 40-base rows -> 5 eight-position items per unit
    b, tiles = _plan(fg, [rows, rows[:2] + [(b"ACGT" * 5, bytes([30] * 20))]], min_reads=3)
    assert tiles[0]["flags"] >> 8 == 0    # mixed consensus lengths: no hint


def test_planner_splits_on_capacity(fg):
    cap = fg.lib.load().fgb_tile_capacity_bytes()
    L = 152
    rows = [(b"A" * L, bytes([30] * L))] * 8
    n_units = 3 * (cap // (8 * L)) + 1
    b, tiles = _plan(fg, [rows] * n_units)
    assert tiles["n_units"].sum() == n_units and tiles["n_reads"].sum() == 8 * n_units
    assert (tiles["byte_len"] <= cap).all() and (tiles["byte_begin"] % 16 == 0).all()
    assert len(tiles) == 4
    # tiles are contiguous in unit order
    assert np.array_equal(tiles["unit_begin"][1:], np.cumsum(tiles["n_units"])[:-1])


def test_planner_flags_oversize_unit_direct(fg):
    cap = fg.lib.load().fgb_tile_capacity_bytes()
    big = [(b"C" * 200, bytes([30] * 200))] * (cap // 200 + 5)
    small = [(b"A" * 20, bytes([30] * 20))] * 2
    b, tiles = _plan(fg, [small, big, small])
    assert len(tiles) == 3
    assert list(tiles["flags"] & 1) == [0, 1, 0]
    many = [(b"A" * 4, bytes([30] * 4))] * (fg.lib.load().fgb_tile_max_reads() + 1)
    b, tiles = _plan(fg, [many])
    assert list(tiles["flags"] & 1) == [1]


def test_planner_rejects_bad_layout(fg):
    lib = fg.lib.load()
    b = fg.pack_source_reads([[(b"ACGTA", bytes([30] * 5))] * 2], 1)
    n = C.c_uint64()

    def plan(batch):
        return lib.fgb_plan_tiles(batch.units.ctypes.data, batch.n_units, batch.reads.ctypes.data,
                                  batch.n_reads, None, 0, C.byref(n))
    assert plan(b) == 0
    bad = fg.pack_source_reads([[(b"ACGTA", bytes([30] * 5))] * 2], 1)
    bad.reads[1] = ((int(bad.reads[1]) >> 16) + 4) << 16 | 5      # misaligned row
    assert plan(bad) == fg.lib.FGB_ERR_LAYOUT
    bad = fg.pack_source_reads([[(b"ACGTA", bytes([30] * 5))] * 2], 1)
    bad.units["out_off"][1] += 8                                   # output rows not dense
    assert plan(bad) == fg.lib.FGB_ERR_LAYOUT
    bad = fg.pack_source_reads([[(b"ACGTA", bytes([30] * 5))] * 2], 1)
    bad.units["cons_len"][0] = 9                                   # longer than any read
    bad.units["out_off"][1] = 16
    assert plan(bad) == fg.lib.FGB_ERR_LAYOUT


def test_consensus_length_rule(fg):
    assert fg.consensus_length([10, 8, 6], 1) == 10
    assert fg.consensus_length([6, 10, 8], 2) == 8
    assert fg.consensus_length([6, 10, 8], 3) == 6


def test_pack8_encode_alphabet(fg):
    """PACK8 host encoder: A,C,G,T with q <= 61, (N, 2) and zero padding encode; anything else is
    reported as not encodable."""
    b = np.frombuffer(b"ACGTN\0", np.uint8).copy()
    q = np.array([0, 61, 30, 7, 2, 0], np.uint8)
    p = fg.pack8_encode(b, q)
    assert p.tolist() == [0, (1 << 6) | 61, (2 << 6) | 30, (3 << 6) | 7, 0x3E, 0]
    for bad_b, bad_q in ((b"a", 30), (b"R", 30), (b"N", 10), (b"A", 62), (b"\0", 1)):
        assert fg.pack8_encode(np.frombuffer(bad_b, np.uint8).copy(), np.array([bad_q], np.uint8)) is None


def _brute_force_hints(batch, t):
    """What the tile hint bits must say, straight from their definitions (fgb_config.h)."""
    u0, nu = int(t["unit_begin"]), int(t["n_units"])
    units, reads = batch.units, batch.reads
    lens, offs, per_unit = [], [], []
    for u in range(u0, u0 + nu):
        rb, re = int(units["read_begin"][u]), int(units["read_begin"][u + 1])
        per_unit.append(re - rb)
        for r in range(rb, re):
            lens.append(int(reads[r]) & 0xFFFF)
            offs.append(int(reads[r]) >> 16)
    cons = [int(units["cons_len"][u]) for u in range(u0, u0 + nu)]
    items = {(c + 7) // 8 for c in cons}
    uniform = len(items) == 1 and 2 <= next(iter(items)) <= 4096
    regular = False
    if lens and uniform and all(n > 0 for n in per_unit):
        L = lens[0]
        stride = (L + 7) // 8 * 8
        regular = (all(x == L for x in lens) and all(c == L for c in cons) and
                   all(o == offs[0] + i * stride for i, o in enumerate(offs)))
    shallow = max(per_unit) <= 64
    return uniform, regular, shallow, (offs[0] != int(t["byte_begin"])) if lens else False


def test_planner_hint_bits_match_their_definitions(fg):
    """Property test: on random layouts (uniform, ragged, gapped, deep) every hint bit the planner sets
    -- regular, first-row skew, shallow, uniform items -- equals its brute-force definition, and the
    tiles cover every unit exactly once within the capacity limits."""
    lib = fg.lib.load()
    cap, max_u, max_r = lib.fgb_tile_capacity_bytes(), lib.fgb_tile_max_units(), lib.fgb_tile_max_reads()
    rng = np.random.default_rng(77)
    seen = {"regular": 0, "irregular": 0, "skew": 0, "deep": 0}
    for trial in range(120):
        style = trial % 4
        units = []
        for _ in range(int(rng.integers(1, 260))):
            if style == 0:                       # one length everywhere
                L, depth = 150, int(rng.integers(1, 12))
                rows = [(b"A" * L, bytes([30] * L))] * depth
            elif style == 1:                     # ragged
                depth = int(rng.integers(1, 10))
                rows = [(b"C" * n, bytes([30] * n)) for n in rng.integers(1, 90, size=depth)]
            elif style == 2:                     # uniform length but an occasional short read
                L, depth = int(rng.integers(9, 60)), int(rng.integers(1, 6))
                rows = [(b"G" * L, bytes([30] * L))] * depth
                if rng.random() < 0.05:
                    rows = rows + [(b"G" * (L - 1), bytes([30] * (L - 1)))]
            else:                                # deep units
                L, depth = 40, int(rng.integers(1, 130))
                rows = [(b"T" * L, bytes([30] * L))] * depth
            units.append(rows)
        batch = fg.pack_source_reads(units, 1)
        tiles = fg.plan_tiles(batch)
        assert int(tiles["n_units"].sum()) == batch.n_units
        assert np.array_equal(tiles["unit_begin"], np.concatenate([[0], np.cumsum(tiles["n_units"])[:-1]]))
        for t in tiles:
            fl = int(t["flags"])
            direct = fl & 1
            if not direct:
                assert t["byte_len"] <= cap and t["n_units"] <= max_u and t["n_reads"] + (int(t["read_begin"]) & 1) <= max_r
            uniform, regular, shallow, skew = _brute_force_hints(batch, t)
            assert ((fl >> 8) != 0) == uniform, (trial, fl)
            if not direct:
                assert bool(fl & 2) == regular, (trial, fl)
                assert bool(fl & 8) == shallow, (trial, fl)
                if regular:
                    assert bool(fl & 4) == skew, (trial, fl)
                    seen["skew"] += skew
                seen["regular" if regular else "irregular"] += 1
                seen["deep"] += not shallow
    assert all(v > 0 for v in seen.values()), seen
