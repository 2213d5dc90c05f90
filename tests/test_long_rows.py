"""Long rows without a GPU: the planner's forms along the length axis, the 65 535-base limit at every entry point
that takes a row, and the record-level host code on long-read families (tests/long_rows.py).

- The ladder of (depth, length) rungs reaches, through `fg.plan_tiles`, every form its rungs claim: shallow-, general-
  and deep-class units voted from HBM because their rows are long, staged regular tiles of one and two units at the
  stage's byte cap, and direct tiles on both sides of the uniform-items hint's 4 096-item edge.
- Planning-only callers (FGB_DEVICE_NONE) plan a 65 535-base read and a 65 535-base CODEC consensus, and refuse one
  base more with FGB_ERR_UNIT_TOO_LARGE; nothing of a refused call stays queued, and the caller keeps working.
- `pack_source_reads` refuses a row of 65 536 bases instead of ORing its length into the offset bits.
- Long-read simplex families through the product's host code over the CPU oracle's vote, against the Python record
  oracle."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import long_rows as LR        # noqa: E402
from tests import oracle_lib as O        # noqa: E402


@pytest.fixture(scope="module")
def ladder(fg):
    return LR.ladder_batch(fg)


def test_ladder_is_derived_from_the_library_limits(fg):
    lib = fg.lib.load()
    cap, max_reads = int(lib.fgb_tile_capacity_bytes()), int(lib.fgb_tile_max_reads())
    assert fg.lib.FGB_MAX_READ_LEN == LR.MAX_READ_LEN == 65535
    _, specs = LR.build(np.random.default_rng(0), LR.ladder(cap, max_reads), cap)
    for s in specs:
        if s["name"].startswith("staged d"):
            d, n = s["depth"], s["lens"][0]
            span = lambda L: LR._r16(s["start"] % 16 + (d - 1) * LR._r8(L) + L)
            assert span(n) <= cap < span(n + 1), s["name"]
    depths = {s["depth"] for s in specs if s["name"].startswith(("staged d", "direct d"))}
    assert depths == set(LR.SHALLOW_DEPTHS + LR.GENERAL_DEPTHS + LR.DEEP_DEPTHS)


def test_ladder_reaches_every_claimed_form(fg, ladder):
    """Each rung lands in the tile form it claims, and the batch as a whole reaches every form the GPU tests rely on."""
    batch, units, specs = ladder
    ut = LR.unit_tiles(fg, batch)
    for u, s in enumerate(specs):
        (cls, direct, regular, hint), t = ut[u]
        assert direct == s["direct"], s["name"]
        assert cls == LR.CLASS_NAMES[1 if s["depth"] <= 4 else 2 if s["depth"] >= 24 else 0], s["name"]
        items = (batch.units["cons_len"][u] + 7) // 8
        if direct:
            assert hint == (2 <= items <= LR.UNIFORM_MAX_ITEMS), s["name"]
        if s["name"].startswith("staged d"):
            assert regular and int(t["n_units"]) == 1, s["name"]
        if s.get("pair"):
            assert regular and int(t["n_units"]) == 2, s["name"]
    want = {(c, True, False, h) for c in ("shallow", "general", "deep") for h in (True, False)}   # direct, +-hint
    want |= {(c, False, True, True) for c in ("shallow", "general", "deep")}                      # staged regular
    want |= {("shallow", False, False, True), ("general", False, False, True)}                   # staged ragged
    assert want <= LR.forms(fg, batch), sorted(want - LR.forms(fg, batch))
    # one-unit staged tiles at the cap hold up to cap / 8 items: ten per voting thread at depth 1
    t = ut[0][1]
    assert int(t["n_units"]) == 1 and (int(batch.units["cons_len"][0]) + 7) // 8 == int(t["byte_len"]) // 8 == 2560


def test_generators_build_what_they_claim(fg, ladder):
    batch, units, specs = ladder
    for u, (s, rows) in enumerate(zip(specs, units)):
        assert [len(b) for b, _ in rows] == s["lens"] and len(rows) == s["depth"], s["name"]
        assert all(len(b) == len(q) for b, q in rows)
        Q = np.concatenate([np.frombuffer(q, np.uint8) for _, q in rows])
        assert 2 <= Q.min() and Q.max() <= 60
        if s["depth"] >= 3 and min(s["lens"]) > s["dissent"][1]:
            B = np.stack([np.frombuffer(b, np.uint8) for b, _ in rows])
            a, e = s["dissent"]
            # share of the reads that disagree with the column's majority
            dis = lambda lo, hi: 1 - np.max([(B[:, lo:hi] == c).sum(0) for c in b"ACGT"], 0).mean() / B.shape[0]
            assert 0.2 < dis(a, e) < 0.35, s["name"]            # dense dissent inside the stretch ...
            assert dis(0, min(a, 2000)) < 0.05, s["name"]       # ... and sparse outside it
    high = [(s, rows) for s, rows in zip(specs, units) if s["name"].startswith("high dissent")]
    assert {s["depth"] for s, _ in high} == {3, 8, 30}
    for s, rows in high:                    # a clean, confident prefix and dense dissent only above position 32 767
        assert s["clean"] == s["dissent"][0] == LR.HIGH_P0 > 32767
        B = np.stack([np.frombuffer(b, np.uint8) for b, _ in rows])
        Q = np.stack([np.frombuffer(q, np.uint8) for _, q in rows])
        assert (B[:, :LR.HIGH_P0] == B[0, :LR.HIGH_P0]).all() and (Q[:, :LR.HIGH_P0] == LR.CLEAN_Q).all()
        assert np.isin(B[0, :LR.HIGH_P0], LR.ACGT).all()
    assert {len(b) for s, rows in zip(specs, units) if s["name"].startswith("limit") for b, _ in rows} == \
        set(range(65528, 65536))
    ragged = [s for s in specs if s["name"].startswith("ragged")]
    assert ragged and all(len(set(s["lens"])) > 1 for s in ragged)
    allb = b"".join(b for rows in units for b, _ in rows)
    for c in b"NacgtnRYKMSWBDHV":
        assert bytes([c]) in allb


def test_pack_source_reads_refuses_rows_past_the_limit(fg):
    rng = np.random.default_rng(3)
    with pytest.raises(ValueError):
        fg.pack_source_reads([[(b"A" * 65536, bytes([30]) * 65536)]], 1)
    with pytest.raises(ValueError):
        fg.pack_source_reads([[(b"A" * 100, bytes([30]) * 100)], [(b"C" * 70000, bytes([30]) * 70000)]], 1)
    rows = LR.long_unit(rng, 2, [65535, 17])
    batch = fg.pack_source_reads([[(b"ACGT" * 4, bytes([30]) * 16)], rows], 1)
    d = batch.reads[:batch.n_reads].astype(np.uint64)
    offs, lens = (d >> np.uint64(16)).tolist(), (d & np.uint64(0xFFFF)).tolist()
    assert lens == [16, 65535, 17] and offs == [0, 16, 16 + 65536]
    for r, (b, q) in zip(range(1, 3), rows):
        assert batch.bases[offs[r]:offs[r] + lens[r]].tobytes() == b
        assert batch.quals[offs[r]:offs[r] + lens[r]].tobytes() == q
    assert int(batch.units["cons_len"][1]) == 65535
    assert len(fg.plan_tiles(batch)) == 2


# ---- the limit through planning-only callers -----------------------------------------------------------------------
def _pending(c):
    p = c.pending()
    return [(u["rows"], u["cons_len"]) for u in p["units"]], p["codec_jobs"].tobytes(), p["n_out"]


def _frag(rng, g, L, rev=False):
    return LR.long_family(rng, g, "frag", 1, (L, L), None, rev)


def test_simplex_planning_at_the_read_length_limit(fg):
    rng = np.random.default_rng(5)
    c = fg.VanillaUmiConsensusCaller("fgumi", "A", fg.VanillaUmiConsensusOptions(min_reads=1), device=fg.lib.FGB_DEVICE_NONE)
    try:
        c.add_group(_frag(rng, 1, 65535))
        c.add_group(_frag(rng, 2, 65535, rev=True))
        before = _pending(c)
        assert [u[1] for u in before[0]] == [65535, 65535]
        # a call whose second group holds a 65 536-base read fails as a whole
        with pytest.raises(fg.lib.FgbError) as e:
            c.add_groups([_frag(rng, 3, 1000), _frag(rng, 4, 65536)])
        assert e.value.status == fg.lib.FGB_ERR_UNIT_TOO_LARGE
        assert _pending(c) == before
        nxt = _frag(rng, 5, 300)
        c.add_group(nxt)
        after = _pending(c)
        assert after[0][:2] == before[0] and len(after[0]) == 3 and after[0][2][1] == 300
    finally:
        c.close()


def _codec_pair(rng, g, cons_len):
    """One CODEC molecule: an FR pair whose reads (each under the limit) span `cons_len` bases together."""
    from tests.test_callers_at_depth import PAD, _pair
    l1 = l2 = min(LR.MAX_READ_LEN, cons_len // 2 + 9000)
    tmpl = LR.ACGT[rng.integers(0, 4, size=2 * PAD + cons_len)].tobytes()
    tags = [(b"MI", "Z", b"%d" % g), (b"RX", "Z", b"ACGTA-CCGTT")]
    return _pair(rng, b"c%d" % g, tmpl, cons_len, l1, l2, False, False, tags)


def test_codec_planning_at_the_consensus_length_limit(fg):
    """A CODEC consensus of 65 535 bases is planned; one of 65 536 fails the call half-way through planning its
    group (after the pair's checks, before its units are queued), and the call rolls back."""
    rng = np.random.default_rng(6)
    c = fg.CodecConsensusCaller("codec", "RG1", device=fg.lib.FGB_DEVICE_NONE)
    try:
        c.add_group(_codec_pair(rng, 1, 65535))
        before = _pending(c)
        assert len(before[0]) == 2 and len(np.frombuffer(before[1], fg.CODEC_JOB_DTYPE)) == 1
        assert int(np.frombuffer(before[1], fg.CODEC_JOB_DTYPE)["len"][0]) == 65535
        with pytest.raises(fg.lib.FgbError) as e:
            c.add_groups([_codec_pair(rng, 2, 40000), _codec_pair(rng, 3, 65536)])
        assert e.value.status == fg.lib.FGB_ERR_UNIT_TOO_LARGE
        assert _pending(c) == before
        c.add_group(_codec_pair(rng, 4, 30000))
        after = _pending(c)
        jobs = np.frombuffer(after[1], fg.CODEC_JOB_DTYPE)
        assert after[0][:2] == before[0] and len(after[0]) == 4 and jobs["len"].tolist() == [65535, 30000]
    finally:
        c.close()


# ---- long-read families through the host code over the CPU oracle's vote ------------------------------------------
def cpu_caller_output(groups, n_threads=4):
    from tests.test_records_input import _cpu_caller
    blob, off, grp = LR.flatten(groups)
    cpu = _cpu_caller(n_threads)
    try:
        p, n, cnt = cpu.process(blob.ctypes.data, off.ctypes.data, grp.ctypes.data, len(groups))
        return C.string_at(p, n), cnt
    finally:
        cpu.close()


def record_oracle_output(groups):
    from oracle import record_oracle as R
    from tests.test_record_oracle_kat import vote_fn
    caller = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(min_reads=1, min_consensus_base_quality=2), vote_fn,
                                   O.builder_call)
    out, count = bytearray(), 0
    for g in groups:
        d, n = caller.consensus_reads(g)
        out += d
        count += n
    return bytes(out), count


def test_long_read_families_through_the_host_code(fg):
    """A subset of the long-read families (every depth up to 64, both strands, overlapping mates): the product's host
    code (prep, mate clip, overlap planning, host assembly) over the CPU oracle's vote equals the record oracle."""
    from tests.test_callers_at_depth import assert_same_stream
    groups = LR.long_families(71, LR.LONG_FAMILIES[:-1])
    got, cnt = cpu_caller_output(groups)
    want, count = record_oracle_output(groups)
    assert cnt == count and count >= len(groups)
    assert_same_stream(got, want)
