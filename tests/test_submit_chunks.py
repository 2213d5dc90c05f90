"""The chunk cuts of the host-buffer submit, without a GPU: the generators of tests/submit_chunks.py build what they
claim, and at the chunk sizes tests/test_submit_chunks_gpu.py runs them with, their cuts reach every case a one-chunk
batch never does -- a chunk that opens on a direct tile, on an odd read, on a tile larger than the chunk size, a chunk
of mixed tile classes, a last chunk whose 16-byte-aligned end lies past `n_bytes`, and BAM4 chunks whose first span
starts at each even offset modulo 32."""
import numpy as np
import pytest

from tests import oracle_lib as O
from tests import submit_chunks as SC

MB = SC.MB


@pytest.fixture(scope="module")
def mixed(fg):
    batch = fg.pack_source_reads(SC.mixed_units(11), 2)
    fg.plan_tiles(batch)
    return batch


@pytest.fixture(scope="module")
def bam4(fg):
    return SC.bam4_batch(fg, 5, MB)


def test_cuts_partition_the_batch(fg, mixed):
    for chunk in (1 * MB, 3 * MB, SC.default_chunk_bytes(mixed.n_bytes)):
        cs = SC.cuts(mixed, chunk)
        assert cs[0]["t0"] == 0 and cs[-1]["t1"] == len(mixed.tiles)
        assert cs[0]["u0"] == 0 and cs[-1]["u1"] == mixed.n_units and cs[-1]["o1"] == mixed.n_out
        for a, b in zip(cs, cs[1:]):
            assert a["t1"] == b["t0"] and a["u1"] == b["u0"] and a["r1"] == b["rf"] and a["o1"] == b["o0"]
        for c in cs:
            assert c["byte0"] % 16 == 0 and c["r0"] % 2 == 0
            assert c["byte1"] - c["byte0"] <= chunk or c["t1"] == c["t0"] + 1
    assert len(SC.cuts(mixed, SC.default_chunk_bytes(mixed.n_bytes))) == 1
    assert len(SC.cuts(mixed, 1 * MB, one_piece=True)) == 1


def test_mixed_batch_reaches_every_chunk_case(fg, mixed):
    T = mixed.tiles
    classes = {int(f >> SC.CLASS_SHIFT) & 3 for f in T["flags"]}
    assert classes == {0, 1, 2}
    direct = T[(T["flags"] & SC.DIRECT) != 0]
    assert {int(f >> SC.CLASS_SHIFT) & 3 for f in direct["flags"]} == {0, 1, 2}
    cl = mixed.units["cons_len"][: mixed.n_units]
    depth = np.diff(mixed.units["read_begin"].astype(np.int64))
    assert ((depth == 1) & (cl == 0)).any()                  # units below min_reads call nothing
    assert mixed.n_bytes % 16 == 8
    assert fg.pack8_encode(mixed.bases, mixed.quals) is not None
    assert (mixed.bases == ord("N")).any() and set(np.unique(mixed.quals[mixed.bases == ord("N")])) == {2}
    assert mixed.quals.max() == 61
    for chunk in (1 * MB, 3 * MB):
        cs = SC.cuts(mixed, chunk)
        assert len(cs) >= (6 if chunk == MB else 3)
        assert any(c["direct_first"] for c in cs[1:])
        assert any(c["rf"] % 2 == 1 for c in cs[1:])
        assert any(len(c["classes"]) > 1 for c in cs)
        assert cs[-1]["byte1"] > mixed.n_bytes
        assert any(c["tile_bytes"] > chunk and c["t0"] > 0 for c in cs)


def test_two_column_variant_needs_the_byte_columns(fg):
    batch = fg.pack_source_reads(SC.mixed_units(12, qmax=93), 2)
    assert batch.quals.max() == 93
    assert fg.pack8_encode(batch.bases, batch.quals) is None
    fg.plan_tiles(batch)
    assert len(SC.cuts(batch, MB)) >= 6


def test_bam4_batch_spans(fg, bam4):
    layout, raw, spans = bam4
    rows = SC.expected_rows(spans, raw.min_input_base_quality)
    rr = raw.raw_reads[: layout.n_reads]
    src, rl = rr["src_off"].astype(np.int64), rr["raw_len"].astype(np.int64)
    assert (src % 2 == 0).all() and (src[1:] >= src[:-1] + rl[:-1]).all()
    assert (src[1:] > src[:-1] + rl[:-1]).any()                                    # gaps between spans
    assert set((src % 32).tolist()) == set(range(0, 32, 2))
    assert (rl % 2 == 1).any() and (rl % 2 == 0).any()
    assert (rr["flags"] == 1).any() and (rr["flags"] == 0).any()
    row_len = (layout.reads[: layout.n_reads] & np.uint64(0xFFFF)).astype(np.int64)
    assert (row_len < rl).any() and (row_len <= rl).all()
    assert raw.quals_raw.max() == 255 and src[-1] + rl[-1] == raw.n_raw
    assert [len(u) for u in rows] == np.diff(layout.units["read_begin"].astype(np.int64)).tolist()
    cs = SC.cuts(layout, MB, raw_reads=raw.raw_reads)
    assert len(cs) >= 16
    assert {c["first_src_off"] % 32 for c in cs} == set(range(0, 32, 2))
    for c in cs:
        assert c["raw_lo"] <= c["first_src_off"] and c["raw_hi"] <= raw.n_raw
        inside = (src[c["rf"]:c["r1"]] >= c["raw_lo"]) & (src[c["rf"]:c["r1"]] + rl[c["rf"]:c["r1"]] <= c["raw_hi"])
        assert inside.all()
    assert any(c["rf"] % 2 == 1 for c in cs[1:]) and any(len(c["classes"]) > 1 for c in cs)
    assert len(SC.cuts(layout, SC.default_chunk_bytes(layout.n_bytes))) == 1


@pytest.mark.parametrize("min_q", [0, 10, 200])
def test_bam4_expected_rows_follow_create_source_read(fg, bam4, min_q):
    """The expected rows against a per-base restatement on a few reads of each strand: decode, orient, mask."""
    layout, raw, spans = bam4
    rows = SC.expected_rows(spans, min_q)
    code = np.frombuffer(SC.NIBBLE_CODES, np.uint8)
    comp = dict(zip(SC.NIBBLE_CODES, SC.COMPLEMENT))
    flat = [r for u in rows for r in u]
    for r in list(range(40)) + list(range(layout.n_reads - 40, layout.n_reads)):
        s, n, rev = int(raw.raw_reads[r]["src_off"]), int(raw.raw_reads[r]["raw_len"]), raw.raw_reads[r]["flags"] & 1
        ln = int(layout.reads[r]) & 0xFFFF
        bases, quals = bytearray(), bytearray()
        for p in range(ln):
            i = s + (n - 1 - p if rev else p)
            nib = (raw.seq4[i >> 1] >> 4) if i % 2 == 0 else raw.seq4[i >> 1] & 15
            b = int(code[nib])
            q = int(raw.quals_raw[i])
            b = comp[b] if rev else b
            if q < min_q:
                b, q = ord("N"), 2
            bases.append(b)
            quals.append(q)
        assert flat[r] == (bytes(bases), bytes(quals)), r
    if min_q == 200:
        assert sum(r[0].count(b"N") for r in flat) > 0.7 * sum(len(r[0]) for r in flat)


def test_bench_shape_cuts_into_about_eight_chunks(fg):
    """At the benchmark's shape the default rule cuts ~30 MB chunks; the GPU test's 200 k units give eight."""
    from fgumi_b200 import synth
    layout = synth.make_descriptors(np.full(200_000, 8), 150, 1)
    chunk = SC.default_chunk_bytes(layout.n_bytes)
    assert 24 * MB < chunk < 32 * MB
    cs = SC.cuts(layout, chunk)
    assert 8 <= len(cs) <= 9
    assert len(SC.boundary_units(layout, cs)) >= 16 * (len(cs) - 1)


@pytest.mark.parametrize("seed,qmax", [(11, 61), (12, 93)])
def test_filter_params_reach_every_status(fg, seed, qmax):
    """The filter thresholds of the GPU test give every status on the oracle's columns of both mixed batches."""
    batch = fg.pack_source_reads(SC.mixed_units(seed, qmax=qmax), 2)
    cols = O.simplex_batch(batch, 45, 40, 2, 2, 8)[:4]
    st = SC.filter_statuses(batch, cols, SC.FILTER)
    assert set(st.tolist()) == {0, 1, 2, 3, 4, 255}
