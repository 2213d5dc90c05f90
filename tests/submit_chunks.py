"""Where the host-buffer submit cuts a batch into chunks, and seeded batches whose cuts land where chunks go wrong.

`fgb_submit`, `fgb_submit_pack8`, `fgb_submit_bam4` and `fgb_submit_ex` (`submit_impl`, csrc/capi.cu) cut a batch at
tile boundaries into chunks of at most `chunk_bytes` bytes per column (a tile larger than that is a chunk of its own)
and rotate the chunks over the handle's slot streams.  Every chunk biases the descriptor pointers by its own origin
(`byte0` / `r0` / `u0` / `o0`), uploads only its own part of the columns and copies back only its own output rows, so a
batch that fits one chunk never exercises any of that.  The helpers here:

  cuts              the chunk loop of `submit_impl`, restated: per chunk the tile range, byte range, unit / read /
                    output ranges and, for BAM4 input, the raw range that is resident on the device
  mixed_units       units of all three tile classes interleaved with long units voted from HBM (the direct rungs of
                    tests/long_rows.py), one unit larger than a 3 MB chunk, units below min_reads, masked (N, Q2)
                    bases; qualities 0-61 (PACK8-encodable) or, for the two-column variant, 0-93
  bam4_batch        a BAM4 batch with its own packer: spans at every even offset modulo 32 with gaps between them,
                    reverse-strand reads, odd raw lengths, rows shorter than their span, raw qualities up to 255; the
                    reads that open the chunks of a given chunk size start at each of the 16 even offsets in turn
  bench_batch       the benchmark's shape (depth 8, 150 bp), built vectorised
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

MB = 1 << 20
CHUNK_DEFAULT = 96 * MB          # kChunkColumnBytes
CHUNK_FLOOR = 24 * MB            # the default rule never goes below this
DIRECT = 1                       # kTileFlagDirect
CLASS_SHIFT = 4                  # kTileClassShift
ACGT = np.frombuffer(b"ACGT", np.uint8)
NIBBLE_CODES = b"=ACMGRSVTWYHKDBN"
COMPLEMENT = b"=TGMCRSVAWYHKDBN"
BAM4_UNITS = 10000               # ~17 MB of rows: at 1 MB chunks, more than 16 chunks
# filter thresholds under which the mixed batch's units reach every status (FGB_FILTER_*)
FILTER = dict(min_reads=3, min_base_quality=20, max_read_error_rate=0.02, max_base_error_rate=0.3,
              min_mean_base_quality=45.0, max_no_call_fraction=0.1, per_base_tags=1)


def default_chunk_bytes(n_bytes: int) -> int:
    """Per-column chunk size when FGB_SUBMIT_CHUNK_MB is not set."""
    return min(CHUNK_DEFAULT, max(CHUNK_FLOOR, n_bytes // 8))


def _r8(n: int) -> int:
    return (n + 7) // 8 * 8


def tile_ends(batch) -> np.ndarray:
    """Exclusive end of every tile's byte range as the chunk loop sees it (a direct tile: its last row, 16-aligned)."""
    T = batch.tiles
    ends = T["byte_begin"].astype(np.int64) + T["byte_len"].astype(np.int64)
    direct = (T["flags"] & DIRECT) != 0
    if direct.any():
        last = batch.reads[(T["read_begin"][direct] + T["n_reads"][direct] - 1).astype(np.int64)]
        ends[direct] = (((last >> np.uint64(16)) + (last & np.uint64(0xFFFF)) + np.uint64(15))
                        & ~np.uint64(15)).astype(np.int64)
    return ends


def tile_starts(batch) -> np.ndarray:
    """Where a chunk that opens on the tile starts (`byte0`): a direct tile starts at its first row, 16-aligned."""
    T = batch.tiles
    starts = T["byte_begin"].astype(np.int64)
    direct = (T["flags"] & DIRECT) != 0
    if direct.any():
        first = batch.reads[T["read_begin"][direct].astype(np.int64)]
        starts[direct] = ((first >> np.uint64(16)) & ~np.uint64(15)).astype(np.int64)
    return starts


def cuts(batch, chunk_bytes: int, one_piece: bool = False, raw_reads: Optional[np.ndarray] = None) -> List[Dict]:
    """The chunks `submit_impl` makes of `batch` (tiles planned) at `chunk_bytes` per column.  With `raw_reads` (the
    BAM4 fgb_raw_read table) each chunk also carries the raw range [raw_lo, raw_hi) it uploads."""
    T = batch.tiles
    n = len(T)
    ends, starts = tile_ends(batch), tile_starts(batch)
    out = []
    t0 = 0
    while t0 < n:
        byte0 = int(starts[t0])
        byte1 = byte0
        t1 = t0
        while t1 < n:
            end = max(int(ends[t1]), byte1)
            if not one_piece and t1 > t0 and end - byte0 > chunk_bytes:
                break
            byte1 = end
            t1 += 1
        first, last = T[t0], T[t1 - 1]
        u0, u1 = int(first["unit_begin"]), int(last["unit_begin"]) + int(last["n_units"])
        rf = int(first["read_begin"])
        r1 = int(last["read_begin"]) + int(last["n_reads"])
        c = dict(t0=t0, t1=t1, byte0=byte0, byte1=byte1, u0=u0, u1=u1, r0=rf & ~1, rf=rf, r1=r1,
                 o0=int(batch.units["out_off"][u0]), o1=int(batch.units["out_off"][u1]),
                 valid_bytes=min(byte1, batch.n_bytes) - min(byte0, batch.n_bytes),
                 classes=sorted({int(f >> CLASS_SHIFT) & 3 for f in T["flags"][t0:t1]}),
                 direct_first=bool(first["flags"] & DIRECT), tile_bytes=int(ends[t0]) - byte0)
        if raw_reads is not None and r1 > rf:
            c["first_src_off"] = int(raw_reads["src_off"][rf])
            c["raw_lo"] = c["first_src_off"] & ~31
            c["raw_hi"] = int(raw_reads["src_off"][r1 - 1]) + int(raw_reads["raw_len"][r1 - 1])
        out.append(c)
        t0 = t1
    return out


# ---- the mixed batch ----------------------------------------------------------------------------------------------
def _rows(rng, depth: int, L: int, qmax: int, ragged: bool) -> List[Tuple[bytes, bytes]]:
    """`depth` rows over one template: ~2 % substitutions, ~3 % masked (N, Q2) bases, qualities 0..qmax."""
    tmpl = ACGT[rng.integers(0, 4, size=L)]
    rows = []
    for _ in range(depth):
        ln = int(rng.integers(max(1, L - 12), L + 1)) if ragged else L
        b = tmpl[:ln].copy()
        sub = rng.random(ln) < 0.02
        b[sub] = ACGT[rng.integers(0, 4, size=int(sub.sum()))]
        q = rng.integers(0, qmax + 1, size=ln).astype(np.uint8)
        m = rng.random(ln) < 0.03
        b[m] = ord("N")
        q[m] = 2
        rows.append((b.tobytes(), q.tobytes()))
    return rows


def mixed_units(seed: int, n_regular: int = 3000, qmax: int = 61, big: Optional[Tuple[int, int]] = (50, 65535)
                ) -> List[List[Tuple[bytes, bytes]]]:
    """Shallow (1-4 reads), general (5-23) and deep (24-40) units interleaved, rows of 1-300 bases; after every
    ~250 of them a unit just too long for one stage (the `direct` rungs of tests/long_rows.py at depths 1, 3, 8 and
    30, one per class), and in the middle one unit of `big` = (depth, length), larger than a 3 MB chunk, whose
    first read has an odd index.  With
    min_reads 2 the one-read units call nothing (cons_len 0).  The batch's byte count is an odd multiple of 8, so the
    last tile's 16-byte-aligned end lies past it."""
    from tests import long_rows as LR
    from fgumi_b200 import lib as _l
    cap = int(_l.load().fgb_tile_capacity_bytes())
    rng = np.random.default_rng(seed)
    units: List[List[Tuple[bytes, bytes]]] = []
    off = 0
    rungs = (1, 3, 8, 30)

    def add(rows):
        nonlocal off
        units.append(rows)
        off += sum(_r8(len(b)) for b, _ in rows)

    for i in range(n_regular):
        if i % 250 == 125:
            d = rungs[(i // 250) % len(rungs)]
            add(_rows(rng, d, LR.longest_staged(d, cap, off) + 1, qmax, ragged=False))
        if big and i == n_regular // 2:            # it opens a chunk of its own, on an odd read
            if sum(len(u) for u in units) % 2 == 0:
                add(_rows(rng, 1, 40, qmax, False))
            add(_rows(rng, big[0], big[1], qmax, ragged=False))
        k = i % 3
        depth = int(rng.integers(1, 5)) if k == 0 else int(rng.integers(5, 24)) if k == 1 else int(rng.integers(24, 41))
        L = int(rng.integers(1, 301)) if rng.random() < 0.2 else int(rng.integers(60, 180))
        add(_rows(rng, depth, L, qmax, ragged=rng.random() < 0.5))
    if off % 16 == 0:
        add(_rows(rng, 1, 5, qmax, False))
    return units


# ---- BAM4 ---------------------------------------------------------------------------------------------------------
def _nibbles(seq: np.ndarray) -> np.ndarray:
    lut = np.full(256, 15, np.uint8)
    for i, c in enumerate(NIBBLE_CODES):
        lut[c] = i
    return lut[seq]


def bam4_batch(fg, seed: int, chunk_bytes: int, n_units: int = BAM4_UNITS, min_q: int = 10, min_reads: int = 2):
    """(layout PackedBatch with tiles, RawColumns, spans per unit: [(raw seq, raw quals, reverse, row length)]).  Raw spans: even offsets with
    gaps of 0-40 bases between them, the reads that open the chunks of `chunk_bytes` at offsets 0, 2, .., 30 modulo
    32 in turn (the others at random even offsets), a third on the reverse strand, odd and even raw lengths, rows up
    to 7 bases shorter than their span, raw qualities 0-255 and a few IUPAC / '=' codes.  The expected rows are those
    `create_source_read` gives (`expected_rows`)."""
    from fgumi_b200.engine import RAW_READ_DTYPE, RawColumns, pack_source_reads, plan_tiles
    rng = np.random.default_rng(seed)
    alphabet = np.frombuffer(b"ACGTACGTACGTACGTACGTNRY=", np.uint8)
    spans = []                      # per unit: [(raw seq, raw quals, reverse, row length)]
    for i in range(n_units):
        depth = int(rng.integers(1, 5)) if i % 3 == 0 else int(rng.integers(5, 24)) if i % 3 == 1 else int(rng.integers(24, 33))
        L = int(rng.integers(20, 200))
        u = []
        for _ in range(depth):
            raw_len = int(rng.integers(max(1, L - 10), L + 1))
            row = raw_len - (int(rng.integers(0, 8)) if rng.random() < 0.4 else 0)
            row = max(1, row)
            seq = alphabet[rng.integers(0, alphabet.size, size=raw_len)]
            q = rng.integers(0, 256, size=raw_len).astype(np.uint8)
            u.append((seq, q, bool(rng.random() < 0.35), row))
        spans.append(u)
    layout = pack_source_reads([[(b"\0" * r[3], b"\0" * r[3]) for r in u] for u in spans], min_reads)
    layout.bases = layout.quals = None
    plan_tiles(layout)
    opens = {c["rf"] for c in cuts(layout, chunk_bytes)}
    flat = [r for u in spans for r in u]
    rr = np.zeros(len(flat) + 1, dtype=RAW_READ_DTYPE)
    src = np.zeros(len(flat), np.int64)
    cursor, k_open = 0, 0
    for r, (seq, q, rev, row) in enumerate(flat):
        start = cursor + 2 * int(rng.integers(0, 21))               # a gap of 0..40 bases
        start += start & 1
        if r in opens:                                              # the chunk's first span: the next residue mod 32
            want = (2 * k_open) % 32
            start += (want - start) % 32
            k_open += 1
        src[r] = start
        rr[r] = (start, len(seq), 1 if rev else 0)
        cursor = start + len(seq)
    n_raw = cursor
    seq_col = np.full(n_raw + (n_raw & 1), ord("="), np.uint8)      # '=' is nibble 0
    qual_col = np.zeros(n_raw + 32, np.uint8)
    for r, (seq, q, _, _) in enumerate(flat):
        seq_col[src[r]:src[r] + len(seq)] = seq
        qual_col[src[r]:src[r] + len(q)] = q
    nib = _nibbles(seq_col)
    seq4 = np.concatenate([((nib[0::2] << 4) | nib[1::2]).astype(np.uint8), np.zeros(32, np.uint8)])
    raw = RawColumns(seq4, qual_col, rr, n_raw, min_q)
    return layout, raw, spans


def expected_rows(spans, min_q: int) -> List[List[Tuple[bytes, bytes]]]:
    """The rows of create_source_read: position p from raw base p (forward) or raw_len - 1 - p complemented (reverse),
    q < min_q -> (N, Q2)."""
    comp = np.arange(256, dtype=np.uint8)
    for a, b in zip(NIBBLE_CODES, COMPLEMENT):
        comp[a] = b
    out = []
    for u in spans:
        rows = []
        for seq, q, rev, row in u:
            if rev:
                b, qq = comp[seq[::-1]][:row], q[::-1][:row]
            else:
                b, qq = seq[:row], q[:row]
            b, qq = b.copy(), qq.copy()
            m = qq < min_q
            b[m] = ord("N")
            qq[m] = 2
            rows.append((b.tobytes(), qq.tobytes()))
        out.append(rows)
    return out


def with_min_q(raw, min_q: int):
    """The same raw columns with another min_input_base_quality."""
    from fgumi_b200.engine import RawColumns
    return RawColumns(raw.seq4, raw.quals_raw, raw.raw_reads, raw.n_raw, min_q)


# ---- the benchmark's shape ----------------------------------------------------------------------------------------
def bench_batch(n_units: int = 200_000, seed: int = 1234):
    """Depth 8, 150 bp, ~0.1 % substitutions and the quality curve of synth.host_pileup, packed with pack_uniform."""
    from fgumi_b200 import synth
    from fgumi_b200.engine import pack_uniform, plan_tiles
    bases, quals = synth.host_pileup(n_units, 8, 150, 1e-3, seed=seed)
    batch = pack_uniform(bases, quals, 1)
    plan_tiles(batch)
    return batch


def unit_rows(batch, u: int) -> List[Tuple[bytes, bytes]]:
    """The rows of unit u of a two-column batch."""
    r0, r1 = int(batch.units["read_begin"][u]), int(batch.units["read_begin"][u + 1])
    rows = []
    for r in range(r0, r1):
        d = int(batch.reads[r])
        o, n = d >> 16, d & 0xFFFF
        rows.append((batch.bases[o:o + n].tobytes(), batch.quals[o:o + n].tobytes()))
    return rows


def boundary_units(batch, chunks: Sequence[Dict]) -> List[int]:
    """Every unit of the tiles on either side of each chunk boundary."""
    T = batch.tiles
    us = set()
    for c in chunks[1:]:
        for t in (c["t0"] - 1, c["t0"]):
            a = int(T[t]["unit_begin"])
            us.update(range(a, a + int(T[t]["n_units"])))
    return sorted(us)


# ---- the filter epilogue ------------------------------------------------------------------------------------------
def filter_statuses(batch, cols, p: Dict) -> np.ndarray:
    """FGB_FILTER_* per unit of the filter rules over voted columns (base, qual, depth, errors): mask positions below
    min_base_quality, below min_reads or above max_base_error_rate, then reject on depth, read error rate, mean
    quality and no-call fraction, in that order; 255 for a unit that called nothing."""
    base, qual, depth, errors = cols
    out = np.full(batch.n_units, 255, np.uint8)
    for u in range(batch.n_units):
        o, n = int(batch.units["out_off"][u]), int(batch.units["cons_len"][u])
        if n == 0:
            continue
        b, q = base[o:o + n].copy(), qual[o:o + n].copy()
        d, e = depth[o:o + n].astype(np.int64), errors[o:o + n].astype(np.int64)
        rate = np.where(d > 0, e / np.maximum(d, 1), 0.0)
        m = (q < p["min_base_quality"]) | (d < p["min_reads"]) | ((d > 0) & (rate > p["max_base_error_rate"]))
        b[m] = ord("N")
        q[m] = 2
        td, te = int(d.sum()), int(e.sum())
        ce = np.float32(0) if td == 0 else np.float32(te) / np.float32(td)
        n_n = int((b == ord("N")).sum())
        mean = float(q[b != ord("N")].astype(np.int64).sum()) / (n - n_n) if n > n_n else 0.0
        if int(d.max()) < p["min_reads"]:
            out[u] = 1
        elif float(ce) > p["max_read_error_rate"]:
            out[u] = 2
        elif mean < p["min_mean_base_quality"]:
            out[u] = 3
        elif n_n / n > p["max_no_call_fraction"]:
            out[u] = 4
        else:
            out[u] = 0
    return out
