"""Synthetic grouped-family generator (restates the model of `fgumi simulate grouped-reads`).

Model (reference, fgumi 0.2.0 src/lib/):
  * template bases uniform over ACGT; every read of a family copies the template
    (commands/simulate/grouped_reads.rs:530-556);
  * qualities from PositionQualityModel::default — ramp 25->37 over the first 10 bases, 37 flat,
    -0.08/base after position 100, + N(0, 2) noise, round, clamp to [2, 41]; R2 gets -2
    (simulate/quality.rs:54-66, 99-124, 187-199);
plus the two knobs BASELINE.json's configs need and the reference's simulator lacks (SURVEY §0
fact 4): a FIXED (or Zipf) family depth and Bernoulli(error_rate) substitution errors, uniform over
the three alternative bases.  The reference's RNG stream (StdRng/ChaCha12) is not reproducible here;
only the model is restated.

`host_pileup` builds small dense pileups with numpy (tests, CPU baseline sample);
`device_batch_fixed` / `device_batch_ragged` build BASELINE-size batches directly in HBM with torch
(plumbing only: the consensus itself never runs in torch).
"""
from __future__ import annotations

import numpy as np

from . import lib as _l
from .engine import PackedBatch, TILE_DTYPE, UNIT_DTYPE, _round_up

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


def _base_quality_curve(L: int) -> np.ndarray:
    pos = np.arange(L, dtype=np.float64)
    q = np.where(pos < 10, 25.0 + (pos / 10.0) * 12.0, 37.0)
    q = np.where(pos >= 100, np.maximum(37.0 - (pos - 100.0) * 0.08, 2.0), q)
    return q


def host_pileup(n_units: int, depth: int, L: int = 150, error_rate: float = 1e-3, seed: int = 42,
                r2: bool = False, n_rate: float = 0.0, min_input_q: int = 10):
    """Dense [U, D, L] bases/quals as SourceRead rows (quality masking of
    vanilla_caller.rs:903-911 already applied: q < min_input_q -> ('N', 2))."""
    rng = np.random.default_rng(seed)
    tmpl = ACGT[rng.integers(0, 4, size=(n_units, 1, L))]
    bases = np.broadcast_to(tmpl, (n_units, depth, L)).copy()
    if error_rate > 0:
        err = rng.random((n_units, depth, L)) < error_rate
        shift = rng.integers(1, 4, size=(n_units, depth, L))
        code = np.searchsorted(ACGT, bases)          # A,C,G,T -> 0..3 (ACGT is sorted in ASCII)
        alt = ACGT[(code + shift) % 4]
        bases = np.where(err, alt, bases)
    q = _base_quality_curve(L)[None, None, :] + rng.normal(0.0, 2.0, size=(n_units, depth, L))
    q = np.clip(np.rint(q), 2, 41)
    if r2:
        q = np.clip(q - 2, 2, 41)
    quals = q.astype(np.uint8)
    if n_rate > 0:
        nm = rng.random((n_units, depth, L)) < n_rate
        bases = np.where(nm, np.uint8(ord("N")), bases)
        quals = np.where(nm, np.uint8(2), quals)
    low = quals < min_input_q
    bases = np.where(low, np.uint8(ord("N")), bases).astype(np.uint8)
    quals = np.where(low, np.uint8(2), quals).astype(np.uint8)
    return bases, quals


def zipf_depths(n_units: int, lo: int = 1, hi: int = 100, s: float = 1.0, seed: int = 42) -> np.ndarray:
    """Truncated Zipf(s) on [lo, hi] (BASELINE.json config 5)."""
    rng = np.random.default_rng(seed)
    k = np.arange(lo, hi + 1, dtype=np.float64)
    p = k ** (-s)
    p /= p.sum()
    return rng.choice(np.arange(lo, hi + 1), size=n_units, p=p).astype(np.int64)


class TorchBatch:
    """A device-resident fgb_batch built by torch (same fields as engine.DeviceBatch)."""

    def __init__(self, bases, quals, reads, units, tiles, host: PackedBatch, class_tiles=(0, 0, 0)):
        self.bases, self.quals, self.reads, self.units, self.tiles = bases, quals, reads, units, tiles
        self.host = host
        self.n_tiles = len(host.tiles)
        self.class_tiles = class_tiles

    def struct(self) -> _l.FgbBatch:
        import ctypes as C
        b = self.host
        return _l.FgbBatch(b.n_units, b.n_reads, b.n_bytes, b.n_out, self.n_tiles,
                           self.bases.data_ptr(), self.quals.data_ptr(), self.reads.data_ptr(),
                           self.units.data_ptr(), self.tiles.data_ptr(), (C.c_uint64 * 3)(*self.class_tiles))


def _hashed_templates(torch, dev, template_ids, L, seed):
    """Template base codes as a stateless hash of (seed, template id, position): units that share a
    template id share a template, independent of how the batch is chunked."""
    x = template_ids.to(dev, torch.int64)[:, None] * 1_000_003 + torch.arange(L, device=dev)[None, :]
    x = x + seed * 7_919
    x = (x ^ (x >> 30)) * -4658895280553007687      # splitmix64 constants (int64 arithmetic wraps)
    x = (x ^ (x >> 27)) * -7723592293110705685
    x = x ^ (x >> 31)
    return (x >> 40) & 3


def _gen_rows(torch, dev, gen, depths_t, L, Lp, error_rate, out_b, out_q, row0, chunk_units,
              template_ids=None, seed=0):
    """Fill rows [row0, row0 + sum(depths)) of the [R, Lp] byte matrices for one chunk of units."""
    U = depths_t.numel()
    acgt = torch.tensor([65, 67, 71, 84], dtype=torch.uint8, device=dev)
    curve = torch.from_numpy(_base_quality_curve(L)).to(dev, torch.float32)
    if template_ids is None:
        tmpl_code = torch.randint(0, 4, (U, L), device=dev, generator=gen, dtype=torch.int64)
    else:
        tmpl_code = _hashed_templates(torch, dev, template_ids, L, seed)
    unit_of_row = torch.repeat_interleave(torch.arange(U, device=dev), depths_t)
    R = unit_of_row.numel()
    code = tmpl_code[unit_of_row]                                   # [R, L]
    if error_rate > 0:
        err = torch.rand((R, L), device=dev, generator=gen) < error_rate
        shift = torch.randint(1, 4, (R, L), device=dev, generator=gen, dtype=torch.int64)
        code = torch.where(err, (code + shift) % 4, code)
    q = curve[None, :] + 2.0 * torch.randn((R, L), device=dev, generator=gen)
    q = torch.clamp(torch.round(q), 2, 41).to(torch.uint8)
    b = acgt[code]
    low = q < 10                                                    # min_input_base_quality mask
    b = torch.where(low, torch.tensor(78, dtype=torch.uint8, device=dev), b)
    q = torch.where(low, torch.tensor(2, dtype=torch.uint8, device=dev), q)
    out_b[row0:row0 + R, :L] = b
    out_q[row0:row0 + R, :L] = q
    return R


def make_descriptors(depths: np.ndarray, L: int = 150, min_reads: int = 1) -> PackedBatch:
    """Read/unit/tile descriptors of a batch whose reads all have length L (columns left empty)."""
    from .engine import plan_tiles
    depths = np.asarray(depths, dtype=np.int64)
    U = int(depths.size)
    Lp = _round_up(L, _l.FGB_READ_ALIGN)
    Lo = _round_up(L, _l.FGB_OUT_ALIGN)
    read_begin = np.zeros(U + 1, dtype=np.int64)
    np.cumsum(depths, out=read_begin[1:])
    R = int(read_begin[-1])
    reads = np.zeros(_round_up(R, 2) + 2, dtype=np.uint64)
    reads[:R] = ((np.arange(R, dtype=np.uint64) * np.uint64(Lp)) << np.uint64(16)) | np.uint64(L)
    units = np.zeros(U + 1, dtype=UNIT_DTYPE)
    units["read_begin"] = read_begin.astype(np.uint32)
    units["out_off"] = np.arange(U + 1, dtype=np.uint64) * np.uint64(Lo)
    units["cons_len"][:U] = np.where(depths >= min_reads, L, 0)
    host = PackedBatch(np.zeros(0, np.uint8), np.zeros(0, np.uint8), reads, units, U, R, R * Lp,
                       U * Lo)
    plan_tiles(host)
    return host


def device_batch(torch, device, depths: np.ndarray, L: int = 150, error_rate: float = 1e-3,
                 seed: int = 42, min_reads: int = 1, chunk_rows: int = 2_000_000,
                 template_ids: np.ndarray = None) -> TorchBatch:
    """Build a batch with per-unit depths `depths` (fixed or ragged), all reads of length L,
    directly in device memory.  Host keeps only the (small) unit/read/tile descriptors."""
    depths = np.asarray(depths, dtype=np.int64)
    U = int(depths.size)
    Lp = _round_up(L, _l.FGB_READ_ALIGN)
    host = make_descriptors(depths, L, min_reads)
    reads, units = host.reads, host.units
    read_begin = units["read_begin"].astype(np.int64)
    R = host.n_reads
    # device columns
    dev = torch.device(device)
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    tot_rows = R + (16 // 4)   # >= 16 bytes of slack so the last tile's 16-byte round-up is in bounds
    bmat = torch.zeros((tot_rows, Lp), dtype=torch.uint8, device=dev)
    qmat = torch.zeros((tot_rows, Lp), dtype=torch.uint8, device=dev)
    u0 = 0
    while u0 < U:
        # take units until ~chunk_rows rows
        u1 = int(np.searchsorted(read_begin, read_begin[u0] + chunk_rows, side="right")) - 1
        u1 = max(u0 + 1, min(U, u1))
        d = torch.from_numpy(depths[u0:u1]).to(dev)
        tid = None if template_ids is None else torch.from_numpy(
            np.ascontiguousarray(template_ids[u0:u1]).astype(np.int64))
        _gen_rows(torch, dev, gen, d, L, Lp, error_rate, bmat, qmat, int(read_begin[u0]), u1 - u0, tid, seed)
        u0 = u1
    to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)
    from .engine import sort_tiles_by_class
    tiles, classes = sort_tiles_by_class(host.tiles) if len(host.tiles) else (np.zeros(1, dtype=TILE_DTYPE), (0, 0, 0))
    return TorchBatch(bmat.reshape(-1), qmat.reshape(-1), to_dev(reads), to_dev(units), to_dev(tiles),
                      host, classes)


def record_families(n_families: int, depth: int = 8, L: int = 150, error_rate: float = 1e-3, seed: int = 42,
                    reverse_fraction: float = 0.0):
    """Synthetic MI-grouped BAM records for the record-level callers, built with numpy (no Python loop):
    `n_families` groups of `depth` unpaired mapped reads of length L (CIGAR `<L>M`), bases and qualities from
    the same model as host_pileup (no masking: the callers do that), tags MI:Z:<8 digits>, RX:Z:<8 bases>.
    Every record has the same size, so the blob is one [reads, record] byte matrix.
    Returns (blob uint8[...], rec_off uint64[R + 1], group_rec uint64[G + 1])."""
    rng = np.random.default_rng(seed)
    U, D = int(n_families), int(depth)
    bases, quals = host_pileup(U, D, L, error_rate, seed=seed, min_input_q=0)      # [U, D, L]
    R = U * D
    bases = bases.reshape(R, L)
    quals = quals.reshape(R, L)
    fam = np.repeat(np.arange(U, dtype=np.int64), D)
    rd = np.tile(np.arange(D, dtype=np.int64), U)
    rev = np.zeros(R, dtype=bool)
    if reverse_fraction > 0:
        rev = np.repeat(rng.random(U) < reverse_fraction, D)
    nseq = (L + 1) // 2
    name_len = 12                                                     # 'q' + 7 digits + '.' + 2 digits + NUL
    rec_len = 32 + name_len + 4 + nseq + L + 12 + 12
    rec = np.zeros((R, rec_len), dtype=np.uint8)

    def put(col, values, dtype):
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=dtype), (R,)))
        rec[:, col:col + v.dtype.itemsize] = v.view(np.uint8).reshape(R, v.dtype.itemsize)

    put(0, 0, "<i4"); put(4, 1000 + (fam % 100000), "<i4")
    rec[:, 8] = name_len; rec[:, 9] = 60
    put(10, 4680, "<u2"); put(12, 1, "<u2"); put(14, np.where(rev, 16, 0), "<u2"); put(16, L, "<u4")
    put(20, -1, "<i4"); put(24, -1, "<i4"); put(28, 0, "<i4")

    def digits(col, values, n):
        v = values.copy()
        for k in range(n - 1, -1, -1):
            rec[:, col + k] = 48 + (v % 10)
            v //= 10

    o = 32
    rec[:, o] = ord("q"); digits(o + 1, fam % 10_000_000, 7); rec[:, o + 8] = ord("."); digits(o + 9, rd % 100, 2)
    o += name_len
    put(o, (L << 4) | 0, "<u4"); o += 4
    # 4-bit sequence; a reverse-strand record stores the reverse complement of the read
    code = np.zeros(256, dtype=np.uint8); code[:] = 15
    for i, ch in enumerate(b"=ACMGRSVTWYHKDBN"):
        code[ch] = i
    comp = np.arange(256, dtype=np.uint8)
    for x, y in (b"AT", b"TA", b"CG", b"GC"):
        comp[x] = y
    sb = np.where(rev[:, None], comp[bases][:, ::-1], bases)
    sq = np.where(rev[:, None], quals[:, ::-1], quals)
    nib = code[sb]
    if L % 2:
        nib = np.concatenate([nib, np.zeros((R, 1), dtype=np.uint8)], axis=1)
    rec[:, o:o + nseq] = (nib[:, 0::2] << 4) | nib[:, 1::2]
    o += nseq
    rec[:, o:o + L] = sq
    o += L
    rec[:, o:o + 3] = np.frombuffer(b"MIZ", np.uint8); digits(o + 3, fam % 100_000_000, 8); o += 12
    rec[:, o:o + 3] = np.frombuffer(b"RXZ", np.uint8)
    umi = ACGT[rng.integers(0, 4, size=(U, 8))]
    rec[:, o + 3:o + 11] = np.repeat(umi, D, axis=0)
    o += 12
    assert o == rec_len
    rec_off = np.arange(R + 1, dtype=np.uint64) * np.uint64(rec_len)
    group_rec = np.arange(U + 1, dtype=np.uint64) * np.uint64(D)
    return rec.reshape(-1), rec_off, group_rec


def umi_families(n_molecules: int, length: int, mean_family: float = 4.0, error_rate: float = 0.01,
                 paired: bool = False, swap_rate: float = 0.5, seed: int = 0):
    """Seeded UMIs of one position group: `n_molecules` true UMIs of `length` bases, family sizes 1 + Poisson
    (mean_family - 1), each base of each read's UMI replaced by another base with probability `error_rate`.
    With `paired` a true UMI is "X-Y" (two halves of `length` bases) and a read of the other strand carries
    "Y-X" with probability `swap_rate`.  Returns a list of str, reads in random order."""
    rng = np.random.default_rng(seed)
    L = length * 2 if paired else length
    true = rng.integers(0, 4, size=(n_molecules, L), dtype=np.uint8)
    sizes = 1 + rng.poisson(max(mean_family - 1.0, 0.0), size=n_molecules)
    reads = np.repeat(true, sizes, axis=0)
    err = rng.random(reads.shape) < error_rate
    reads = np.where(err, (reads + rng.integers(1, 4, size=reads.shape, dtype=np.uint8)) % 4, reads)
    reads = reads[rng.permutation(len(reads))]
    txt = ACGT[reads]
    out = [bytes(r).decode() for r in txt]
    if paired:
        swap = rng.random(len(out)) < swap_rate
        out = [(u[length:] + "-" + u[:length]) if s else (u[:length] + "-" + u[length:]) for u, s in zip(out, swap)]
    return out


def mapped_templates(n_sites: int, molecules: int = 3, mean_family: float = 3.0, umi_length: int = 8,
                     paired_umis: bool = False, umi_error_rate: float = 0.02, n_umi_rate: float = 0.0,
                     no_dash_rate: float = 0.0, low_mapq_rate: float = 0.0, qc_fail_rate: float = 0.0,
                     unmapped_mate_rate: float = 0.0, secondary_rate: float = 0.0, reverse_rate: float = 0.3,
                     cross_contig_rate: float = 0.0, amplicon_molecules: int = 0, read_length: int = 20,
                     seed: int = 0):
    """Seeded template-coordinate-sorted mapped paired-end templates, as `fgumi group` takes them: (SAM header text,
    record bodies uint8[...], rec_off uint64[n + 1]).

    Each site is one position: `molecules` true UMIs (RX, "X-Y" with `paired_umis`, the halves swapped on the
    templates of the other strand), family sizes 1 + Poisson(mean_family - 1), each UMI base substituted with
    probability `umi_error_rate`.  Each molecule has its own R1 and R2 sequences, copied into its reads with 2 %
    substitutions and qualities 20-40.  Records carry RX, MC, MQ, RG (three read groups, two sharing a library) and CB
    (one cell per site).  Per template, with the given rates: an upper-case N in the UMI, a UMI without its '-',
    MAPQ 0 on one read, the QC-fail flag, a supplementary and a secondary record after the primaries, and the pair
    on the other contig.  With `unmapped_mate_rate` a site is followed by a site of templates whose R2 is unmapped.
    `amplicon_molecules` > 0 adds one site with that many molecules (one large call)."""
    import struct
    rng = np.random.default_rng(seed)
    header = ("@HD\tVN:1.6\tSO:unsorted\tGO:query\tSS:unsorted:template-coordinate\n"
              "@SQ\tSN:chr1\tLN:100000000\n@SQ\tSN:chr2\tLN:100000000\n"
              "@RG\tID:A\tSM:s\tLB:L1\n@RG\tID:B\tSM:s\tLB:L1\n@RG\tID:C\tSM:s\tLB:L2\n"
              "@PG\tID:bwa\tPN:bwa\tCL:bwa mem\n").encode()
    L = read_length
    nib = np.array([1, 2, 4, 8], np.uint8)             # A C G T in BAM's 4-bit code
    cig = struct.pack("<I", (L << 4) | 0)
    mc = b"%dM" % L
    out = []
    tnum = 0

    def read_bytes(true):
        """Packed SEQ and QUAL of one read of a molecule: 2 % substitutions, qualities 20-40."""
        b = np.where(rng.random(L) < 0.02, (true + rng.integers(1, 4, size=L)) % 4, true)
        n = nib[b]
        if L % 2:
            n = np.concatenate([n, np.zeros(1, np.uint8)])
        return ((n[0::2] << 4) | n[1::2]).tobytes() + rng.integers(20, 41, size=L, dtype=np.uint8).tobytes()

    def rec(name, flag, ref, pos, mapq, mref, mpos, tags, true):
        r = (struct.pack("<iiBBHHHIiii", ref, pos, len(name) + 1, mapq, 4680, 0 if flag & 4 else 1, flag, L, mref,
                         mpos, 0) + name + b"\0" + (b"" if flag & 4 else cig) + read_bytes(true) + tags)
        out.append(r)

    def ztag(t, v):
        return t + b"Z" + v + b"\0"

    def umi_str(true, strand_b):
        u = true.copy()
        err = rng.random(len(u)) < umi_error_rate
        u = np.where(err, (u + rng.integers(1, 4, size=len(u))) % 4, u)
        s = bytearray(ACGT[u].tobytes())
        if rng.random() < n_umi_rate:
            s[int(rng.integers(0, len(s)))] = ord("N")
        if paired_umis:
            h = len(s) // 2
            a, b = bytes(s[:h]), bytes(s[h:])
            if strand_b:
                a, b = b, a
            return a + b + b"" if rng.random() < no_dash_rate else a + b"-" + b
        return bytes(s)

    def site(pos, n_mol, unmapped_mates):
        nonlocal tnum
        rg = [b"A", b"B", b"C"][int(rng.integers(0, 3))]
        cb = b"CELL%d" % int(rng.integers(0, 4))
        width = 2 * umi_length if paired_umis else umi_length
        trues = rng.integers(0, 4, size=(n_mol, width))
        bases = rng.integers(0, 4, size=(n_mol, 2, L))     # the molecule's R1 and R2 sequences
        sizes = 1 + rng.poisson(max(mean_family - 1.0, 0.0), size=n_mol)
        cross = (not unmapped_mates) and rng.random() < cross_contig_rate
        for m in range(n_mol):
            for _ in range(int(sizes[m])):
                tnum += 1
                name = b"t%09d" % tnum
                rev = rng.random() < reverse_rate    # R1 reverse, R2 forward: the other strand of the molecule
                u = umi_str(trues[m], rev)
                q1 = 0 if rng.random() < low_mapq_rate else 60
                qc = 0x200 if rng.random() < qc_fail_rate else 0
                common = ztag(b"RX", u) + ztag(b"RG", rg) + ztag(b"CB", cb)
                if unmapped_mates:
                    rec(name, 0x1 | 0x8 | 0x40 | qc, 0, pos, q1, 0, pos, common, bases[m, 0])
                    rec(name, 0x1 | 0x4 | 0x80, 0, pos, 0, 0, pos, common, bases[m, 1])
                    continue
                r2ref = 1 if cross else 0
                r2pos = pos if cross else pos + 50
                f1 = 0x1 | 0x2 | 0x40 | qc | (0x10 if rev else 0x20)
                f2 = 0x1 | 0x2 | 0x80 | (0x20 if rev else 0x10)
                mq = b"MQi" + struct.pack("<i", 60)
                if rev:   # R1 on the reverse strand at the right end; R2 forward at the left
                    p1, ref1, p2, ref2 = r2pos, r2ref, pos, 0
                else:
                    p1, ref1, p2, ref2 = pos, 0, r2pos, r2ref
                rec(name, f1, ref1, p1, q1, ref2, p2, common + ztag(b"MC", mc) + mq, bases[m, 0])
                rec(name, f2, ref2, p2, 60, ref1, p1, common + ztag(b"MC", mc) + b"MQi" + struct.pack("<i", q1), bases[m, 1])
                if rng.random() < secondary_rate:
                    rec(name, f1 | 0x800, ref1, p1 + 7, 60, ref2, p2, common, bases[m, 0])
                    rec(name, f1 | 0x100, ref1, p1 + 9, 60, ref2, p2, common, bases[m, 0])

    for s in range(n_sites):
        site(1000 + 200 * s, molecules, False)
        if rng.random() < unmapped_mate_rate:
            site(1000 + 200 * s + 100, max(1, molecules // 2), True)
    if amplicon_molecules:
        site(1000 + 200 * n_sites + 500, amplicon_molecules, False)
    off = np.zeros(len(out) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in out])
    return header, np.frombuffer(b"".join(out) or b"\0", np.uint8)[:int(off[-1])].copy(), off
