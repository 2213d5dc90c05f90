"""Seeded raw records for the sort tests: every kind of record the sort keys treat differently."""
import struct

import numpy as np

from tests.bam_builder import make_record

HEADER = (b"@HD\tVN:1.6\tSO:unsorted\n@SQ\tSN:chr1\tLN:1000000\n"
          b"@RG\tID:A\tSM:s\tLB:libB\n@RG\tID:B\tSM:s\tLB:libA\n@RG\tID:C\tSM:s\n"
          b"@RG\tID:D\tSM:s\tLB:unknown\n@RG\tID:E\tSM:s\tLB:libA\n@PG\tID:bwa\tPN:bwa\n")
MC_VALUES = [b"10M", b"5S10M", b"3H2S10M4S1H", b"10M5S3M2S", b"4M2D3N2=1X6S", b"", b"abc", b"12", b"M5S",
             b"99999999999M", b"2S99999999999S8M", b"0S10M0H", b"\xff\xfe10M", b"10M\xc3"]
MI_Z = [b"123", b"45/A", b"6/B", b"/A", b"", b"12x", b"99999999999999999999999", b"7/C", b"8/", b"0/B", b"//B"]
TIDS = [-1, 0, 1, 2, 65534, 65535, 65536, 70000, 2 ** 31 - 1]
POS = [-1, 0, 1, 99, 100, 101, 5000, 2 ** 31 - 1, -5]


def _cigar(rng):
    ops = []
    if rng.random() < 0.3:
        ops.append("%dH" % rng.integers(1, 6))
    if rng.random() < 0.4:
        ops.append("%dS" % rng.integers(1, 8))
    for _ in range(int(rng.integers(1, 4))):
        ops.append("%d%s" % (rng.integers(1, 30), "MMMIDN=X"[int(rng.integers(0, 8))]))
    if rng.random() < 0.4:
        ops.append("%dS" % rng.integers(1, 8))
    if rng.random() < 0.3:
        ops.append("%dH" % rng.integers(1, 6))
    return "".join(ops)


def _aux(rng, cell_values):
    out = b""
    for _ in range(int(rng.integers(0, 7))):
        k = int(rng.integers(0, 9))
        if k == 0:
            out += b"MCZ" + MC_VALUES[int(rng.integers(0, len(MC_VALUES)))] + b"\0"
        elif k == 1:
            out += b"MCZ" + _cigar(rng).encode() + b"\0"
        elif k == 2:
            out += b"MIZ" + MI_Z[int(rng.integers(0, len(MI_Z)))] + b"\0"
        elif k == 3:
            t = "cCsSiI"[int(rng.integers(0, 6))]
            lo, hi = {"c": (-128, 127), "C": (0, 255), "s": (-32768, 32767), "S": (0, 65535),
                      "i": (-2 ** 31, 2 ** 31 - 1), "I": (0, 2 ** 32 - 1)}[t]
            v = int(rng.integers(lo, hi, endpoint=True))
            out += b"MI" + t.encode() + struct.pack({"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i",
                                                     "I": "<I"}[t], v)
        elif k == 4:
            out += b"RGZ" + [b"A", b"B", b"C", b"D", b"E", b"ZZ", b""][int(rng.integers(0, 7))] + b"\0"
        elif k == 5:
            out += b"CBZ" + cell_values[int(rng.integers(0, len(cell_values)))] + b"\0"
        elif k == 6:
            out += b"XXi" + struct.pack("<i", int(rng.integers(0, 1000)))
        elif k == 7:
            n = int(rng.integers(0, 4))
            out += b"ZBBs" + struct.pack("<I", n) + struct.pack("<%dh" % n, *range(n))
        else:
            out += [b"MIf" + struct.pack("<f", 1.5), b"QQ?xyz", b"MIA7", b"ZZZtrunc"][int(rng.integers(0, 4))]
    return out


def random_records(n: int, seed: int, n_names: int = 0):
    """n records (no block_size prefix).  Names come from a pool of n_names (0: about n / 2), so templates share
    names and planted exact duplicates test stability."""
    rng = np.random.default_rng(seed)
    names = [b"q%d" % i + b"x" * int(rng.integers(0, 12)) for i in range(n_names or max(1, n // 2))]
    cells = [b"AAAA", b"CCGT", b"", b"TTTTTTTT", b"\xff"]
    recs = []
    while len(recs) < n:
        if recs and rng.random() < 0.05:             # an exact duplicate of an earlier record
            recs.append(recs[int(rng.integers(0, len(recs)))])
            continue
        flag = 0
        for bit, p in ((0x1, 0.8), (0x4, 0.15), (0x8, 0.15), (0x10, 0.4), (0x20, 0.4), (0x40, 0.5), (0x80, 0.5),
                       (0x100, 0.05), (0x800, 0.05)):
            if rng.random() < p:
                flag |= bit
        tid = TIDS[int(rng.integers(0, len(TIDS)))] if rng.random() < 0.3 else int(rng.integers(0, 3))
        pos = POS[int(rng.integers(0, len(POS)))] if rng.random() < 0.3 else int(rng.integers(0, 400))
        mtid = TIDS[int(rng.integers(0, len(TIDS)))] if rng.random() < 0.2 else int(rng.integers(0, 3))
        mpos = POS[int(rng.integers(0, len(POS)))] if rng.random() < 0.2 else int(rng.integers(0, 400))
        seq_len = int(rng.integers(0, 12))
        seq = bytes(b"ACGT"[int(x)] for x in rng.integers(0, 4, size=seq_len))
        cig = "" if rng.random() < 0.1 else _cigar(rng)
        r = make_record(name=names[int(rng.integers(0, len(names)))], flags=flag, ref_id=tid, pos=pos,
                        cigar=cig if cig else [], mate_ref_id=mtid, mate_pos=mpos, seq=seq)
        r = bytearray(r + _aux(rng, cells))
        u = rng.random()
        if u < 0.03 and len(r) > 34:                  # aux or fields cut short
            r = r[:int(rng.integers(32, len(r)))]
        elif u < 0.05:                                # a read name that runs past the record
            r[8] = 255
        elif u < 0.07:                                # a CIGAR that runs past the record
            struct.pack_into("<H", r, 12, 60000)
        elif u < 0.08:                                # l_seq past the record: no aux block
            struct.pack_into("<I", r, 16, 10 ** 6)
        recs.append(bytes(r))
    return recs


def pack(recs):
    """(bodies uint8[...], rec_off uint64[n + 1])"""
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in recs]) if recs else []
    return np.frombuffer(b"".join(recs) or b"\0", np.uint8)[:int(off[-1])].copy(), off


# ---- inputs at the sizes users sort (tests/test_sort_records_scale_gpu.py) -------------------------------------------
# Bulk inputs tile a pool of distinct records with numpy and then overwrite fixed fields: tid, pos, the strand bits of
# the flag and the mate's tid and pos, drawn from small ranges so that keys tie often, and a per-record serial in
# MAPQ, bin and TLEN (bytes 9-11 and 28-31), which neither key reads.  With the serial every record is byte-unique,
# so a wrong permutation, a lost record or an unstable tie changes the output bytes.
STAGE_BYTES = 64 << 20                        # one page-locked staging buffer of the device sort (sort_host.cpp)
SERIAL_BYTES = (9, 10, 11, 28, 29, 30, 31)
TIE_TIDS = np.array([-1, 0, 1, 2], np.int32)
TIE_POS = (-1, 24)                            # [lo, hi)


def fit(r: bytes, n: int) -> bytes:
    """r cut or padded to exactly n >= 32 bytes: the padding is one XP:Z tag, or NULs when fewer than 4 are missing."""
    if len(r) >= n:
        return r[:n]
    k = n - len(r)
    return r + (b"XPZ" + b"p" * (k - 4) + b"\0" if k >= 4 else b"\0" * k)


def _fixed(tid, pos, l_read_name, n_cigar, flag, l_seq, mtid, mpos):
    return struct.pack("<iiBBHHHIiii", tid, pos, l_read_name, 60, 4680, n_cigar, flag, l_seq, mtid, mpos, 0)


def minimal_record() -> bytes:
    """The smallest well-formed record: the 32-byte fixed part and a 1-byte (empty) read name."""
    return _fixed(0, 0, 1, 0, 0, 0, -1, -1) + b"\0"


def big_record(length: int, seed: int, name: bytes = b"big", flags: int = 0x1 | 0x20, aux: bytes = b"") -> bytes:
    """A record of exactly `length` bytes, most of them SEQ and QUAL, built without a per-base loop."""
    rng = np.random.default_rng(seed)
    m = (length - 32 - len(name) - 1 - 8 - len(aux) - 8) * 2 // 3
    head = _fixed(0, 100, len(name) + 1, 2, flags, m, 0, 150) + name + b"\0" + struct.pack("<2I", (3 << 4) | 4,
                                                                                             ((m - 3) << 4) | 0)
    seq = rng.integers(0, 256, (m + 1) // 2, dtype=np.uint8).tobytes()
    qual = rng.integers(0, 42, m, dtype=np.uint8).tobytes()
    return fit(head + seq + qual + aux, length)


def long_cigar_ops(n_ops: int, tail: int):
    """n_ops CIGAR ops: a soft clip, then M / I / D / N / = / X in turn, the last ref-consuming op `tail` long, then a
    soft and a hard clip.  Records that differ only in `tail` differ only in their 5' end on the reverse strand."""
    cycle = (0, 1, 2, 3, 7, 8)
    ops = [(2 << 4) | 4] + [((1 + i % 3) << 4) | cycle[i % 6] for i in range(n_ops - 4)]
    return ops + [(tail << 4) | 0, (4 << 4) | 4, (1 << 4) | 5]


def cigar_text(ops) -> bytes:
    return "".join("%d%s" % (op >> 4, "MIDNSHP=X"[op & 0xF]) for op in ops).encode()


def long_cigar_record(ops, name: bytes, flags: int, pos: int, mpos: int, mc: bytes) -> bytes:
    """A mapped, paired record with the CIGAR `ops` (up to 65 535 of them) and an MC of the mate's CIGAR."""
    seq_len = sum(op >> 4 for op in ops if op & 0xF in (0, 1, 4, 7, 8))
    head = _fixed(0, pos, len(name) + 1, len(ops), flags, seq_len, 0, mpos) + name + b"\0"
    body = np.array(ops, "<u4").tobytes() + bytes((seq_len + 1) // 2) + bytes([30]) * seq_len
    return head + body + b"MCZ" + mc + b"\0" + b"RGZA\0"


def length_grid(lo: int, hi: int, copies: int, seed: int):
    """`copies` records of every length in [lo, hi), cut from or padded around random records, shuffled."""
    rng = np.random.default_rng(seed)
    base = random_records(64, seed=seed + 1)
    recs = [fit(base[int(rng.integers(0, len(base)))], n) for n in range(lo, hi) for _ in range(copies)]
    return [recs[i] for i in rng.permutation(len(recs))]


def stamp_serials(recs):
    """The records with their index written into MAPQ, bin and TLEN: byte-unique, keys unchanged."""
    out = []
    for i, r in enumerate(recs):
        r = bytearray(r)
        r[9:12] = (i & 0xFFFFFF).to_bytes(3, "little")
        r[28:32] = (i >> 24).to_bytes(4, "little")
        out.append(bytes(r))
    return out


def pack_at(recs, lead: int, skew: int):
    """pack() with `lead` noise bytes before the first record (rec_off[0] = lead) and the bodies array starting
    `skew` bytes into its allocation."""
    b, off = pack(recs)
    raw = np.empty(skew + lead + len(b), np.uint8)
    raw[skew:skew + lead] = np.random.default_rng(lead).integers(0, 256, lead, dtype=np.uint8)
    raw[skew + lead:] = b
    return raw[skew:], off + np.uint64(lead)


def gather_grid(seed: int):
    """Records at the record gather's edges, in an order the sort has to change: every length 32-400 three times;
    stretches of 32-35-byte and of 128-136-byte records whose keys are equal in both orders (the name, CIGAR or aux
    lies past the cut), so that each stretch is contiguous in the output; records of 65 535, 65 536, 65 537 and
    1 MiB + 3 bytes; three reverse-strand records with 65 535 CIGAR ops and three with a 65 535-op MC, each three
    differing only in the last ref-consuming op and placed against their order.  Serials make every record unique."""
    rng = np.random.default_rng(seed)
    recs = length_grid(32, 401, 3, seed)
    short = _fixed(1, 7, 11, 2, 0x1 | 0x10, 60, 1, 9) + b"stretch_01\0"
    mid = short + struct.pack("<2I", (2 << 4) | 4, (58 << 4) | 0) + bytes(30) + bytes([30]) * 60 + b"RGZA\0"
    stretches = [[fit(short, int(n)) for n in rng.integers(32, 36, 160)],
                 [fit(mid, int(n)) for n in rng.integers(128, 137, 160)]]
    big = [big_record(65535, seed, b"b65535"), big_record(65536, seed + 1, b"b65536", 0x1 | 0x10),
           big_record(65537, seed + 2, b"b65537", 0x1 | 0x80, b"MCZ4S6M\0"),
           big_record((1 << 20) + 3, seed + 3, b"b1m", 0x1 | 0x10 | 0x20, b"RGZB\0MIZ7/B\0")]
    long_cigar = [long_cigar_record(long_cigar_ops(65535, t), b"lcig", 0x1 | 0x10 | 0x40, 200, 150, b"20M")
                  for t in (13, 9, 5)]
    long_mc = [long_cigar_record([(20 << 4) | 0], b"lmc", 0x1 | 0x20 | 0x80, 210, 200,
                                 cigar_text(long_cigar_ops(65535, t))) for t in (13, 9, 5)]
    for group in stretches + [big, long_cigar, long_mc]:
        at = np.sort(rng.integers(0, len(recs) + 1, len(group)))
        for k, r in reversed(list(zip(at, group))):
            recs.insert(int(k), r)
    return stamp_serials(recs)


def bulk_pool(seed: int):
    """(common, rare): records of every kind random_records makes plus every length 32-400, and the long shapes --
    a 1 000-op CIGAR with a matching 1 000-op MC, and 65 535 / 65 536 / 65 537-byte records."""
    common = random_records(2000, seed=seed) + length_grid(32, 401, 1, seed)
    ops = long_cigar_ops(1000, 5)
    rare = [long_cigar_record(ops, b"lc%d" % seed, 0x1 | 0x10 | 0x20 | 0x40, 50, 60, cigar_text(ops)),
            big_record(65535, seed, aux=b"MCZ3S7M\0"), big_record(65536, seed + 1, b"big2", 0x1 | 0x10),
            big_record(65537, seed + 2, b"big3", 0x1 | 0x10 | 0x80, b"RGZB\0")]
    return common, rare


def bulk_fields(n: int, seed: int, common: int, rare: int, rare_each: int = 4):
    """Per-record choices: a pool index (common records uniformly, each rare one `rare_each` times) and the fixed
    fields written over it."""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, common, n).astype(np.int64)
    for k in range(rare):
        idx[rng.choice(n, rare_each, replace=False)] = common + k
    return dict(idx=idx, tid=TIE_TIDS[rng.integers(0, len(TIE_TIDS), n)], pos=rng.integers(*TIE_POS, n),
                strand=(rng.integers(0, 4, n) << 4).astype(np.uint8),
                mtid=TIE_TIDS[rng.integers(0, len(TIE_TIDS), n)], mpos=rng.integers(*TIE_POS, n))


def _put(body, at, value, width):
    v = np.asarray(value).astype(np.int64)
    for j in range(width):
        body[at + j] = (v >> (8 * j)) & 0xFF


def materialize(pool, f, lead: int = 0, skew: int = 0, chunk: int = 8 << 20):
    """(bodies, rec_off) of the records pool[f["idx"]] with f's fixed fields and the serial written over them.
    rec_off[0] = lead (the bytes before it are noise), and the bodies array starts `skew` bytes into its allocation,
    so that with skew = 1 its address is not 4-aligned.  Copied in chunks of about `chunk` bytes: no index array is
    as large as the stream."""
    lens = np.array([len(r) for r in pool], np.int64)
    flat = np.frombuffer(b"".join(pool), np.uint8)
    start = np.zeros(len(pool) + 1, np.int64)
    start[1:] = np.cumsum(lens)
    idx = f["idx"]
    n = len(idx)
    size = lens[idx]
    off = np.empty(n + 1, np.int64)
    off[0] = lead
    off[1:] = lead + np.cumsum(size)
    raw = np.empty(skew + int(off[-1]), np.uint8)
    body = raw[skew:]
    body[:lead] = np.random.default_rng(lead).integers(0, 256, lead, dtype=np.uint8)
    a = 0
    while a < n:
        b = min(n, max(a + 1, int(np.searchsorted(off, off[a] + chunk, "right")) - 1))
        within = np.arange(off[b] - off[a]) - np.repeat(off[a:b] - off[a], size[a:b])
        body[off[a]:off[b]] = flat[np.repeat(start[idx[a:b]], size[a:b]) + within]
        a = b
    at = off[:-1]
    _put(body, at, f["tid"], 4)
    _put(body, at + 4, f["pos"], 4)
    body[at + 14] = (body[at + 14] & 0xCF) | f["strand"]
    _put(body, at + 20, f["mtid"], 4)
    _put(body, at + 24, f["mpos"], 4)
    serial = np.arange(n, dtype=np.int64)
    _put(body, at + 9, serial, 3)
    _put(body, at + 28, serial >> 24, 4)
    return body, off.astype(np.uint64)


def records_of(bodies, rec_off, which):
    return [bodies[int(rec_off[i]):int(rec_off[i + 1])].tobytes() for i in which]


def _field(bodies, at, k, dtype):
    w = np.dtype(dtype).itemsize
    return bodies[(at + k)[:, None] + np.arange(w)].copy().view(dtype).ravel()


def coordinate_keys(bodies, rec_off, chunk: int = 1 << 20) -> np.ndarray:
    """oracle/sort_oracle.py coordinate_key in numpy from the fixed fields: all ones for tid < 0, else
    (tid << 34) | ((pos + 1) << 1) | reverse with the int64 -> uint64 wrap."""
    n = len(rec_off) - 1
    out = np.empty(n, np.uint64)
    for a in range(0, n, chunk):
        at = rec_off[a:min(n, a + chunk)].astype(np.int64)
        tid = _field(bodies, at, 0, "<i4").astype(np.int64)
        pos = _field(bodies, at, 4, "<i4").astype(np.int64)
        rev = ((bodies[at + 14] >> 4) & 1).astype(np.uint64)
        k = (tid.astype(np.uint64) << np.uint64(34)) | ((pos + 1).astype(np.uint64) << np.uint64(1)) | rev
        k[tid < 0] = np.uint64(2 ** 64 - 1)
        out[a:a + len(at)] = k
    return out


def sorted_order(keys: np.ndarray) -> np.ndarray:
    """The stable order of uint64[n, 5] template-coordinate key words (np.lexsort: last key first) or of uint64[n]
    coordinate keys."""
    if keys.ndim == 1:
        return np.argsort(keys, kind="stable")
    return np.lexsort(tuple(keys[:, w] for w in range(keys.shape[1] - 1, -1, -1)))


def stream_offsets(rec_off, perm) -> np.ndarray:
    """Offsets of the [u32 block_size][record] blocks of the records in the order perm, and the total at the end."""
    size = (rec_off[1:] - rec_off[:-1]).astype(np.int64)[perm]
    out = np.zeros(len(perm) + 1, np.int64)
    out[1:] = np.cumsum(size + 4)
    return out


def alignments(rec_off, perm) -> set:
    """The (source offset mod 4, output offset mod 4, length mod 4) combinations of the record gather, with the
    records in one run: source offsets count from the first record, output offsets from the stream's start."""
    at = stream_offsets(rec_off, perm)[:-1] + 4
    src = (rec_off[:-1].astype(np.int64) - int(rec_off[0]))[perm]
    size = (rec_off[1:] - rec_off[:-1]).astype(np.int64)[perm]
    return set(zip((src % 4).tolist(), (at % 4).tolist(), (size % 4).tolist()))


def expected_stream(bodies, rec_off, perm, lo: int, hi: int) -> np.ndarray:
    """The [u32 block_size][record] bytes of the records perm[lo:hi], by numpy gathers."""
    p = perm[lo:hi]
    size = (rec_off[1:] - rec_off[:-1]).astype(np.int64)[p]
    d0 = np.zeros(len(p), np.int64)
    d0[1:] = np.cumsum(size + 4)[:-1]
    out = np.empty(int(d0[-1] + size[-1] + 4), np.uint8)
    out[(d0[:, None] + np.arange(4)).ravel()] = size.astype("<u4").view(np.uint8)
    rs = np.zeros(len(p), np.int64)
    rs[1:] = np.cumsum(size)[:-1]
    within = np.arange(int(size.sum())) - np.repeat(rs, size)
    out[np.repeat(d0 + 4, size) + within] = bodies[np.repeat(rec_off[p].astype(np.int64), size) + within]
    return out


def assert_stream(out, bodies, rec_off, perm, chunk: int = 8 << 20) -> None:
    """out == the records in the order perm as [u32 block_size][record]..., compared in chunks of about `chunk` bytes;
    a difference names the first output record it is in."""
    so = stream_offsets(rec_off, perm)
    assert len(out) == so[-1], f"output of {len(out)} bytes, expected {so[-1]}"
    got = np.frombuffer(out, np.uint8)
    n = len(perm)
    a = 0
    while a < n:
        b = min(n, max(a + 1, int(np.searchsorted(so, so[a] + chunk, "right")) - 1))
        want = expected_stream(bodies, rec_off, perm, a, b)
        have = got[so[a]:so[b]]
        if not np.array_equal(have, want):
            d = int(np.flatnonzero(have != want)[0]) + int(so[a])
            i = int(np.searchsorted(so, d, "right")) - 1
            raise AssertionError(f"output record {i} (input record {int(perm[i])}, {int(so[i + 1] - so[i] - 4)} bytes) "
                                 f"differs at byte {d - int(so[i])} of its block (stream byte {d})")
        a = b


def run_plan(rec_off, budget: int, words: int):
    """The run boundaries fgb_sort_records chooses for `device_bytes = budget` (sort_host.cpp: records are added to
    a run while 2 x its bytes + its records x (68 + 8 words + 4) fit the budget, at least one per run)."""
    per = 68 + 8 * words + 4
    off = np.asarray(rec_off, np.int64)
    n = len(off) - 1
    g = 2 * off[1:] + np.arange(1, n + 1, dtype=np.int64) * per
    begin = [0]
    while begin[-1] < n:
        b = begin[-1]
        begin.append(min(n, max(b + 1, int(np.searchsorted(g, budget + 2 * off[b] + b * per, "right")))))
    return begin


def budget_for(rec_off, first_run_end: int, words: int) -> int:
    """The device_bytes whose first run is exactly the records [0, first_run_end)."""
    return int(2 * (int(rec_off[first_run_end]) - int(rec_off[0])) + first_run_end * (68 + 8 * words + 4))
