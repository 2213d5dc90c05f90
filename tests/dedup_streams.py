"""Seeded template-coordinate-sorted streams for the `dedup` tests: synth.mapped_templates with its supplementary and
secondary records, then edits a real input has and the generator does not make -- records flagged 0x400 already,
qualities below 15 (the cap of the template score, so that scores differ within a family), existing MI tags of other
lengths and types, signed and oversized mate MQ values, tc tags on some secondary and
supplementary records, those records moved before their primaries, and orphan supplementary records alone at the start
and between position groups."""
from __future__ import annotations

import struct

import numpy as np


def records_of(bodies, off):
    return [bodies[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def pack(records):
    off = np.zeros(len(records) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in records])
    return np.frombuffer(b"".join(records) or b"\0", np.uint8)[:int(off[-1])].copy(), off


def _name(r):
    return r[32:32 + r[8] - 1]


def _orphan(name, pos):
    """A supplementary record of a read whose primaries are elsewhere, with a tc tag."""
    return (struct.pack("<iiBBHHHIiii", 0, pos, len(name) + 1, 60, 4680, 1, 0x1 | 0x40 | 0x800, 4, -1, -1, 0) + name +
            b"\0" + struct.pack("<I", 4 << 4) + b"\x12\x48" + bytes([30] * 4) + b"tcZx\0")


def edit(records, seed):
    rng = np.random.default_rng(seed)
    out = []
    for r in records:
        r = bytearray(r)
        f = struct.unpack_from("<H", r, 14)[0]
        if rng.random() < 0.6:   # qualities below the cap of 15, so that the template scores differ
            n_cig, l_seq = struct.unpack_from("<H", r, 12)[0], struct.unpack_from("<I", r, 16)[0]
            qo = 32 + r[8] + 4 * n_cig + (l_seq + 1) // 2
            q = np.frombuffer(bytes(r[qo:qo + l_seq]), np.uint8).copy()
            low = rng.random(l_seq) < 0.5
            q[low] = rng.integers(0, 15, size=int(low.sum()), dtype=np.uint8)
            r[qo:qo + l_seq] = q.tobytes()
        if rng.random() < 0.15:
            struct.pack_into("<H", r, 14, f | 0x400)
        mq = r.find(b"MQi", 32)
        if mq > 0 and rng.random() < 0.2:   # a mate MQ the filter reads signed (MQ:c:-1) or without wrapping (300)
            kind = int(rng.integers(0, 3))
            if kind == 0:
                r[mq:mq + 7] = b"MQc" + struct.pack("<b", -1) + b"XYC" + bytes([0])   # MQ:c:-1, then XY:C:0
            elif kind == 1:
                r[mq + 3:mq + 7] = struct.pack("<i", 300)
            else:
                r[mq + 3:mq + 7] = struct.pack("<i", 256)
        if rng.random() < 0.2:
            r += [b"MIZ9\0", b"MIZ12345\0", b"MIZ\0", b"MIi" + struct.pack("<i", 7), b"MIC\x07"][int(rng.integers(0, 5))]
        if f & 0x900 and rng.random() < 0.5:
            r += b"tci" + struct.pack("<i", 1)
        out.append(bytes(r))
    # move a template's secondary / supplementary records before its primaries, sometimes
    i, moved = 0, []
    while i < len(out):
        j = i + 1
        while j < len(out) and _name(out[j]) == _name(out[i]):
            j += 1
        run = out[i:j]
        if rng.random() < 0.5:
            extra = [r for r in run if struct.unpack_from("<H", r, 14)[0] & 0x900]
            run = extra + [r for r in run if not struct.unpack_from("<H", r, 14)[0] & 0x900]
        moved += run
        i = j
    # orphans: two at the start (they share the default key), and some between templates
    final = [_orphan(b"orphan_a", 10), _orphan(b"orphan_b", 20)]
    for k, r in enumerate(moved):
        if k and _name(r) != _name(moved[k - 1]) and rng.random() < 0.03:
            final.append(_orphan(b"orphan_%d" % k, 30 + k))
        final.append(r)
    return final
