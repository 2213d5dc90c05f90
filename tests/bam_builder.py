"""Test helper: build raw BAM records (no block_size prefix), like the reference's SamBuilder
(fgumi-raw-bam/src/builder.rs:285) does for its unit tests."""
import struct

SEQ_CODE = {c: i for i, c in enumerate(b"=ACMGRSVTWYHKDBN")}
CIGAR_OPS = "MIDNSHP=X"
B_FORMATS = {"Bc": "b", "BC": "B", "Bs": "h", "BS": "H", "Bi": "i", "BI": "I", "Bf": "f"}


def encode_op(op: int, length: int) -> int:
    return (length << 4) | op


def cigar_from_string(s: str):
    ops, num = [], ""
    for ch in s:
        if ch.isdigit():
            num += ch
        else:
            ops.append(encode_op(CIGAR_OPS.index(ch), int(num)))
            num = ""
    return ops


def make_record(name=b"r", flags=0, ref_id=0, pos=0, mapq=60, cigar=None, mate_ref_id=-1, mate_pos=-1,
                tlen=0, seq=b"", quals=None, tags=()):
    """tags: sequence of (b"XX", type, value): "A" (one byte), "Z" / "H" (bytes), "c" "C" "s" "S" "i" "I" "f" (a
    number), "Bc" "BC" "Bs" "BS" "Bi" "BI" "Bf" (a list of numbers), or "raw": the tag, then `value`'s bytes as they
    are -- the type byte and value of an entry that may be malformed or cut short."""
    cigar = cigar if cigar is not None else ([encode_op(0, len(seq))] if len(seq) else [])
    if isinstance(cigar, str):
        cigar = cigar_from_string(cigar)
    quals = bytes([30] * len(seq)) if quals is None else bytes(quals)
    rec = bytearray(struct.pack("<iiBBHHHIiii", ref_id, pos, len(name) + 1, mapq, 4680, len(cigar), flags,
                                len(seq), mate_ref_id, mate_pos, tlen))
    rec += name + b"\0"
    for op in cigar:
        rec += struct.pack("<I", op)
    for i in range(0, len(seq) - 1, 2):
        rec.append((SEQ_CODE.get(seq[i] & 0xDF if chr(seq[i]).isalpha() else seq[i], 15) << 4) |
                   SEQ_CODE.get(seq[i + 1] & 0xDF if chr(seq[i + 1]).isalpha() else seq[i + 1], 15))
    if len(seq) % 2:
        c = seq[-1]
        rec.append(SEQ_CODE.get(c & 0xDF if chr(c).isalpha() else c, 15) << 4)
    rec += quals
    for tag, typ, val in tags:
        rec += tag
        if typ in ("Z", "H"):
            rec += typ.encode() + bytes(val) + b"\0"
        elif typ == "A":
            rec += b"A" + bytes(val)[:1]
        elif typ == "raw":
            rec += bytes(val)
        elif typ == "i":
            rec += b"i" + struct.pack("<i", val)
        elif typ == "C":
            rec += b"C" + struct.pack("<B", val)
        elif typ in ("c", "s", "S", "I"):
            rec += typ.encode() + struct.pack({"c": "<b", "s": "<h", "S": "<H", "I": "<I"}[typ], val)
        elif typ == "f":
            rec += b"f" + struct.pack("<f", val)
        elif typ in B_FORMATS:
            rec += typ.encode() + struct.pack("<I", len(val)) + struct.pack("<%d%s" % (len(val), B_FORMATS[typ]), *val)
        else:
            raise ValueError(typ)
    return bytes(rec)


def parse_records(data: bytes):
    """Split a ConsensusOutput byte stream into record dicts (name, flags, bases, quals, tags)."""
    out, p = [], 0
    while p < len(data):
        (bs,) = struct.unpack_from("<I", data, p)
        rec = data[p + 4:p + 4 + bs]
        p += 4 + bs
        (ref_id, pos, l_rn, mapq, bin_, n_cig, flag, l_seq, mref, mpos, tlen) = struct.unpack_from("<iiBBHHHIiii", rec, 0)
        q = 32
        name = rec[q:q + l_rn - 1]; q += l_rn + 4 * n_cig
        packed = rec[q:q + (l_seq + 1) // 2]; q += (l_seq + 1) // 2
        bases = bytes(b"=ACMGRSVTWYHKDBN"[(packed[i // 2] >> 4) if i % 2 == 0 else (packed[i // 2] & 0xF)]
                      for i in range(l_seq))
        quals = rec[q:q + l_seq]; q += l_seq
        tags = {}
        order = []
        while q < len(rec):
            tag, typ = rec[q:q + 2], chr(rec[q + 2]); q += 3
            if typ == "Z":
                e = rec.index(b"\0", q); val = rec[q:e]; q = e + 1
            elif typ in "cC":
                val = struct.unpack_from("<b" if typ == "c" else "<B", rec, q)[0]; q += 1
            elif typ in "sS":
                val = struct.unpack_from("<h" if typ == "s" else "<H", rec, q)[0]; q += 2
            elif typ in "iI":
                val = struct.unpack_from("<i" if typ == "i" else "<I", rec, q)[0]; q += 4
            elif typ == "f":
                val = struct.unpack_from("<f", rec, q)[0]; q += 4
            elif typ == "B":
                sub = chr(rec[q]); n = struct.unpack_from("<I", rec, q + 1)[0]; q += 5
                fmt = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}[sub]
                val = list(struct.unpack_from("<%d%s" % (n, fmt), rec, q)); q += n * struct.calcsize(fmt)
            else:
                raise ValueError(typ)
            tags[bytes(tag)] = val
            order.append(bytes(tag))
        out.append(dict(name=bytes(name), flags=flag, ref_id=ref_id, pos=pos, bases=bases, quals=bytes(quals),
                        tags=tags, tag_order=order, bin=bin_, mapq=mapq, n_cigar=n_cig, mate_ref_id=mref,
                        mate_pos=mpos, tlen=tlen))
    return out
