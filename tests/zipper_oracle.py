"""CPU restatement of `fgumi zipper` on raw BAM records, replaying the reference's edits literally (each remove_tag,
update_*_tag and append in the order the code runs them), so that the library's closed-form tag layout can be
compared against it.  Citations: zipper.rs = src/lib/commands/zipper.rs, template.rs = src/lib/template.rs, tags.rs =
crates/fgumi-raw-bam/src/tags.rs, cigar.rs = crates/fgumi-raw-bam/src/cigar.rs, umi = crates/fgumi-umi/src/lib.rs."""
import struct

# TagSets (umi lib.rs:200-210): the reference's list exactly, without ce
CONSENSUS_REVERSE = ["ad", "ae", "bd", "be", "cd"]
CONSENSUS_REVCOMP = ["aD", "bD", "cD"]
FIXED = {b"A": 1, b"c": 1, b"C": 1, b"s": 2, b"S": 2, b"i": 4, b"I": 4, b"f": 4}


def tag_info(remove, reverse, revcomp):
    """TagInfo::new (umi lib.rs:246-267): the name Consensus expands in the reverse and revcomp lists."""
    rev, rc = set(), set()
    for t in reverse:
        rev.update(CONSENSUS_REVERSE if t == "Consensus" else [t])
    for t in revcomp:
        rc.update(CONSENSUS_REVCOMP if t == "Consensus" else [t])
    return set(remove), rev, rc


def value_size(t, d):
    """tag_value_size (fields.rs:289-310); None for an unknown type or a cut-short value."""
    t = bytes([t])
    if t in FIXED:
        return FIXED[t]
    if t in (b"Z", b"H"):
        z = d.find(b"\0")
        return None if z < 0 else z + 1
    if t == b"B" and len(d) >= 5 and bytes(d[0:1]) in FIXED:
        return 5 + struct.unpack_from("<I", d, 1)[0] * FIXED[bytes(d[0:1])]
    return None


def aux_off(r):
    nc, L = struct.unpack_from("<HI", r, 12)[0], struct.unpack_from("<I", r, 16)[0]
    return 32 + r[8] + 4 * nc + (L + 1) // 2 + L


def flags(r):
    return struct.unpack_from("<H", r, 14)[0]


def set_flags(r, f):
    struct.pack_into("<H", r, 14, f)


def i32(r, at):
    return struct.unpack_from("<i", r, at)[0]


def set_i32(r, at, v):
    struct.pack_into("<i", r, at, v)


def name(r):
    return bytes(r[32:32 + r[8] - 1]) if r[8] else b""


def find_position(r, tag):
    """find_tag_position (tags.rs:13-34): (offset, type) of the first entry named tag."""
    p, a = aux_off(r), len(r)
    while p + 3 <= a:
        if r[p:p + 2] == tag:
            return p, r[p + 2]
        s = value_size(r[p + 2], r[p + 3:])
        if s is None:
            break
        p += 3 + s
    return None


def find_bounds(r, tag):
    """find_tag_bounds (tags.rs:79-84)."""
    f = find_position(r, tag)
    if f is None:
        return None
    s = value_size(f[1], r[f[0] + 3:])
    return None if s is None else (f[0], f[0] + 3 + s)


def find_int(r, tag):
    """find_int_tag (tags.rs:118-151)."""
    f = find_position(r, tag)
    if f is None:
        return None
    fmt = {ord("c"): "<b", ord("C"): "<B", ord("s"): "<h", ord("S"): "<H", ord("i"): "<i", ord("I"): "<I"}.get(f[1])
    if fmt is None or f[0] + 3 + struct.calcsize(fmt) > len(r):
        return None
    return struct.unpack_from(fmt, r, f[0] + 3)[0]


def remove_tag(r, tag):
    """remove_tag (tags.rs:670-683)."""
    b = find_bounds(r, tag)
    if b:
        del r[b[0]:b[1]]


def append_int(r, tag, v):
    """append_int_tag (tags.rs:533-553): unsigned preferred."""
    if -128 <= v <= 127:
        r += tag + b"c" + struct.pack("<b", v)
    elif 0 <= v <= 255:
        r += tag + b"C" + struct.pack("<B", v)
    elif 0 <= v <= 65535:
        r += tag + b"S" + struct.pack("<H", v)
    elif -32768 <= v <= 32767:
        r += tag + b"s" + struct.pack("<h", v)
    else:
        r += tag + b"i" + struct.pack("<i", v)


def append_signed(r, tag, v):
    """append_signed_int_tag (tags.rs:937-951)."""
    if -128 <= v <= 127:
        r += tag + b"c" + struct.pack("<b", v)
    elif -32768 <= v <= 32767:
        r += tag + b"s" + struct.pack("<h", v)
    else:
        r += tag + b"i" + struct.pack("<i", v)


def update_int(r, tag, v):
    """update_int_tag (tags.rs:729-750)."""
    b = find_bounds(r, tag)
    if b:
        if r[b[0] + 2] in b"iI" and b[1] - b[0] == 7:
            struct.pack_into("<i", r, b[0] + 3, v)
            return
        del r[b[0]:b[1]]
    append_int(r, tag, v)


def update_string(r, tag, val):
    """update_string_tag (tags.rs:694-721)."""
    b = find_bounds(r, tag)
    if b:
        if b[1] - b[0] - 4 == len(val):
            r[b[0] + 3:b[0] + 3 + len(val)] = val
        else:
            r[b[0]:b[1]] = tag + b"Z" + val + b"\0"
        return
    r += tag + b"Z" + val + b"\0"


def normalize(r, tag):
    """normalize_int_tag_to_smallest_signed (tags.rs:910-929)."""
    v = find_int(r, tag)
    if v is None or not -2 ** 31 <= v < 2 ** 31:
        return
    remove_tag(r, tag)
    append_signed(r, tag, v)


def complement(c):
    return {65: 84, 97: 84, 84: 65, 116: 65, 67: 71, 99: 71, 71: 67, 103: 67}.get(c, c)


def reverse_in_place(r, tag, typ, rc):
    """reverse / revcomp_tag_in_place_raw_by_type (zipper.rs:540-581, tags.rs:754-836) on the first entry named tag."""
    f = find_position(r, tag)
    if f is None or f[1] != typ:
        return
    p = f[0] + 3
    if typ == ord("Z"):
        e = r.index(b"\0", p)
        v = r[p:e][::-1]
        r[p:e] = bytes(complement(c) for c in v) if rc else v
    elif typ == ord("B"):
        es, n = FIXED[bytes(r[p:p + 1])], struct.unpack_from("<I", r, p + 1)[0]
        el = [r[p + 5 + k * es:p + 5 + (k + 1) * es] for k in range(n)]
        r[p + 5:p + 5 + n * es] = b"".join(el[::-1])


def cigar_ops(r):
    nc = struct.unpack_from("<H", r, 12)[0]
    return [struct.unpack_from("<I", r, 32 + r[8] + 4 * k)[0] for k in range(nc)]


def cigar_text(r):
    """cigar_to_string_from_raw (cigar.rs:115-129)."""
    return "".join("%d%s" % (o >> 4, "MIDNSHP=X"[o & 0xF]) for o in cigar_ops(r)).encode()


def ref_len(r):
    return sum(o >> 4 for o in cigar_ops(r) if o & 0xF in (0, 2, 3, 7, 8))


def w32(v):
    """i32 arithmetic as the reference's release build does it: wrapping."""
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


def insert_size(a, b):
    """compute_insert_size_raw (template.rs:714-746)."""
    if flags(a) & 4 or flags(b) & 4 or i32(a, 0) != i32(b, 0):
        return 0
    p1, p2 = w32(i32(a, 4) + 1), w32(i32(b, 4) + 1)
    f1 = w32(p1 + ref_len(a) - 1) if flags(a) & 0x10 else p1
    f2 = w32(p2 + ref_len(b) - 1) if flags(b) & 0x10 else p2
    return w32(f2 - f1 + (1 if f2 >= f1 else -1))


def unclipped_5prime(r):
    """unclipped_5prime_from_raw_bam (cigar.rs:201-228)."""
    f = flags(r)
    if f & 4:
        return 0
    ops = cigar_ops(r)
    if not ops:
        return 2 ** 31 - 1
    pos = w32(i32(r, 4) + 1)
    if not f & 0x10:
        clipped = 0
        for o in ops:
            if o & 0xF in (4, 5):
                clipped += o >> 4
            else:
                break
        return w32(pos - clipped)
    rl = trailing = 0
    saw = False
    for o in ops:
        if o & 0xF in (0, 2, 3, 7, 8):
            rl += o >> 4
            trailing = 0
            saw = True
        elif o & 0xF in (4, 5) and saw:
            trailing += o >> 4
    return w32(pos + rl + trailing - 1)


class Template:
    """Template::from_records (template.rs:159-330): R1, R2, then the R1 / R2 supplementary and the R1 / R2 secondary
    records, each list reversed."""

    def __init__(self, recs):
        self.name = name(recs[0])
        r1 = r2 = None
        lists = [[], [], [], []]
        for r in recs:
            f = flags(r)
            is_r1 = not f & 1 or f & 0x40
            if f & 0x100:
                lists[2 if is_r1 else 3].append(r)
            elif f & 0x800:
                lists[0 if is_r1 else 1].append(r)
            elif is_r1:
                if r1 is not None:
                    raise ValueError("Multiple non-secondary, non-supplemental R1 records for read '%s'" % self.name)
                r1 = r
            else:
                if r2 is not None:
                    raise ValueError("Multiple non-secondary, non-supplemental R2 records for read '%s'" % self.name)
                r2 = r
        self.records = [x for x in (r1, r2) if x is not None]
        self.r1 = 0 if r1 is not None else None
        self.r2 = (1 if r1 is not None else 0) if r2 is not None else None
        self.spans = []
        for lst in lists:
            s = len(self.records)
            self.records += lst[::-1]
            self.spans.append((s, len(self.records)))
        self.records = [bytearray(x) for x in self.records]

    def segment(self, first):
        """collect_mapped_indices (zipper.rs:337-361)."""
        p = self.r1 if first else self.r2
        out = [p] if p is not None else []
        sup, sec = (self.spans[0], self.spans[2]) if first else (self.spans[1], self.spans[3])
        return out + list(range(*sup)) + list(range(*sec))


def set_mate_flags(r, rev, unm):
    f = flags(r) & ~0x28
    set_flags(r, f | (0x20 if rev else 0) | (0x08 if unm else 0))


def fix_mate_info(t):
    """Template::fix_mate_info (template.rs:411-547)."""
    rr = t.records
    if not rr:
        return
    if t.r1 is not None and t.r2 is not None:
        a, b = rr[t.r1], rr[t.r2]
        au, bu = flags(a) & 4, flags(b) & 4
        a_as, b_as = find_int(a, b"AS"), find_int(b, b"AS")
        if not au and not bu:   # set_mate_info_both_mapped (:550-611)
            ins = insert_size(a, b)
            for x, y in ((a, b), (b, a)):
                set_i32(x, 20, i32(y, 0)); set_i32(x, 24, i32(y, 4))
                set_mate_flags(x, flags(y) & 0x10, False)
                update_int(x, b"MQ", y[9])
                c = cigar_text(y)
                update_string(x, b"MC", c) if c else remove_tag(x, b"MC")
            set_i32(a, 28, ins); set_i32(b, 28, w32(-ins))
        elif au and bu:         # set_mate_info_both_unmapped (:614-644)
            ar, br = flags(a) & 0x10, flags(b) & 0x10
            for x, yr in ((a, br), (b, ar)):
                for at in (0, 4, 20, 24):
                    set_i32(x, at, -1)
                set_mate_flags(x, yr, True)
                remove_tag(x, b"MQ"); remove_tag(x, b"MC")
                set_i32(x, 28, 0)
        else:                   # set_mate_info_one_unmapped (:647-693)
            m, u = (b, a) if au else (a, b)
            mref, mpos, mrev, mq, mc = i32(m, 0), i32(m, 4), flags(m) & 0x10, m[9], cigar_text(m)
            urev = flags(u) & 0x10
            set_i32(u, 0, mref); set_i32(u, 4, mpos)
            set_i32(m, 20, mref); set_i32(m, 24, mpos)
            set_mate_flags(m, urev, True)
            remove_tag(m, b"MQ"); remove_tag(m, b"MC")
            set_i32(m, 28, 0)
            set_i32(u, 20, mref); set_i32(u, 24, mpos)
            set_mate_flags(u, mrev, False)
            update_int(u, b"MQ", mq)
            update_string(u, b"MC", mc) if mc else remove_tag(u, b"MC")
            set_i32(u, 28, 0)
        for x, v in ((a, b_as), (b, a_as)):   # ms (:442-455)
            if v is not None and -2 ** 31 <= v < 2 ** 31:
                remove_tag(x, b"ms")
                append_signed(x, b"ms", v)
    for mate_i, span in ((t.r2, t.spans[0]), (t.r1, t.spans[1])):   # supplementary arms (:458-544)
        if mate_i is None:
            continue
        m = rr[mate_i]
        mref, mpos, mf, mtlen, mq, mc, mas = i32(m, 0), i32(m, 4), flags(m), i32(m, 28), m[9], cigar_text(m), \
            find_int(m, b"AS")
        for k in range(*span):
            x = rr[k]
            set_i32(x, 20, mref); set_i32(x, 24, mpos)
            set_mate_flags(x, mf & 0x10, mf & 4)
            set_i32(x, 28, w32(-mtlen))
            update_int(x, b"MQ", mq)
            update_string(x, b"MC", mc) if mc and not mf & 4 else remove_tag(x, b"MC")
            if mas is not None and -2 ** 31 <= mas < 2 ** 31:
                remove_tag(x, b"ms")
                append_signed(x, b"ms", mas)


def entries(r):
    """RawRecordView::tags() of a well-formed record: (tag, type, raw entry bytes)."""
    p, out = aux_off(r), []
    while p + 3 <= len(r):
        s = value_size(r[p + 2], r[p + 3:])
        out.append((bytes(r[p:p + 2]), r[p + 2], bytes(r[p:p + 3 + s])))
        p += 3 + s
    return out


def merge(u, m, info, skip_tc):
    """merge_raw (zipper.rs:373-521) of unmapped template u into mapped template m, in place."""
    remove, rev, rc = info
    fix_mate_info(m)
    for r in m.records:   # step 2
        for t in remove:
            if len(t) == 2:
                remove_tag(r, t.encode())
    for ui in [i for i in (u.r1, u.r2) if i is not None]:   # steps 3-4
        ur = u.records[ui]
        uf = flags(ur)
        idx = m.segment(not uf & 1 or bool(uf & 0x40))
        tags = entries(ur)
        for want_rev in (False, True):
            for i in idx:
                r = m.records[i]
                if bool(flags(r) & 0x10) != want_rev:
                    continue
                has_pg = find_position(r, b"PG") is not None
                for tag, typ, raw in tags:
                    if tag == b"PG" and has_pg:
                        continue
                    ts = tag.decode("latin-1")
                    if ts in remove:
                        continue
                    remove_tag(r, tag)
                    r += raw
                    if want_rev and (rev or rc):
                        if ts in rev:
                            reverse_in_place(r, tag, typ, False)
                        elif ts in rc:
                            reverse_in_place(r, tag, typ, typ == ord("Z"))
        for i in idx:
            r = m.records[i]
            set_flags(r, (flags(r) | 0x200) if uf & 0x200 else (flags(r) & ~0x200))
    for r in m.records:   # step 5
        normalize(r, b"AS")
        normalize(r, b"XS")
    if not skip_tc:       # step 6, add_template_coordinate_tags_raw (:259-332)
        if not any(flags(r) & 0x900 for r in m.records):
            return
        info_ = []
        for i in (m.r1, m.r2):
            if i is None or flags(m.records[i]) & 4:
                info_.append(None)
            else:
                r = m.records[i]
                info_.append((i32(r, 0), unclipped_5prime(r), int(bool(flags(r) & 0x10))))
        a, b = info_
        if a and b:
            v = a + b if (a[0], a[1]) <= (b[0], b[1]) else b + a
        elif a or b:
            v = (a or b) * 2
        else:
            return
        for r in m.records:
            if flags(r) & 0x900:
                remove_tag(r, b"tc")
                r += b"tcBi" + struct.pack("<I6i", 6, *v)


def runs(recs):
    out, i = [], 0
    while i < len(recs):
        j = i + 1
        while j < len(recs) and name(recs[j]) == name(recs[i]):
            j += 1
        out.append(recs[i:j])
        i = j
    return out


def zipper(unmapped, mapped, remove=(), reverse=(), revcomp=(), exclude_missing=False, skip_tc=False,
           last_call=True):
    """process_raw (zipper.rs:826-941) over record lists: (output records, mapped records consumed, stats
    [merged, unmapped-only, excluded, records out]).  Raises ValueError where the reference fails."""
    info = tag_info(remove, reverse, revcomp)
    mt = runs(mapped)
    out, k, consumed = [], 0, 0
    stats = [0, 0, 0, 0]
    for ur in runs(unmapped):
        u = Template(ur)
        m = Template(mt[k]) if k < len(mt) else None
        if m is not None and m.name == u.name:
            merge(u, m, info, skip_tc)
            out += [bytes(r) for r in m.records]
            consumed += len(mt[k])
            k += 1
            stats[0] += 1
        elif exclude_missing:
            stats[2] += 1
        else:
            out += [bytes(r) for r in u.records]
            stats[1] += 1
    if last_call and k < len(mt):
        raise ValueError("mapped reads remaining: '%s'" % name(mt[k][0]).decode())
    stats[3] = len(out)
    return out, consumed, stats


def stream(recs):
    return b"".join(struct.pack("<I", len(r)) + r for r in recs)


# ---- header (build_output_header, zipper.rs:210-256; add_pg_record) ---------------------------------------------

def _lines(text, kind):
    return [ln for ln in text.decode().split("\n") if ln.startswith(kind)]


def _id(ln):
    return next((f[3:] for f in ln.split("\t")[1:] if f.startswith("ID:")), None)


def output_header(unmapped_text, mapped_text, dict_text, command_line):
    """@HD from the unmapped header, @SQ from the dictionary, @RG / @PG mapped first then unmapped IDs not present, the
    new @PG last among the programs (add_pg_record adds it to the program map; its ID made unique with .1, .2, ...,
    PP = the last program no other names as PP), @CO unmapped then mapped; lines in noodles' order HD, SQ, RG, PG, CO."""
    out = _lines(unmapped_text, "@HD")[:1] + _lines(dict_text, "@SQ")
    for kind in ("@RG", "@PG"):
        seen = []
        for ln in _lines(mapped_text, kind) + _lines(unmapped_text, kind):
            if _id(ln) not in [_id(x) for x in seen]:
                seen.append(ln)
        out += seen
    pgs = [ln for ln in out if ln.startswith("@PG")]
    ids = [_id(ln) for ln in pgs]
    pp = {f[3:] for ln in pgs for f in ln.split("\t")[1:] if f.startswith("PP:")}
    last = next((i for i in reversed(ids) if i not in pp), ids[-1] if ids else None)
    uid, k = "fgumi_b200", 0
    while uid in ids:
        k += 1
        uid = "fgumi_b200.%d" % k
    out.append("@PG\tID:%s\tPN:fgumi_b200" % uid + ("\tPP:%s" % last if last else "") + "\tCL:" + command_line)
    out += _lines(unmapped_text, "@CO") + _lines(mapped_text, "@CO")
    return ("\n".join(out) + "\n").encode()
