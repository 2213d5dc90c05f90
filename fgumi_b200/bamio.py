"""File-level run of the consensus path (SURVEY section 8f N4): a grouped BAM file in, a consensus BAM file out.

    BGZF inflate (fgb_bgzf_decompress, members on threads) -> BAM header + record split -> MI grouping
    (fgb_host_group_by_mi) -> record-level caller (fgb_caller_add_groups + fgb_caller_flush: the GPU vote)
    -> output header + ConsensusOutput stream -> BGZF deflate (fgb_bgzf_compress)

What `fgumi simplex -i grouped.bam -o consensus.bam` does around the hot path (commands/simplex.rs,
consensus_runner.rs:120-163 for the header: one @RG, SO:unknown GO:query, @PG appended); everything heavy is
in the library, this module only strings the calls together.
"""
from __future__ import annotations

import ctypes as C
import time
from typing import Dict, Tuple

import numpy as np

from . import lib as _l


def read_bam(path: str, n_threads: int = 4) -> Tuple[bytes, np.ndarray, np.ndarray, Dict[str, float]]:
    """(SAM header text, record bodies uint8[...], rec_off uint64[n + 1], timings)."""
    lib = _l.load()
    t0 = time.perf_counter()
    comp = np.fromfile(path, dtype=np.uint8)
    size = C.c_size_t()
    st = lib.fgb_bgzf_uncompressed_size(comp.ctypes.data, len(comp), C.addressof(size))
    if st != 0:
        raise _l.FgbError(st, "fgb_bgzf_uncompressed_size")
    raw = np.empty(size.value + 16, dtype=np.uint8)
    n = C.c_size_t()
    t1 = time.perf_counter()
    st = lib.fgb_bgzf_decompress(comp.ctypes.data, len(comp), n_threads, raw.ctypes.data, size.value, C.addressof(n))
    if st != 0:
        raise _l.FgbError(st, "fgb_bgzf_decompress")
    t2 = time.perf_counter()
    toff, tlen, roff = C.c_size_t(), C.c_size_t(), C.c_size_t()
    nref = C.c_uint32()
    st = lib.fgb_bam_read_header(raw.ctypes.data, n.value, C.addressof(toff), C.addressof(tlen), C.addressof(nref), C.addressof(roff))
    if st != 0:
        raise _l.FgbError(st, "fgb_bam_read_header")
    text = raw[toff.value:toff.value + tlen.value].tobytes()
    stream = raw[roff.value:n.value]
    cap = max(1, len(stream) // 36)
    rec_off = np.zeros(cap + 1, dtype=np.uint64)
    nrec, used = C.c_uint64(), C.c_size_t()
    st = lib.fgb_bam_split_records(stream.ctypes.data, len(stream), stream.ctypes.data, rec_off.ctypes.data, cap,
                                   C.addressof(nrec), C.addressof(used))       # in place: bodies move down
    if st != 0:
        raise _l.FgbError(st, "fgb_bam_split_records")
    if used.value != len(stream):
        raise ValueError("truncated BAM record stream")
    t3 = time.perf_counter()
    timings = {"read_s": t1 - t0, "inflate_s": t2 - t1, "split_s": t3 - t2, "compressed_bytes": float(len(comp)),
               "uncompressed_bytes": float(n.value)}
    return text, stream[:int(rec_off[nrec.value])], rec_off[:nrec.value + 1], timings


def group_by_mi(bodies: np.ndarray, rec_off: np.ndarray, tag: bytes = b"MI", strip_strand_suffix: bool = False):
    """fgb_host_group_by_mi: group table over the kept records (all of them when every record has the tag)."""
    lib = _l.load()
    n = len(rec_off) - 1
    keep = np.zeros(max(n, 1), dtype=np.uint8)
    gb = np.zeros(n + 2, dtype=np.uint64)
    ng = C.c_uint64()
    st = lib.fgb_host_group_by_mi(bodies.ctypes.data, rec_off.ctypes.data, n, tag, int(strip_strand_suffix), None,
                                  keep.ctypes.data, gb.ctypes.data, C.addressof(ng))
    if st != 0:
        raise _l.FgbError(st, "fgb_host_group_by_mi")
    if int(keep[:n].sum()) != n:
        raise ValueError("records without the MI tag: drop them before calling (the table indexes kept records)")
    return gb[:ng.value + 1]


def output_header(input_text: bytes, read_group_id: str, command_line: str = "fgumi_b200 simplex") -> bytes:
    """consensus_runner.rs:120-163 in spirit: unsorted / query-grouped, one @RG carrying the inputs' SM / LB / PL
    (collapsed when they agree), one @CO, the inputs' @PG chain with ours appended."""
    fields = {}
    pgs = []
    for line in input_text.decode("utf-8", "replace").splitlines():
        if line.startswith("@RG"):
            for f in line.split("\t")[1:]:
                k, _, v = f.partition(":")
                if k in ("SM", "LB", "PL", "PU", "CN", "DS"):
                    fields.setdefault(k, set()).add(v)
        elif line.startswith("@PG"):
            pgs.append(line)
    rg = "@RG\tID:" + read_group_id + "".join("\t%s:%s" % (k, ",".join(sorted(v))) for k, v in sorted(fields.items()))
    out = ["@HD\tVN:1.6\tSO:unknown\tGO:query", rg, "@CO\tconsensus reads called by fgumi_b200"] + pgs
    out.append("@PG\tID:fgumi_b200\tPN:fgumi_b200\tCL:" + command_line)
    return ("\n".join(out) + "\n").encode()


def _write_bgzf(f, payload, level: int, n_threads: int, eof: bool = True) -> int:
    """payload (bytes, bytearray or a uint8 array) as BGZF members, with the EOF member when eof, written to the open
    file f; returns the compressed length."""
    lib = _l.load()
    src = np.frombuffer(payload, dtype=np.uint8)
    cap = lib.fgb_bgzf_bound(len(src))
    comp = np.empty(max(cap, 1), dtype=np.uint8)
    cn = C.c_size_t()
    st = lib.fgb_bgzf_compress(src.ctypes.data, len(src), level, n_threads, int(eof), comp.ctypes.data, cap,
                               C.addressof(cn))
    if st != 0:
        raise _l.FgbError(st, "fgb_bgzf_compress")
    f.write(comp[:cn.value])
    return cn.value


def simplex_file(in_path: str, out_path: str, caller, n_threads: int = 4, level: int = 1) -> Dict[str, float]:
    """One file-level run with an existing VanillaUmiConsensusCaller (its options decide everything else)."""
    lib = _l.load()
    text, bodies, rec_off, tm = read_bam(in_path, n_threads)
    t0 = time.perf_counter()
    groups = group_by_mi(bodies, rec_off)
    t1 = time.perf_counter()
    st = lib.fgb_caller_add_groups(caller._h, bodies.ctypes.data, rec_off.ctypes.data, groups.ctypes.data, len(groups) - 1)
    if st != 0:
        caller._check(st, "fgb_caller_add_groups")
    data, n, cnt = C.c_void_p(), C.c_uint64(), C.c_uint64()
    st = lib.fgb_caller_flush(caller._h, C.byref(data), C.byref(n), C.byref(cnt))
    if st != 0:
        caller._check(st, "fgb_caller_flush")
    t2 = time.perf_counter()
    hdr_text = output_header(text, caller._rg.decode() if hasattr(caller, "_rg") else "A")
    hdr = np.empty(len(hdr_text) + 16, dtype=np.uint8)
    hn = C.c_size_t()
    st = lib.fgb_bam_header(hdr_text, len(hdr_text), hdr.ctypes.data, len(hdr), C.addressof(hn))
    if st != 0:
        raise _l.FgbError(st, "fgb_bam_header")
    payload = np.empty(hn.value + n.value, dtype=np.uint8)
    payload[:hn.value] = hdr[:hn.value]
    if n.value:
        C.memmove(payload.ctypes.data + hn.value, data.value, n.value)
    t3 = time.perf_counter()
    with open(out_path, "wb") as f:
        cn = _write_bgzf(f, payload, level, n_threads)
    t4 = time.perf_counter()
    tm.update({"group_s": t1 - t0, "caller_s": t2 - t1, "deflate_s": t4 - t3, "input_records": float(len(rec_off) - 1),
               "groups": float(len(groups) - 1), "consensus_reads": float(cnt.value), "output_bytes": float(len(payload)),
               "output_compressed_bytes": float(cn)})
    return tm


def group_header(input_text: bytes, command_line: str = "fgumi_b200 group") -> bytes:
    """The input header with one @PG appended, chained by PP to the last program of the input's chain
    (header.rs:136-144): the last @PG no other @PG names as PP; its ID made unique with .1, .2, ..."""
    lines = input_text.decode("utf-8", "replace").rstrip("\n").split("\n") if input_text else []
    pgs = [dict(f.split(":", 1) for f in ln.split("\t")[1:] if ":" in f) for ln in lines if ln.startswith("@PG")]
    ids = [p.get("ID") for p in pgs]
    referenced = {p.get("PP") for p in pgs}
    last = next((i for i in reversed(ids) if i not in referenced), ids[-1] if ids else None)
    uid, k = "fgumi_b200", 0
    while uid in ids:
        k += 1
        uid = "fgumi_b200.%d" % k
    pg = "@PG\tID:%s\tPN:fgumi_b200" % uid + ("\tPP:%s" % last if last else "") + "\tCL:" + command_line
    return ("\n".join([ln for ln in lines if ln] + [pg]) + "\n").encode()


def sort_header(input_text: bytes, order: str, command_line: str = "fgumi_b200 sort") -> bytes:
    """`fgumi sort`'s output header (sort/mod.rs:72-129, raw.rs:1530-1535): the input header with one @PG chained as
    group_header chains it, then SO / GO / SS of the @HD line removed and set again -- SO:coordinate, SO:unsorted
    GO:query SS:template-coordinate, or SO:queryname with SS:lexicographic or SS:natural (no GO) -- keeping VN and the
    other @HD fields; an @HD line is created when there is none."""
    tags = {"coordinate": [("SO", "coordinate")],
            "template-coordinate": [("SO", "unsorted"), ("GO", "query"), ("SS", "template-coordinate")],
            "queryname": [("SO", "queryname"), ("SS", "lexicographic")],
            "queryname::natural": [("SO", "queryname"), ("SS", "natural")]}[order]
    lines = group_header(input_text, command_line).decode("utf-8", "replace").rstrip("\n").split("\n")
    at = next((i for i, ln in enumerate(lines) if ln.startswith("@HD")), None)
    fields = [] if at is None else [f for f in lines[at].split("\t")[1:] if f[:3] not in ("SO:", "GO:", "SS:")]
    hd = "\t".join(["@HD"] + fields + ["%s:%s" % kv for kv in tags])
    if at is None:
        lines.insert(0, hd)
    else:
        lines[at] = hd
    return ("\n".join(lines) + "\n").encode()


def sort_file(in_path: str, out_path: str, sorter, n_threads: int = 4, level: int = 1) -> Dict[str, float]:
    """`fgumi sort -i in.bam -o out.bam --order <sorter's order>` with an existing sort.RecordSorter.  Returns the
    phase timings: read / inflate / split (read_bam), device (the sort call, with the sorter's own phases), compress."""
    text, bodies, rec_off, tm = read_bam(in_path, n_threads)
    t0 = time.perf_counter()
    stream = sorter.sort(text, bodies, rec_off)
    t1 = time.perf_counter()
    payload = mapped_bam_header(sort_header(text, sorter.order)) + stream
    t2 = time.perf_counter()
    with open(out_path, "wb") as f:
        _write_bgzf(f, payload, level, n_threads)
    t3 = time.perf_counter()
    tm.update({"device_s": t1 - t0, "compress_s": t3 - t2, "input_records": float(len(rec_off) - 1),
               "output_bytes": float(len(payload))})
    tm.update({k: v for k, v in sorter.last_timing().items()})
    return tm


def check_group_sort_order(text: bytes, allow_unmapped: bool) -> None:
    """group.rs:797-817: template-coordinate input (SO:unsorted GO:query, SS ending in template-coordinate if
    present), or queryname-sorted input with --allow-unmapped."""
    hd = next((ln for ln in text.decode("utf-8", "replace").split("\n") if ln.startswith("@HD")), "")
    f = dict(x.split(":", 1) for x in hd.split("\t")[1:] if ":" in x)
    tc = f.get("SO") == "unsorted" and f.get("GO") == "query" and ("SS" not in f or
                                                                    f["SS"].rsplit(":", 1)[-1] == "template-coordinate")
    if not (tc or (allow_unmapped and f.get("SO") == "queryname")):
        raise ValueError("input BAM must be template-coordinate sorted" +
                         (" or queryname sorted when unmapped reads are allowed" if allow_unmapped else ""))


def mapped_bam_header(text: bytes) -> bytes:
    """The binary BAM header of `text` with its reference list taken from the @SQ lines (SAM spec 4.2)."""
    import struct
    out = [b"BAM\1", struct.pack("<i", len(text)), text]
    sq = []
    for ln in text.split(b"\n"):
        if ln.startswith(b"@SQ"):
            f = dict(x.split(b":", 1) for x in ln.split(b"\t")[1:] if b":" in x)
            sq.append((f[b"SN"], int(f[b"LN"])))
    out.append(struct.pack("<i", len(sq)))
    for nm, ln in sq:
        out.append(struct.pack("<i", len(nm) + 1) + nm + b"\0" + struct.pack("<i", ln))
    return b"".join(out)


def group_records(text: bytes, bodies: np.ndarray, rec_off: np.ndarray, grouper, cell_tag: bytes = b"CB") -> bytes:
    """`fgumi group` on a record stream in memory: position grouping, then the grouper; the MI-tagged stream
    ([u32 block_size][record]...)."""
    from .group import compact, group_by_position
    keep, groups = group_by_position(bodies, rec_off, text, cell_tag)
    bodies, rec_off = compact(bodies, rec_off, keep)
    grouper.add_groups(bodies, rec_off, groups)
    return grouper.flush()


def group_file(in_path: str, out_path: str, grouper, n_threads: int = 4, level: int = 1,
               cell_tag: bytes = b"CB") -> Dict[str, float]:
    """`fgumi group -i mapped.bam -o grouped.bam` with an existing ReadGrouper (its options decide the rest)."""
    text, bodies, rec_off, tm = read_bam(in_path, n_threads)
    check_group_sort_order(text, grouper.opt.umi.rules == _l.FGB_UMI_RULES_UNMAPPED)
    t0 = time.perf_counter()
    stream = group_records(text, bodies, rec_off, grouper, cell_tag)
    t1 = time.perf_counter()
    payload = mapped_bam_header(group_header(text)) + stream
    with open(out_path, "wb") as f:
        _write_bgzf(f, payload, level, n_threads)
    tm.update({"group_s": t1 - t0, "input_records": float(len(rec_off) - 1), "output_bytes": float(len(payload))})
    return tm


def dedup_records(text: bytes, bodies: np.ndarray, rec_off: np.ndarray, deduper, cell_tag: bytes = b"CB") -> bytes:
    """`fgumi dedup` on a template-coordinate-sorted record stream in memory: position grouping that keeps secondary
    and supplementary records, then the deduper; the MI-tagged stream with duplicates flagged 0x400 (or removed)."""
    from .dedup import group_by_position
    check_group_sort_order(text, False)   # is_template_coordinate_sorted (dedup.rs:971-978)
    _, groups = group_by_position(bodies, rec_off, text, cell_tag)
    deduper.add_groups(bodies, rec_off, groups)
    return deduper.flush()


def dedup_file(in_path: str, out_path: str, deduper, n_threads: int = 4, level: int = 1,
               cell_tag: bytes = b"CB") -> Dict[str, float]:
    """`fgumi dedup -i sorted.bam -o deduped.bam` with an existing dedup.Deduper (its options decide the rest).  Like
    the reference (dedup.rs:1167-1179) it raises ValueError after writing the output when secondary or supplementary
    records of this input lack the `tc` tag; the deduper may be reused across inputs."""
    text, bodies, rec_off, tm = read_bam(in_path, n_threads)
    missing_before = deduper.stats()["missing_tc_tag"]   # a deduper may have run on other input before
    t0 = time.perf_counter()
    stream = dedup_records(text, bodies, rec_off, deduper, cell_tag)
    t1 = time.perf_counter()
    payload = mapped_bam_header(group_header(text, "fgumi_b200 dedup")) + stream
    with open(out_path, "wb") as f:
        _write_bgzf(f, payload, level, n_threads)
    tm.update({"dedup_s": t1 - t0, "input_records": float(len(rec_off) - 1), "output_bytes": float(len(payload))})
    missing = deduper.stats()["missing_tc_tag"] - missing_before
    if missing:
        raise ValueError(f"{missing} secondary/supplementary reads are missing the `tc` tag, which correct UMI-aware "
                         "deduplication of secondary and supplementary alignments needs (`fgumi zipper` adds it)")
    return tm


def split_stream(stream: bytes) -> Tuple[np.ndarray, np.ndarray]:
    """[u32 block_size][record]... -> (record bodies back to back, rec_off) through fgb_bam_split_records."""
    lib = _l.load()
    buf = np.frombuffer(stream, np.uint8).copy() if stream else np.zeros(1, np.uint8)
    cap = max(1, len(stream) // 36)
    rec_off = np.zeros(cap + 1, np.uint64)
    n, used = C.c_uint64(), C.c_size_t()
    st = lib.fgb_bam_split_records(buf.ctypes.data, len(stream), buf.ctypes.data, rec_off.ctypes.data, cap,
                                   C.addressof(n), C.addressof(used))
    if st != 0:
        raise _l.FgbError(st, "fgb_bam_split_records")
    if used.value != len(stream):
        raise ValueError("truncated record stream")
    return buf[:int(rec_off[n.value])], rec_off[:n.value + 1]


def group_and_call(in_path: str, grouper, caller, n_threads: int = 4, cell_tag: bytes = b"CB"):
    """Mapped BAM -> `group` -> `simplex` or `duplex`, in memory: the grouper's MI-tagged stream goes through the MI
    grouping (fgb_host_group_by_mi; the base MI for a DuplexConsensusCaller) into the caller, whose ConsensusOutput
    is returned.  Records the grouper left without an MI (templates without a molecule) are not passed on, as the MI
    grouping of `simplex` / `duplex` skips them."""
    from .caller import ConsensusOutput, DuplexConsensusCaller
    from .group import compact
    lib = _l.load()
    text, bodies, rec_off, _ = read_bam(in_path, n_threads)
    check_group_sort_order(text, grouper.opt.umi.rules == _l.FGB_UMI_RULES_UNMAPPED)
    gb, goff = split_stream(group_records(text, bodies, rec_off, grouper, cell_tag))
    n = len(goff) - 1
    keep = np.zeros(max(n, 1), np.uint8)
    begin = np.zeros(n + 2, np.uint64)
    ng = C.c_uint64()
    st = lib.fgb_host_group_by_mi(gb.ctypes.data, goff.ctypes.data, n, bytes(grouper.opt.assign_tag),
                                  int(isinstance(caller, DuplexConsensusCaller)), None, keep.ctypes.data,
                                  begin.ctypes.data, C.addressof(ng))
    if st != 0:
        raise _l.FgbError(st, "fgb_host_group_by_mi")
    gb, goff = compact(gb, goff, keep[:n])
    st = lib.fgb_caller_add_groups(caller._h, gb.ctypes.data, goff.ctypes.data, begin.ctypes.data, ng.value)
    caller._check(st, "fgb_caller_add_groups")
    data, ln, cnt = C.c_void_p(), C.c_uint64(), C.c_uint64()
    caller._check(lib.fgb_caller_flush(caller._h, C.byref(data), C.byref(ln), C.byref(cnt)), "fgb_caller_flush")
    return ConsensusOutput(C.string_at(data.value, ln.value) if ln.value else b"", cnt.value)


def qname_batches(bodies: np.ndarray, rec_off: np.ndarray, batch_records: int):
    """[begin, end) record ranges of about batch_records records each, every cut at a QNAME change, so that each
    range holds whole templates."""
    n = len(rec_off) - 1
    name = lambda i: bytes(bodies[int(rec_off[i]) + 32:int(rec_off[i]) + 32 + int(bodies[int(rec_off[i]) + 8])])
    b = 0
    while b < n:
        e = min(n, b + max(1, batch_records))
        while e < n and name(e) == name(e - 1):
            e += 1
        yield b, e
        b = e


def filter_file(in_path: str, out_path: str, record_filter, reference=None, rejects: str = None, stats: str = None,
                n_threads: int = 4, level: int = 1, batch_records: int = 1_000_000) -> Dict[str, float]:
    """`fgumi filter -i in.bam -o out.bam [--ref ref.fa] [--rejects rejects.bam] [--stats stats.txt]` with an existing
    filter.RecordFilter (its options decide the rest; rejects need it made with track_rejects=True) and an optional
    filter.Reference.  Both outputs get the input header with one @PG.  The input is read into memory whole; it is
    filtered in batches of about batch_records records cut at QNAME changes, and each batch's output is compressed and
    written before the next, so that the outputs are never held whole.  A failing batch raises with
    record_filter.bad_record set to the index in the whole input."""
    from .filter import filter_stats_text
    text, bodies, rec_off, tm = read_bam(in_path, n_threads)
    header = mapped_bam_header(group_header(text, "fgumi_b200 filter"))
    outs = [(open(path, "wb"), header) for path in (out_path, rejects) if path is not None]

    counts = {"total": 0, "passed": 0, "failed": 0, "bases_masked": 0}
    t_filter = out_bytes = 0.0
    try:
        for b, e in qname_batches(bodies, rec_off, batch_records):
            t0 = time.perf_counter()
            try:
                kept, rej, c = record_filter.filter(text, bodies[int(rec_off[b]):int(rec_off[e])],
                                                    rec_off[b:e + 1] - rec_off[b], reference)
            except Exception:
                if record_filter.bad_record is not None:
                    record_filter.bad_record += b
                raise
            t_filter += time.perf_counter() - t0
            for k in counts:
                counts[k] += c[k]
            out_bytes += len(kept)
            for k, stream in enumerate((kept, rej)[:len(outs)]):
                _write_bgzf(outs[k][0], outs[k][1] + stream, level, n_threads, False)
                outs[k] = (outs[k][0], b"")   # the header goes with the first batch only
        for k in range(len(outs)):
            _write_bgzf(outs[k][0], outs[k][1], level, n_threads)   # the header of an empty input, and the EOF member
    finally:
        for f, _ in outs:
            f.close()
    if stats is not None:
        with open(stats, "w") as f:
            f.write(filter_stats_text(counts))
    tm.update({"filter_s": t_filter, "input_records": float(len(rec_off) - 1), "output_bytes": float(out_bytes)})
    tm.update({k: float(v) for k, v in counts.items()})
    return tm


_METRICS_SUFFIX = {"family_sizes": ".family_sizes.txt", "duplex_family_sizes": ".duplex_family_sizes.txt",
                   "umi_counts": ".umi_counts.txt", "duplex_umi_counts": ".duplex_umi_counts.txt"}


def _metrics_file(in_path: str, prefix: str, duplex: bool, intervals: str, n_threads: int, batch_records: int,
                  device: int, **opts) -> Dict[str, float]:
    from .metrics import MetricsCollector
    text, bodies, rec_off, tm = read_bam(in_path, n_threads)
    iv = None
    if intervals is not None:
        with open(intervals, "rb") as f:
            iv = f.read()
    m = MetricsCollector(text, duplex=duplex, intervals=iv, device=device, n_threads=n_threads, **opts)
    t0 = time.perf_counter()
    try:
        for b, e in qname_batches(bodies, rec_off, batch_records):   # bad_record counts over every call already
            m.add_records(bodies[int(rec_off[b]):int(rec_off[e])], rec_off[b:e + 1] - rec_off[b])
        tables = m.finish()
        tm["metrics_s"] = time.perf_counter() - t0
        tm.update({k: float(v) for k, v in m.stats().items()})
    finally:
        m.close()
    suffix = dict(_METRICS_SUFFIX, yield_metrics=".duplex_yield_metrics.txt" if duplex else ".simplex_yield_metrics.txt")
    for name, body in tables.items():
        with open(prefix + suffix[name], "w") as f:
            f.write(body)
    return tm


def duplex_metrics_file(in_path: str, prefix: str, intervals: str = None, min_ab_reads: int = 1, min_ba_reads: int = 1,
                        duplex_umi_counts: bool = False, n_threads: int = 4, batch_records: int = 1_000_000,
                        device: int = 0) -> Dict[str, float]:
    """`fgumi duplex-metrics -i in.bam -o prefix [-l intervals] [--min-ab-reads] [--min-ba-reads]
    [--duplex-umi-counts]`: writes <prefix>.family_sizes.txt, .duplex_family_sizes.txt, .duplex_yield_metrics.txt,
    .umi_counts.txt and, with duplex_umi_counts, .duplex_umi_counts.txt.  The input is read into memory whole and fed
    in batches cut at QNAME changes; a failure raises metrics.MetricsError naming the record in the whole input."""
    return _metrics_file(in_path, prefix, True, intervals, n_threads, batch_records, device,
                         min_ab_reads=min_ab_reads, min_ba_reads=min_ba_reads, duplex_umi_counts=duplex_umi_counts)


def simplex_metrics_file(in_path: str, prefix: str, intervals: str = None, min_reads: int = 1, n_threads: int = 4,
                         batch_records: int = 1_000_000, device: int = 0) -> Dict[str, float]:
    """`fgumi simplex-metrics -i in.bam -o prefix [-l intervals] [--min-reads]`: writes <prefix>.family_sizes.txt,
    .simplex_yield_metrics.txt and .umi_counts.txt, as duplex_metrics_file does."""
    return _metrics_file(in_path, prefix, False, intervals, n_threads, batch_records, device, min_reads=min_reads)


def find_dict_path(reference_path: str) -> str:
    """find_dict_path (reference.rs): ref.dict beside ref.fa, then ref.fa.dict."""
    import os
    for p in (os.path.splitext(reference_path)[0] + ".dict", reference_path + ".dict"):
        if os.path.exists(p):
            return p
    raise FileNotFoundError(f"reference dictionary not found for {reference_path}: tried "
                            f"{os.path.splitext(reference_path)[0]}.dict and {reference_path}.dict")


def zipper_header(unmapped_text: bytes, mapped_text: bytes, dict_text: bytes,
                  command_line: str = "fgumi_b200 zipper") -> bytes:
    """build_output_header (zipper.rs:210-256), then one @PG chained as group_header chains it: @HD from the unmapped
    header, @SQ from the sequence dictionary, @RG and @PG from the mapped header first and the unmapped IDs not already
    present after them and the new @PG last among them, @CO from the unmapped header then the mapped one; lines kept
    verbatim, in the order HD, SQ, RG, PG, CO."""
    def lines(text, kind):
        return [ln for ln in text.decode("utf-8", "replace").split("\n") if ln.startswith(kind)]

    def ident(ln):
        return next((f[3:] for f in ln.split("\t")[1:] if f.startswith("ID:")), None)

    out = lines(unmapped_text, "@HD")[:1] + lines(dict_text, "@SQ")
    for kind in ("@RG", "@PG"):
        kept, seen = [], set()
        for ln in lines(mapped_text, kind) + lines(unmapped_text, kind):
            if ident(ln) not in seen:
                seen.add(ident(ln))
                kept.append(ln)
        out += kept
    # add_pg_record puts the program into the header's program map, which noodles writes before the comments
    head = group_header(("\n".join(out) + "\n").encode() if out else b"", command_line)
    comments = lines(unmapped_text, "@CO") + lines(mapped_text, "@CO")
    return head + ("\n".join(comments) + "\n").encode() if comments else head


def _check_sort(text: bytes, what: str) -> None:
    """check_sort: a header that is not queryname-sorted only warns."""
    import warnings
    hd = next((ln for ln in text.decode("utf-8", "replace").split("\n") if ln.startswith("@HD")), "")
    if "SO:queryname" not in hd.split("\t"):
        warnings.warn(f"the {what} input does not declare SO:queryname; its templates must still be grouped by name "
                      "in the same order as the other input")


def zipper_file(unmapped_path: str, mapped_path: str, reference_path: str, out_path: str, zipper, n_threads: int = 4,
                level: int = 1, batch_records: int = 1_000_000,
                command_line: str = "fgumi_b200 zipper") -> Dict[str, float]:
    """`fgumi zipper -u unmapped.bam -i mapped.bam -r ref.fa -o out.bam` with an existing zipper.Zipper (its options
    decide the rest).  The mapped input must be BAM; the sequence dictionary beside the reference gives the @SQ lines.
    Both inputs are read into memory whole; the unmapped stream is zipped in batches of about batch_records records
    cut at QNAME changes, each call taking the mapped records the previous calls left, and each batch's output is
    compressed and written before the next.  A failing batch raises with zipper.bad_record set to the index in the
    whole unmapped input, or the number of unmapped records plus the index in the whole mapped input."""
    with open(find_dict_path(reference_path), "rb") as f:
        dict_text = f.read()
    ut, ub, uo, tm = read_bam(unmapped_path, n_threads)
    mt, mb, mo, _ = read_bam(mapped_path, n_threads)
    _check_sort(ut, "unmapped")
    _check_sort(mt, "mapped")
    header = mapped_bam_header(zipper_header(ut, mt, dict_text, command_line))
    n_u, n_m = len(uo) - 1, len(mo) - 1
    counts = dict.fromkeys(_l.ZIPPER_STAT_NAMES, 0)
    t_zip = out_bytes = 0.0
    m0 = 0
    batches = list(qname_batches(ub, uo, batch_records)) or [(0, 0)]
    with open(out_path, "wb") as f:
        for k, (b, e) in enumerate(batches):
            t0 = time.perf_counter()
            try:
                # offsets are relative to the bodies passed: views, no copy of the remaining mapped offsets
                data, used, c = zipper.zip(ub, uo[b:e + 1], mb, mo[m0:], last_call=k == len(batches) - 1)
            except Exception:
                if zipper.bad_record is not None:
                    r = zipper.bad_record
                    zipper.bad_record = b + r if r < e - b else n_u + m0 + (r - (e - b))
                raise
            t_zip += time.perf_counter() - t0
            m0 += used
            for key in counts:
                counts[key] += c[key]
            out_bytes += len(data)
            _write_bgzf(f, header + data, level, n_threads, False)
            header = b""
        _write_bgzf(f, header, level, n_threads)
    assert m0 == n_m
    tm.update({"zipper_s": t_zip, "input_records": float(n_u + n_m), "output_bytes": float(out_bytes)})
    tm.update({key: float(v) for key, v in counts.items()})
    return tm
