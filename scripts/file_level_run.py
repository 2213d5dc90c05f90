"""One file-level parity run (SURVEY section 8d / BASELINE.md section 2): a synthetic MI-grouped paired-end BAM file
with overlapping mates -> fgumi_b200 simplex with the overlapping-bases pre-pass ON -> consensus BAM file; the
output is read back and compared record by record with the record oracle run on the same groups
(`compare bams --mode content` semantics: same records in the same order, docs/compare-cli.md:33-55).
usage: python scripts/file_level_run.py [groups] [out_dir]     (needs a GPU; the oracle is the checker only)"""
import gzip
import os
import struct
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import fgumi_b200 as fg
from fgumi_b200 import bamio
from oracle import record_oracle as R
from tests import oracle_lib as O
from tests.bam_builder import make_record
from tests.test_record_oracle_kat import vote_fn

P, F1, F2, REV, MREV = R.PAIRED, R.FIRST_SEGMENT, R.LAST_SEGMENT, R.REVERSE, R.MATE_REVERSE
ACGT = np.frombuffer(b"ACGT", np.uint8)
COMP = bytes.maketrans(b"ACGTN", b"TGCAN")


def paired_groups(rng, n_groups, L=100):
    """FR pairs whose mates overlap by a random amount, a few read errors, varying qualities."""
    groups = []
    for g in range(n_groups):
        depth = int(rng.integers(1, 7))
        insert = int(rng.integers(L // 2 + 10, 2 * L + 20))
        tmpl = ACGT[rng.integers(0, 4, size=insert + L)].tobytes()
        start1 = 1000 + g * 7
        start2 = start1 + max(0, insert - L)
        recs = []
        for d in range(depth):
            def mut(seq):
                s = np.frombuffer(seq, np.uint8).copy()
                m = rng.random(len(s)) < 0.02
                s[m] = ACGT[rng.integers(0, 4, size=int(m.sum()))]
                return s.tobytes()
            q1 = rng.integers(8, 41, size=L).astype(np.uint8).tobytes()
            q2 = rng.integers(8, 41, size=L).astype(np.uint8).tobytes()
            tags = [(b"MI", "Z", b"%d" % g), (b"RX", "Z", b"ACGT-TTGA"), (b"MC", "Z", b"%dM" % L)]
            name = b"g%d_%d" % (g, d)
            recs.append(make_record(name=name, flags=P | F1 | MREV, pos=start1 - 1, mate_ref_id=0, mate_pos=start2 - 1,
                                    tlen=insert, seq=mut(tmpl[:L]), quals=q1, tags=tags))
            recs.append(make_record(name=name, flags=P | F2 | REV, pos=start2 - 1, mate_ref_id=0, mate_pos=start1 - 1,
                                    tlen=-insert, seq=mut(tmpl[start2 - start1:start2 - start1 + L]), quals=q2, tags=tags))
        groups.append(recs)
    return groups


def write_grouped_bam(path, groups, threads=4):
    text = b"@HD\tVN:1.6\tSO:unsorted\tGO:query\n@SQ\tSN:chr1\tLN:100000000\n@RG\tID:A\tSM:sample\tLB:lib\tPL:ILLUMINA\n@PG\tID:fgumi-group\tPN:fgumi\n"
    hdr = b"BAM\1" + struct.pack("<I", len(text)) + text + struct.pack("<I", 1) + struct.pack("<I", 5) + b"chr1\0" + struct.pack("<I", 100000000)
    body = b"".join(struct.pack("<I", len(r)) + r for g in groups for r in g)
    data = hdr + body
    open(path, "wb").write(fg.bgzf_compress(data, 1, threads, True))
    return len(data)


def read_bam_records(path):
    raw = gzip.open(path, "rb").read()            # BGZF is a sequence of gzip members
    assert raw[:4] == b"BAM\1"
    l_text = struct.unpack_from("<I", raw, 4)[0]
    p = 8 + l_text
    n_ref = struct.unpack_from("<I", raw, p)[0]
    assert n_ref == 0
    return raw[8:8 + l_text], raw[p + 4:]


def main():
    G = int(sys.argv[1]) if len(sys.argv) > 1 else 3000
    out_dir = sys.argv[2] if len(sys.argv) > 2 else os.path.join(tempfile.gettempdir(), "fgumi_file_level")
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(99)
    t0 = time.perf_counter()
    groups = paired_groups(rng, G)
    inp, outp = os.path.join(out_dir, "file_level_in.bam"), os.path.join(out_dir, "file_level_out.bam")
    nbytes = write_grouped_bam(inp, groups)
    print(f"input: {G} groups, {sum(len(g) for g in groups)} records, {nbytes} bytes uncompressed, "
          f"{os.path.getsize(inp)} on disk ({time.perf_counter() - t0:.1f} s to generate)")
    threads = min(16, len(os.sched_getaffinity(0)))
    caller = fg.VanillaUmiConsensusCaller("fgumi", "A", fg.VanillaUmiConsensusOptions(min_reads=1, min_consensus_base_quality=2),
                                          consensus_call_overlapping_bases=True, n_threads=threads)
    tm = bamio.simplex_file(inp, outp, caller, n_threads=threads)
    st = caller.statistics()
    caller.close()
    print("timings / sizes:", {k: (round(v, 4) if v < 1e3 else int(v)) for k, v in tm.items()})
    print(f"inflate {tm['uncompressed_bytes'] / tm['inflate_s'] / 1e6:.0f} MB/s on {threads} threads, "
          f"deflate {tm['output_bytes'] / tm['deflate_s'] / 1e6:.0f} MB/s (level 1)")
    # ---- the checker: the record oracle on the same groups, overlapping consensus on ----
    ov = R.OverlappingOracle()
    oc = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(min_reads=1, min_consensus_base_quality=2), vote_fn, O.builder_call)
    want = bytearray()
    for g in groups:
        recs = [bytearray(r) for r in g]
        ov.apply(recs)
        data, _ = oc.consensus_reads([bytes(r) for r in recs])
        want += data
    text, got = read_bam_records(outp)
    ok = bytes(want) == got
    print("header:", text.decode().strip().replace("\n", " | "))
    print(f"records: {int(tm['consensus_reads'])} consensus reads, {len(got)} bytes; identical to the oracle stream: {ok}")
    want_stats = ov.stats()
    got_stats = (st["overlapping_bases"], st["overlap_bases_agreeing"], st["overlap_bases_disagreeing"], st["overlap_bases_corrected"])
    print("overlap statistics (device pre-pass):", got_stats, "oracle:", want_stats, "equal:", tuple(want_stats) == got_stats)
    if not ok or tuple(want_stats) != got_stats:
        raise SystemExit(1)
    print("FILE-LEVEL PARITY OK")


if __name__ == "__main__":
    main()
