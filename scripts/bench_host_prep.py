"""Host-prep throughput of the record-level callers on the CPU alone (planning-only callers, no vote): input
reads per second of fgb_caller_add_groups.  Simplex measures the product's simplex planning: the staging copy
of the records plus the header-only group decisions (the rows are built on the device later); duplex and CODEC
measure group rules + source-read decode + packing."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import fgumi_b200 as fg
from tests.bam_builder import make_record

rng = np.random.default_rng(3)
G, D, L = int(sys.argv[1]) if len(sys.argv) > 1 else 5000, 8, 150
P, F1, F2, REV, MREV = 1, 0x40, 0x80, 0x10, 0x20
acgt = np.frombuffer(b"ACGT", np.uint8)
recs = []
for g in range(G):
    tmpl = acgt[rng.integers(0, 4, size=400)].tobytes()
    for d in range(D):
        q = bytes(rng.integers(25, 40, size=L).astype(np.uint8))
        tags = [(b"MI", "Z", b"%d" % g), (b"RX", "Z", b"ACGTAC-TTGACA"), (b"MC", "Z", b"150M")]
        recs.append(make_record(name=b"r%d_%d" % (g, d), flags=P | F1 | MREV, pos=1000, mate_ref_id=0, mate_pos=1200,
                                tlen=350, seq=tmpl[:L], quals=q, tags=tags))
        recs.append(make_record(name=b"r%d_%d" % (g, d), flags=P | F2 | REV, pos=1200, mate_ref_id=0, mate_pos=1000,
                                tlen=-350, seq=tmpl[200:200 + L], quals=q, tags=tags))
blob = np.frombuffer(b"".join(recs), np.uint8)
off = np.zeros(len(recs) + 1, dtype=np.uint64); off[1:] = np.cumsum([len(r) for r in recs])
grp = np.arange(G + 1, dtype=np.uint64) * np.uint64(2 * D)
threads = [int(t) for t in sys.argv[2].split(",")] if len(sys.argv) > 2 else [1, 4, 8]
for overlap in (False, True):
    for T in threads:
        best = 0.0
        for rep in range(3):
            c = fg.VanillaUmiConsensusCaller("fgumi", "A", fg.VanillaUmiConsensusOptions(min_reads=1, min_consensus_base_quality=2),
                                             device=fg.lib.FGB_DEVICE_NONE, n_threads=T, consensus_call_overlapping_bases=overlap)
            t0 = time.perf_counter()
            assert c._lib.fgb_caller_add_groups(c._h, blob.ctypes.data, off.ctypes.data, grp.ctypes.data, G) == 0
            dt = time.perf_counter() - t0
            best = max(best, len(recs) / dt / 1e6)
            c.close()
        print(f"simplex{'+overlap' if overlap else ''} threads {T}: {best:.2f} M input reads/s")

# duplex and CODEC planning throughput (random MI groups of the parity tests, 150 bp)
from tests.test_caller_parity import random_duplex_groups, random_codec_groups
for name, gen, mk in (("duplex", random_duplex_groups, lambda: fg.DuplexConsensusCaller("fgumi", "A", min_reads=(1, 1, 0), device=fg.lib.FGB_DEVICE_NONE)),
                      ("codec", random_codec_groups, lambda: fg.CodecConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE))):
    groups = gen(np.random.default_rng(5), 1500, L=150)
    recs = [r for g in groups for r in g]
    blob = np.frombuffer(b"".join(recs), np.uint8)
    off = np.zeros(len(recs) + 1, dtype=np.uint64); off[1:] = np.cumsum([len(r) for r in recs])
    grp = np.zeros(len(groups) + 1, dtype=np.uint64); grp[1:] = np.cumsum([len(g) for g in groups])
    best = 0.0
    for rep in range(3):
        c = mk()
        t0 = time.perf_counter()
        assert c._lib.fgb_caller_add_groups(c._h, blob.ctypes.data, off.ctypes.data, grp.ctypes.data, len(groups)) == 0
        best = max(best, len(recs) / (time.perf_counter() - t0) / 1e6)
        c.close()
    print(f"{name} threads 1: {best:.2f} M input reads/s ({len(recs)} reads, {len(recs) / len(groups):.1f} per group)")
