"""Small end-to-end exercise of every kernel for compute-sanitizer (memcheck / racecheck / initcheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import fgumi_b200 as fg
from tests import oracle_lib as O

rng = np.random.default_rng(5)
units = []
for i in range(1500):
    depth = int(rng.integers(1, 14))
    L = int(rng.integers(3, 170))
    rows = []
    for _ in range(depth):
        ln = int(rng.integers(max(1, L - 9), L + 1))
        b = rng.choice(np.frombuffer(b"ACGTN", np.uint8), p=[.24, .24, .24, .24, .04], size=ln)
        q = rng.integers(2, 45, size=ln).astype(np.uint8)
        q[b == ord("N")] = 2
        rows.append((b.tobytes(), q.tobytes()))
    units.append(rows)
def deep_unit(depth, L):
    t = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=L)
    rows = []
    for _ in range(depth):
        b = t.copy()
        m = rng.random(L) < 0.01
        b[m] = rng.choice(np.frombuffer(b"ACGTN", np.uint8), size=int(m.sum()))
        q = rng.integers(20, 42, size=L).astype(np.uint8)
        q[b == ord("N")] = 2
        rows.append((b.tobytes(), q.tobytes()))
    return rows
for i in range(40):                                               # deep class: lane-group form (several units per tile) ...
    units.append(deep_unit(int(rng.integers(24, 60)), int(rng.integers(30, 60))))
for i in range(12):                                               # ... and the flat form (one unit of >= 64 reads per tile)
    units.append(deep_unit(int(rng.integers(70, 120)), 150))
units.append([(b"ACGT" * 6000, bytes([30] * 24000))] * 3)        # oversize unit: direct path
batch = fg.pack_source_reads(units, 1)
eng = fg.Engine(0, 45, 40, 1, 2)
want = O.simplex_batch(batch, 45, 40, 1, 2)
got = eng.vote(batch)
n = batch.n_out
assert np.array_equal(got.base[:n], want[0][:n]) and np.array_equal(got.qual[:n], want[1][:n])
packed = fg.pack8_encode(batch.bases, batch.quals)
out8 = fg.HostColumns(np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8))
eng.submit_ex(batch, out8, packed=packed, narrow=True); eng.wait()
assert np.array_equal(out8.base, got.base[:n])
# filter epilogue through the caller, duplex and codec callers
from tests.test_caller_parity import random_groups, random_duplex_groups, random_codec_groups
c = fg.VanillaUmiConsensusCaller("f", "A", fg.VanillaUmiConsensusOptions(min_reads=1, min_consensus_base_quality=2),
                                 filter=fg.ConsensusFilter(min_reads=2, max_read_error_rate=0.1, max_base_error_rate=0.2, min_base_quality=10),
                                 consensus_call_overlapping_bases=True, n_threads=3)
c.add_groups(random_groups(rng, 60)); c.flush(); c.close()
c = fg.VanillaUmiConsensusCaller("f", "A", fg.VanillaUmiConsensusOptions(min_reads=1, min_consensus_base_quality=2),
                                 consensus_call_overlapping_bases=True, n_threads=3)          # no filter: records assembled on the device (K5)
c.add_groups(random_groups(rng, 60)); c.flush(); c.close()
c = fg.DuplexConsensusCaller("f", "A", min_reads=(1, 1, 0)); c.consensus_reads_batch(random_duplex_groups(rng, 60)); c.close()
c = fg.CodecConsensusCaller("c", "R"); c.consensus_reads_batch(random_codec_groups(rng, 60)); c.close()
# duplex combine in the vote kernels' epilogue (all three class kernels, attached and stray jobs, pending clean-up)
from tests.test_combine_parity import _duplex_molecules, _duplex_against_oracle
du, dp = _duplex_molecules(rng, 120, depth_hi=41, len_lo=100, len_hi=151, iupac=True)
dp += [(4 * m, 4 * (m + 30) + 1) for m in range(0, 80, 9)]
_duplex_against_oracle(fg, du, dp, True)
du, dp = _duplex_molecules(rng, 200)
_duplex_against_oracle(fg, du, dp, True)
# the fallback kernels of K4, K2 and K3 (column pointers that are not aligned for the word kernels)
from tests.test_fallback_kernels import FILTER_GRID, codec_forms, duplex_forms, filter_forms
filter_forms(fg, FILTER_GRID[0], 11, set())
du, dp = _duplex_molecules(rng, 40, iupac=True)
dp.append((5, 5))
duplex_forms(fg, du, dp)
codec_forms(fg, 78)
# K0z: BGZF members inflated on the device (good and damaged members)
from tests.test_bgzf import test_bgzf_members_inflated_on_the_device
test_bgzf_members_inflated_on_the_device()
# BAM4
layout, raw = fg.pack_raw_reads([[(b"ACGTNACGTACGTTTGA", bytes(range(5, 22)), bool(i & 1), 17 - (i % 3))] * (1 + i % 4) for i in range(200)], 1, 10)
o = fg.HostColumns.alloc(layout.n_out)
eng.submit_bam4(layout, raw, o); eng.wait()
# record filter: pass 1, decision, scans and pass 2 against the oracle (both modes, tag reversal, rejects)
import tempfile
from fgumi_b200 import filter as F
from tests import filter_oracle as FO, filter_streams as FS
contigs = FS.genome(3)
with tempfile.TemporaryDirectory() as d:
    with open(os.path.join(d, "g.fa"), "wb") as f:
        f.write(FS.fasta(contigs))
    ref = F.Reference(os.path.join(d, "g.fa"))
recs = FS.records(4, contigs, n_templates=120)
fb, foff = FS.pack(recs)
for tmpl in (True, False):
    rf = F.RecordFilter(filter_by_template=tmpl, reverse_per_base_tags=True, track_rejects=True,
                        max_no_call_fraction=0.5, max_base_error_rate=(0.3,))
    assert rf.filter(FS.header(contigs), fb, foff, ref) == FO.filter_records(
        recs, FS.header(contigs), FO.Config(filter_by_template=tmpl, reverse_per_base_tags=True,
                                            max_no_call_fraction=0.5, max_base_error_rate=(0.3,)),
        FO.parse_fasta(FS.fasta(contigs)))
    rf.close()
ref.close()
eng.close()
print("sanitize run ok")
