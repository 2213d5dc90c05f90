"""CPU pin of the proof tables the vote kernels trust without looking (host_tables.cpp): qt (unanimous SWAR
threshold), qt3 (near-unanimous threshold of the deep kernel), pair_q (two-read units) and sumt (shallow
sum-of-qualities proof).  tests/native/proof_tables.cpp builds each table over a 15 x 15 grid of
(error_rate_pre_umi, error_rate_post_umi), degenerate values included, and runs the worst pileup every entry admits
through the oracle's ConsensusBaseBuilder add / call.  The minimum counts keep a table that switched itself off
everywhere from passing without checking anything."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# table -> (minimum checks, minimum settings with the table on) over the 225 settings
MINIMA = {
    "qt": (100_000, 180),
    "qt3": (1_000_000, 170),
    "pair_q": (1_500_000, 225),
    "sumt3": (1_000_000, 130),
    "sumt4": (15_000_000, 130),
    "degenerate": (7_800, 30),   # post = 0 (tables not finite, nmax2 = 0) and post = 1 (every D negative)
}


def test_proof_tables_against_oracle(tmp_path):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    exe = tmp_path / "proof_tables"
    csrc = os.path.join(ROOT, "fgumi_b200", "csrc")
    r = subprocess.run([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-I" + csrc, "-o", str(exe),
                        os.path.join(ROOT, "tests", "native", "proof_tables.cpp"), os.path.join(csrc, "host_tables.cpp"),
                        os.path.join(ROOT, "oracle", "fgumi_oracle.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("ok"), r.stdout[-2000:] + r.stderr[-2000:]
    got = {m[0]: (int(m[1]), int(m[2])) for m in re.findall(r"^table (\S+) checks (\d+) active (\d+)$", r.stdout, re.M)}
    assert set(got) == set(MINIMA), got
    for name, (checks, active) in MINIMA.items():
        assert got[name][0] >= checks and got[name][1] >= active, (name, got[name], (checks, active))
