"""Seeded UMI calls for the UMI-assignment tests: families with errors plus the awkward inputs (mixed case, N and
other bytes, dashes in different places, single-key and empty calls)."""
from __future__ import annotations

import random

from fgumi_b200 import synth
from oracle import umi_oracle as U


def noisy_call(rng: random.Random, strategy: int, rules: int, k: int, length: int = None, max_umis: int = 30):
    paired = strategy == U.PAIRED
    L = length or rng.choice([1, 2, 4, 6, 8])
    n_mol = rng.randint(1, 6)
    umis = synth.umi_families(n_mol, L, mean_family=rng.choice([1.5, 3.0, 6.0]),
                              error_rate=rng.choice([0.0, 0.05, 0.2]), paired=paired, seed=rng.randrange(1 << 30))
    umis = umis[:max_umis]
    out = []
    for u in umis:
        r = rng.random()
        if r < 0.1:
            u = u.lower()
        elif r < 0.15:
            i = rng.randrange(len(u))
            u = u[:i] + rng.choice("Nn.X") + u[i + 1:]
        elif r < 0.2 and not paired and len(u) > 1:
            i = rng.randrange(1, len(u))
            u = u[:i] + "-" + u[i:]                    # dash variants: same BitEnc, different string
        elif r < 0.23 and paired:
            a, b = u.split("-")
            j = rng.randrange(0, len(a) + 1)
            u = a[:j] + "-" + a[j:] + b                 # dash moved
        out.append(u.encode())
    if paired and rules == U.MAPPED and rng.random() < 0.5:
        try:
            out = [U.umi_for_read(u, rng.random() < 0.5, strategy, rules, k) for u in out]
        except U.UmiError:
            pass                                       # a UMI without exactly one '-': the call fails as it is
    return out


def calls(seed: int, strategy: int, rules: int, k: int, n: int):
    rng = random.Random(seed)
    res = []
    for _ in range(n):
        c = rng.random()
        if c < 0.05:
            res.append([])
        elif c < 0.1:
            u = noisy_call(rng, strategy, rules, k)[:1]
            res.append(u * rng.randint(1, 4))          # single key
        else:
            res.append(noisy_call(rng, strategy, rules, k))
    return res


def oracle_ok(strategy, rules, k, umis, min_len=None):
    """The oracle's answer, or None when the reference would fail the call."""
    try:
        return U.assign_call(strategy, rules, k, umis, min_len)
    except U.UmiError:
        return None
