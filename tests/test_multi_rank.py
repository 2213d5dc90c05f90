"""N>1 host logic on CPU: 2 gloo ranks range-partition a batch, each rank calls consensus on its
own shard (the oracle stands in for the GPU here — this test is about the partition, the output
order and the counter reduction), and the summed counters / concatenated outputs equal the
single-process result."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _units(seed=3, n=120):
    sys.path.insert(0, ROOT)
    from fgumi_b200 import synth
    rng = np.random.default_rng(seed)
    depths = synth.zipf_depths(n, 1, 30, 1.0, seed=seed)
    units = []
    for d in depths:
        b, q = synth.host_pileup(1, int(d), 60, 0.02, seed=int(rng.integers(1 << 30)))
        units.append([(b[0, r].tobytes(), q[0, r].tobytes()) for r in range(int(d))])
    return depths, units


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    import fgumi_b200 as fg
    from fgumi_b200 import shard
    from tests import oracle_lib as O
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    depths, units = _units()
    lo, hi = shard.partition_by_reads(depths, world)[rank]
    batch = fg.pack_source_reads(units[lo:hi], 1)
    ob, oq, od, oe, cl = O.simplex_batch(batch, 45, 40, 1, 2)
    rows = [(bytes(ob[s]), bytes(oq[s])) for s in batch.unit_slices()]
    counters = torch.tensor([hi - lo, int(cl.sum()), int((ob[:batch.n_out] == ord("N")).sum()),
                             batch.n_reads], dtype=torch.int64)
    shard.all_reduce_counters(counters, dist)
    np.save(os.path.join(out_dir, f"counters_{rank}.npy"), counters.numpy())
    import pickle
    with open(os.path.join(out_dir, f"rows_{rank}.pkl"), "wb") as f:
        pickle.dump((lo, hi, rows), f)
    dist.barrier()
    dist.destroy_process_group()


def test_partition_by_reads_balances_and_covers():
    sys.path.insert(0, ROOT)
    from fgumi_b200 import shard, synth
    depths = synth.zipf_depths(10000, 1, 100, 1.0, seed=1)
    for world in (1, 2, 3, 8):
        parts = shard.partition_by_reads(depths, world)
        assert parts[0][0] == 0 and parts[-1][1] == len(depths)
        assert all(parts[i][1] == parts[i + 1][0] for i in range(world - 1))
        loads = [int(depths[a:b].sum()) for a, b in parts]
        assert max(loads) - min(loads) <= 2 * 100          # within one max-depth family
    assert shard.partition_by_reads(np.array([], dtype=np.int64), 4) == [(0, 0)] * 4


def test_two_rank_gloo_shards_match_single_process(tmp_path):
    import pickle
    import torch.multiprocessing as mp
    world = 2
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    sys.path.insert(0, ROOT)
    import fgumi_b200 as fg
    from tests import oracle_lib as O
    depths, units = _units()
    full = fg.pack_source_reads(units, 1)
    ob, oq, od, oe, cl = O.simplex_batch(full, 45, 40, 1, 2)
    want_rows = [(bytes(ob[s]), bytes(oq[s])) for s in full.unit_slices()]
    got_rows = []
    for r in range(world):
        lo, hi, rows = pickle.load(open(tmp_path / f"rows_{r}.pkl", "rb"))
        assert lo == len(got_rows)                   # rank order == input order
        got_rows += rows
    assert got_rows == want_rows
    c0 = np.load(tmp_path / "counters_0.npy"); c1 = np.load(tmp_path / "counters_1.npy")
    assert np.array_equal(c0, c1)                    # every rank holds the global sums
    assert c0[0] == full.n_units and c0[1] == int(cl.sum()) and c0[3] == full.n_reads
    assert c0[2] == int((ob[:full.n_out] == ord("N")).sum())


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` runs on host cores only: one JSON line with the contract's keys
    (impl, metric, value, unit, cpu_baseline, e2e with zero transfer bytes ...) and a positive rate."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, FGB_REF_SAMPLE_UNITS="20000")
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "3"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stdout.strip().splitlines()
    assert len(lines) == 1 and lines[0].startswith("{")          # stdout carries the JSON line and nothing else
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["value"] > 0 and d["warmup"] >= 3 and d["higher_is_better"] is True
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and "workload" in d["config"]
    meta = json.load(open(os.path.join(root, "BASELINE.json")))
    assert d["metric"].split(" (")[0] in meta["metric"]


def test_clock_sampler_uses_the_samples_inside_the_timed_region():
    """bench.py's clocks line: the sampler runs from before the warm-up, stamps every sample and
    summarises those inside begin()..end(); a missing tool or garbage output never raises."""
    import importlib.util
    import time
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(root, "bench.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    fake = [sys.executable, "-u", "-c",
            "import time\nfor i in range(300):\n print('%d, 1965, Not Active, Not Active, Not Active, %s' % "
            "(1000 + i, 'Active' if 40 <= i < 45 else 'Not Active'), flush=True); time.sleep(0.01)"]
    c = b.ClockSampler(0, fake)
    c.start()
    c.wait_ready()
    assert c.samples
    time.sleep(0.35)
    c.begin(); time.sleep(0.25); c.end()
    r = c.stop()
    assert r["window"] == "timed region" and 10 <= r["samples"] <= 40 and r["sm_max_mhz"] == 1965.0
    assert 1020 < r["sm_mhz"] < 1075 and r["reasons"] in ([], ["sw_power_cap"])
    dead = b.ClockSampler(0, ["/nonexistent/tool"])
    dead.start(); dead.wait_ready(0.2)
    assert dead.stop()["sm_mhz"] is None
    quiet = b.ClockSampler(0, [sys.executable, "-c", "import time; time.sleep(5)"])
    quiet.start()
    t0 = time.perf_counter(); quiet.wait_ready(0.3)
    assert time.perf_counter() - t0 < 1.0
    quiet.begin(); quiet.end()
    assert quiet.stop()["sm_mhz"] is None
    c = b.ClockSampler(0, [sys.executable, "-c", "print('garbage')"])
    c.start(); c.begin(); c.end()
    assert c.stop()["sm_mhz"] is None


def test_bench_dump_outputs_writes_a_fixed_float_sample(tmp_path):
    """`bench.py --dump-outputs DIR`: the four consensus columns of a fixed, seeded sample of families, every called
    position of each, as float32 .npy (plus the sampled family indices), well under 64 MB."""
    import importlib.util
    from types import SimpleNamespace
    import torch
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(root, "bench.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    U, Lo = 20000, 152
    units = np.zeros(U + 1, dtype=[("out_off", "<u8"), ("read_begin", "<u4"), ("cons_len", "<u4")])
    units["out_off"] = np.arange(U + 1, dtype=np.uint64) * np.uint64(Lo)
    host = SimpleNamespace(n_units=U, units=units)
    g = torch.Generator().manual_seed(1)
    out = SimpleNamespace(base=torch.randint(0, 256, (U * Lo,), dtype=torch.uint8, generator=g),
                          qual=torch.randint(0, 94, (U * Lo,), dtype=torch.uint8, generator=g),
                          depth=torch.randint(0, 40000, (U * Lo,), generator=g).to(torch.int16),
                          errors=torch.randint(0, 9, (U * Lo,), generator=g).to(torch.int16))
    b.dump_outputs(str(tmp_path / "a"), torch, out, host)
    b.dump_outputs(str(tmp_path / "b"), torch, out, host)
    names = ("base", "qual", "depth", "errors", "family_index")
    total = 0
    fam = np.load(tmp_path / "a" / "family_index.npy").astype(np.int64)
    assert len(fam) == b.DUMP_FAMILIES and np.all(np.diff(fam) > 0)
    for name in names:
        x, y = np.load(tmp_path / "a" / f"{name}.npy"), np.load(tmp_path / "b" / f"{name}.npy")
        assert x.dtype in (np.float32, np.float64) and np.array_equal(x, y)
        total += x.nbytes
        if name != "family_index":
            col = getattr(out, name).numpy()
            col = col.view(np.uint16) if col.dtype == np.int16 else col
            want = col.reshape(U, Lo)[fam, :b.READ_LEN]
            assert x.shape == want.shape and np.array_equal(x, want.astype(np.float32))
    assert total <= 64 << 20
