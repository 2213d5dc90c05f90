"""Measurement legs shared by bench.py and scripts/bench_modes.py: BASELINE configs 3, 4, 5 device resident
(per-kernel time and fraction of the HBM roofline, algorithmic bytes per SURVEY section 8d) and the
record-level boundary (raw BAM records -> ConsensusOutput bytes).  Synthetic inputs from synth.py."""
from __future__ import annotations

import ctypes as C
import json
import os
import threading
import time

import numpy as np

from . import lib as _l
from . import synth

L = 150
Lo = (L + 7) // 8 * 8


def hbm_peak() -> float:
    try:
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"])
    except Exception:
        return 3350.0       # H100 SXM data sheet


def timed(torch, fn, n=6):
    fn(); torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    ev[0].record()
    for i in range(n):
        fn(); ev[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(n)]))


def vote_bytes(depths: np.ndarray, read_len: int = L) -> int:
    """SURVEY 8(d): per unit 2 * sum(len) in + 6 * cons_len out + 8 * (n_reads + 1) + 8 index bytes."""
    nr, nu = int(depths.sum()), int(len(depths))
    return 2 * nr * read_len + 6 * nu * read_len + 8 * (nr + nu) + 8 * nu


def duplex_leg(torch, fg, dev, device_index: int, molecules: int, seed: int = 43):
    """Config 3: duplex, 4 + 4 reads per strand -> four single-strand units of depth 4 and two combine jobs
    per molecule (K1 then K2)."""
    M = int(molecules); U = 4 * M
    depths = np.full(U, 4, dtype=np.int64)
    m = np.arange(M, dtype=np.int64)
    tid = np.empty(U, dtype=np.int64)
    tid[0::4], tid[3::4], tid[1::4], tid[2::4] = 2 * m, 2 * m, 2 * m + 1, 2 * m + 1
    tb = synth.device_batch(torch, dev, depths, L, 1e-3, seed=seed, template_ids=tid)
    eng = fg.Engine(device_index, 45, 40, 1, 2)
    ss = fg.DeviceColumns(tb.host.n_out, dev)
    jobs = np.zeros(2 * M, dtype=fg.DUPLEX_JOB_DTYPE)
    jobs["unit_a"][0::2], jobs["unit_b"][0::2] = 4 * m, 4 * m + 3
    jobs["unit_a"][1::2], jobs["unit_b"][1::2] = 4 * m + 1, 4 * m + 2
    jobs["out_off"] = np.arange(2 * M, dtype=np.uint64) * np.uint64(Lo)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(dev)
    n_out = 2 * M * Lo
    ob = torch.zeros(n_out, dtype=torch.uint8, device=dev); oq = torch.zeros_like(ob)
    oe = torch.zeros(n_out, dtype=torch.int16, device=dev)
    st = torch.zeros(2 * M, dtype=torch.uint8, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    t1 = timed(torch, lambda: eng.vote_device(tb, ss, s))
    t2 = timed(torch, lambda: eng.duplex_combine_device(tb, ss, tj, 2 * M, ob, oq, oe, st, s))
    # the same work with the combine in the vote kernels' epilogue (fgb_plan_tiles_jobs + fgb_vote_duplex_device):
    # tiles cut at molecule boundaries, K2 reads the SS words back through L2 and the source rows from the stage
    from .engine import plan_tiles_jobs
    tiles, class_tiles, tile_jobs, job_index, n_attached = plan_tiles_jobs(tb.host, jobs)
    t8 = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)
    tbf = synth.TorchBatch(tb.bases, tb.quals, tb.reads, tb.units, t8(tiles), tb.host, class_tiles)
    tbf.n_tiles = len(tiles)
    d_tj, d_ji = t8(tile_jobs), t8(job_index)
    ref = (ob.clone(), oq.clone(), oe.clone(), ss.base.clone(), ss.errors.clone())
    ob.zero_(); oq.zero_(); oe.zero_(); st.fill_(77)
    tf = timed(torch, lambda: eng.vote_duplex_device(tbf, ss, tj, 2 * M, d_tj, d_ji, ob, oq, oe, st, s))
    valid = lambda x: x[: x.numel() // Lo * Lo].reshape(-1, Lo)[:, :L]        # the called positions of every row
    same = all(bool(torch.equal(valid(x), valid(y))) for x, y in zip(ref, (ob, oq, oe, ss.base, ss.errors))) and int(st.max()) == 0
    del ref
    k1_bytes = vote_bytes(depths)
    # SURVEY 8(d): K2 traffic per job = the two single-strand rows in (2 x 6 L) + (base, qual, errors) out (4 L): 2 400 B,
    # 13 392 B per molecule with the four votes.  The exact error recount also re-reads the 8 pooled source rows
    # (8 L more per job, not in SURVEY's figure): `*_touched` counts them (and only the three SS columns K2 reads).
    k2_bytes = 2 * M * (2 * 6 * L + 4 * L)
    k2_touched = 2 * M * (2 * 4 * L + 4 * L + 8 * L + 16)
    peak = hbm_peak()
    eng.close()
    del tb, ss
    two = {"value": M / ((t1 + t2) * 1e-3), "k1_ms": t1, "k2_ms": t2,
           "k1_frac": k1_bytes / t1 / 1e6 / peak, "k2_frac": k2_bytes / t2 / 1e6 / peak,
           "frac": (k1_bytes + k2_bytes) / (t1 + t2) / 1e6 / peak,
           "k2_frac_touched": k2_touched / t2 / 1e6 / peak,
           "frac_touched": (k1_bytes + k2_touched) / (t1 + t2) / 1e6 / peak,
           "bytes_per_molecule_touched": (k1_bytes + k2_touched) / M,
           "api": "fgb_vote_device + fgb_duplex_combine_device"}
    epi = {"value": M / (tf * 1e-3), "ms": tf, "frac": (k1_bytes + k2_bytes) / tf / 1e6 / peak,
           "jobs_in_epilogue": int(n_attached), "jobs": 2 * M, "equals_two_kernel_form": same,
           "api": "fgb_plan_tiles_jobs + fgb_vote_duplex_device (K2 in the vote kernels' epilogue)"}
    best = two if two["value"] >= epi["value"] else epi
    return {"workload": "BASELINE.json configs[2]: duplex, 4+4 reads per strand, 150bp", "molecules": M,
            "value": best["value"], "unit": "molecules/s", "frac": best["frac"], "form": best["api"],
            "k1_ms": t1, "k2_ms": t2, "k1_frac": two["k1_frac"], "k2_frac": two["k2_frac"],
            "bytes_per_molecule": (k1_bytes + k2_bytes) / M,
            "two_kernels": two, "epilogue": epi,
            "bytes": "frac uses SURVEY 8(d)'s 13 392 B per molecule (four votes + two combines, SS columns written and read "
                     "once each); two_kernels.*_touched add the 8 pooled source rows the standalone K2 re-reads per job; "
                     "value / frac are the faster of the two forms"}


def codec_leg(torch, fg, dev, device_index: int, molecules: int, seed: int = 44, sort_by_depth: bool = True):
    """Config 4: CODEC, k ~ U[2, 20] read pairs per molecule -> two single-strand units and one combine job.
    sort_by_depth: the packer lays the molecules out in order of k (every tile then holds units of one depth and
    takes the descriptor-free scan); a molecule's OUTPUT row stays where its input position puts it."""
    M = int(molecules)
    rng = np.random.default_rng(seed)
    k = rng.integers(2, 21, size=M)
    insert = np.clip(np.round(rng.normal(300, 50, size=M)), L, 2 * L).astype(np.int64)
    r1n = rng.random(M) < 0.5
    lc_pad = (insert + 7) // 8 * 8
    out_off = np.zeros(M, dtype=np.uint64)
    out_off[1:] = np.cumsum(lc_pad)[:-1]                    # output rows in INPUT order
    perm = np.argsort(k, kind="stable") if sort_by_depth else np.arange(M)
    k, insert, r1n, out_off = k[perm], insert[perm], r1n[perm], out_off[perm]
    depths = np.repeat(k, 2).astype(np.int64)
    tb = synth.device_batch(torch, dev, depths, L, 1e-3, seed=seed)
    eng = fg.Engine(device_index, 45, 40, 1, 0)
    ss = fg.DeviceColumns(tb.host.n_out, dev)
    jobs = np.zeros(M, dtype=fg.CODEC_JOB_DTYPE)
    jobs["unit_a"], jobs["unit_b"] = 2 * np.arange(M), 2 * np.arange(M) + 1
    jobs["out_off"] = out_off
    jobs["len"] = insert
    jobs["rc_a"], jobs["rc_b"], jobs["rc_out"] = r1n, ~r1n, r1n
    jobs["pad_a_left"] = np.where(r1n, insert - L, 0)
    jobs["pad_b_left"] = np.where(~r1n, insert - L, 0)
    tj = torch.from_numpy(jobs.view(np.uint8).reshape(-1)).to(dev)
    out = fg.DeviceColumns(int(lc_pad.sum()), dev)
    st = torch.zeros(M, dtype=torch.uint8, device=dev)
    dis = torch.zeros(M, dtype=torch.int32, device=dev); dup = torch.zeros_like(dis)
    cp = fg.lib.FgbCodecParams(-1, -1, 5, 0xFFFFFFFF, 1.0)
    s = torch.cuda.current_stream().cuda_stream
    t1 = timed(torch, lambda: eng.vote_device(tb, ss, s))
    t3 = timed(torch, lambda: eng.codec_combine_device(tb, ss, tj, M, cp, out, st, dis, dup, s))
    k1_bytes = vote_bytes(depths)
    k3_bytes = M * 2 * 6 * L + int(insert.sum()) * 6 + 32 * M
    peak = hbm_peak()
    eng.close()
    classes = list(tb.class_tiles)
    del tb, ss, out
    return {"workload": "BASELINE.json configs[3]: CODEC, 2-20 pairs per molecule, 2x150bp", "molecules": M,
            "value": M / ((t1 + t3) * 1e-3), "unit": "molecules/s", "k1_ms": t1, "k3_ms": t3,
            "k1_frac": k1_bytes / t1 / 1e6 / peak, "k3_frac": k3_bytes / t3 / 1e6 / peak,
            "frac": (k1_bytes + k3_bytes) / (t1 + t3) / 1e6 / peak, "bytes_per_molecule": (k1_bytes + k3_bytes) / M,
            "class_tiles": classes,
            "layout": "molecules packed in order of depth, output rows in input order" if sort_by_depth else "input order"}


def depth_classes(depths: np.ndarray) -> np.ndarray:
    """fgb_config.h unit_class: 1 shallow (<= 4 reads), 2 deep (>= 24), 0 general."""
    return np.where(depths <= 4, 1, np.where(depths >= 24, 2, 0))


def zipf_leg(torch, fg, dev, device_index: int, total_families: int, world: int, rank: int, seed: int = 42,
             shard_of: int = 16):
    """Config 5: `total_families` simplex families with Zipf(1) depths on 1..100, range-sharded by cumulative
    READ count (shard.partition_by_reads) over max(world, shard_of) ranks; this rank votes its own range (one
    sixteenth of 100 M families is ~36 GB of source rows, what an 80 GB H100 holds with its outputs).  The
    packer lays a rank's families out in order of depth (every tile then holds units of one depth, and the
    general / shallow / deep tile classes come in three runs); the output rows follow the packed order and a
    host-side permutation (what the record-level caller keeps per unit anyway) maps them back to input order."""
    from .shard import partition_by_reads
    parts_n = max(world, shard_of)
    depths_all = synth.zipf_depths(int(total_families), 1, 100, 1.0, seed=seed).astype(np.int64)
    parts = partition_by_reads(depths_all, parts_n)
    loads = np.array([int(depths_all[a:b].sum()) for a, b in parts], dtype=np.float64)
    lo, hi = parts[rank if world > 1 else 0]
    depths = depths_all[lo:hi]
    order = np.argsort(depths, kind="stable")                      # pack by depth
    tb = synth.device_batch(torch, dev, depths[order], L, 1e-3, seed=seed + rank)
    eng = fg.Engine(device_index, 45, 40, 1, 2)
    out = fg.DeviceColumns(tb.host.n_out, dev)
    s = torch.cuda.current_stream().cuda_stream
    t1 = timed(torch, lambda: eng.vote_device(tb, out, s), n=4)
    k1_bytes = vote_bytes(depths)
    peak = hbm_peak()
    eng.close()
    res = {"workload": f"BASELINE.json configs[4]: simplex, {int(total_families)} families, Zipf(1) depth 1-100, "
                       f"read-balanced range split over {parts_n} ranks (this line: rank {rank if world > 1 else 0})",
           "families_this_rank": int(hi - lo), "reads_this_rank": int(depths.sum()), "k1_ms": t1,
           "value": (hi - lo) / (t1 * 1e-3), "unit": UNIT_READS, "frac": k1_bytes / t1 / 1e6 / peak,
           "rank_load_imbalance": float(loads.max() / loads.mean() - 1.0), "class_tiles": list(tb.class_tiles),
           "layout": "families packed in order of depth within the rank (outputs in packed order)"}
    del tb, out
    return res


UNIT_READS = "consensus_reads/s"


# ---- record level ----------------------------------------------------------------------------------------
class _Caller:
    """fgb_caller_* through ctypes without copying the output (the timed call is the C-ABI itself)."""

    def __init__(self, lib, device: int, n_threads: int, overlap: bool = False, zero_copy: bool = True,
                 min_reads: int = 1):
        o = _l.FgbCallerOptions()
        o.mode = 0; o.error_rate_pre_umi = 45; o.error_rate_post_umi = 40; o.min_input_base_quality = 10
        o.min_consensus_base_quality = 2; o.produce_per_base_tags = 1; o.trim = 0
        o.consensus_call_overlapping_bases = int(overlap)
        o.min_reads = min_reads; o.tag = b"MI"; o.read_name_prefix = b"fgumi"; o.read_group_id = b"A"
        o.n_threads = n_threads
        o.zero_copy_records = int(zero_copy)     # the legs pass page-locked records that stay put until the flush returns
        self._keep = o
        self.lib = lib
        self.h = C.c_void_p()
        st = lib.fgb_caller_create(device, C.byref(o), C.byref(self.h))
        if st != 0:
            raise _l.FgbError(st, "fgb_caller_create")

    def process(self, blob_ptr, off_ptr, grp_ptr, n_groups):
        lib = self.lib
        st = lib.fgb_caller_add_groups(self.h, blob_ptr, off_ptr, grp_ptr, n_groups)
        if st != 0:
            raise _l.FgbError(st, "fgb_caller_add_groups")
        data, n, cnt = C.c_void_p(), C.c_uint64(), C.c_uint64()
        st = lib.fgb_caller_flush(self.h, C.byref(data), C.byref(n), C.byref(cnt))
        if st != 0:
            buf = C.create_string_buffer(256)
            lib.fgb_caller_last_error(self.h, buf, 256)
            raise _l.FgbError(st, "fgb_caller_flush", buf.value.decode(errors="replace"))
        return data.value, int(n.value), int(cnt.value)

    def stats(self):
        arr = (C.c_uint64 * _l.FGB_NSTATS)()
        self.lib.fgb_caller_stats(self.h, arr)
        return [int(x) for x in arr]

    def close(self):
        if self.h:
            self.lib.fgb_caller_destroy(self.h)
            self.h = C.c_void_p()


def make_record_batch(torch, families: int, depth: int = 8, seed: int = 42, base_families: int = 25000):
    """`families` MI groups of `depth` raw BAM records in PAGE-LOCKED host memory.  The numpy generator makes
    base_families of them; the rest are copies with their own MI values and names (the reads' content does not
    change the host cost, the group structure does)."""
    base_n = min(int(families), int(base_families))
    blob, off, grp = synth.record_families(base_n, depth, L, 1e-3, seed=seed)
    rec_len = int(off[1])
    reps = (int(families) + base_n - 1) // base_n
    G = int(families)
    R = G * depth
    pinned = torch.empty(R * rec_len + 64, dtype=torch.uint8).pin_memory()
    m = pinned.numpy()[:R * rec_len].reshape(R, rec_len)
    src = blob.reshape(base_n * depth, rec_len)
    for k in range(reps):
        a = k * base_n * depth
        b = min(R, a + base_n * depth)
        m[a:b] = src[:b - a]
    fam = np.repeat(np.arange(G, dtype=np.int64), depth)
    for col, n in ((32 + 1, 7), (rec_len - 24 + 3, 8)):            # the name's and the MI tag's digits
        v = fam % (10 ** n)
        for j in range(n - 1, -1, -1):
            m[:, col + j] = 48 + (v % 10)
            v //= 10
    rec_off = np.arange(R + 1, dtype=np.uint64) * np.uint64(rec_len)
    group_rec = np.arange(G + 1, dtype=np.uint64) * np.uint64(depth)
    return pinned, rec_off, group_rec, rec_len


def records_leg(torch, fg, lib, device_index: int, families: int, n_threads: int, steps: int = 5, warmup: int = 2,
                callers: int = 2, depth: int = 8):
    """Raw BAM records (page-locked host memory) -> fgb_caller_add_groups + fgb_caller_flush -> ConsensusOutput
    bytes in host memory, wall clock over `steps` batches of `families` MI groups.  With callers = 2, two callers
    (each with its own engine handle and half of the host threads) work on alternating batches from two threads,
    so one's host phases overlap the other's transfers -- the reference's one-caller-per-worker pattern."""
    pinned, rec_off, group_rec, rec_len = make_record_batch(torch, families, depth)
    bp, op, gp = pinned.data_ptr(), rec_off.ctypes.data, group_rec.ctypes.data
    G = len(group_rec) - 1
    res = {}

    def run(ncall, threads_each):
        cs = [_Caller(lib, device_index, threads_each) for _ in range(ncall)]
        out = {"count": 0, "bytes": 0, "stats": None}

        def worker(c, n):
            for _ in range(n):
                _, nb, cnt = c.process(bp, op, gp, G)
                out["count"] = cnt; out["bytes"] = nb
        try:
            for c in cs:
                worker(c, warmup)
            t0 = time.perf_counter()
            if ncall == 1:
                worker(cs[0], steps)
            else:
                th = [threading.Thread(target=worker, args=(c, steps)) for c in cs]
                for t in th:
                    t.start()
                for t in th:
                    t.join()
            dt = time.perf_counter() - t0
            st = np.zeros(_l.FGB_NSTATS, dtype=np.int64)
            for c in cs:
                st += np.array(c.stats(), dtype=np.int64)
            out["stats"] = st
        finally:
            for c in cs:
                c.close()
        return G * steps * ncall / dt, out

    v1, o1 = run(1, n_threads)
    res["one_caller"] = {"value": v1, "host_threads": n_threads}
    best = v1
    if callers > 1:
        # a caller's threads idle while its batch is on the link / the device: several callers (the reference's
        # one-caller-per-worker pattern) fill that time.  Threads are either split between the callers or every
        # caller gets the full count (oversubscribed: the waiting caller's threads sleep).
        v2, _ = run(callers, max(1, n_threads // callers))
        res["two_callers"] = {"value": v2, "host_threads": max(1, n_threads // callers) * callers}
        best = max(best, v2)
        multi = {}
        for ncall, each in ((2, n_threads), (3, n_threads), (4, max(1, n_threads // 2))):
            try:
                v, _ = run(ncall, each)
                multi[f"{ncall}x{each}"] = v
                best = max(best, v)
            except Exception as ex:      # pragma: no cover
                multi[f"{ncall}x{each}"] = repr(ex)[:80]
        res["callers_x_threads"] = multi
    R = G * depth
    res.update({"value": best, "unit": UNIT_READS, "families_per_batch": G, "reads_per_family": depth,
                "h2d_bytes_per_batch": int(R * rec_len + R * 24 + G * 16), "d2h_bytes_per_batch": int(G * Lo * 4),
                "input_bytes_per_batch": int(R * rec_len), "output_bytes_per_batch": int(o1["bytes"]),
                "consensus_reads_per_batch": int(o1["count"]),
                "caller_stats": [int(x) for x in o1["stats"]],
                "api": "fgb_caller_add_groups + fgb_caller_flush (raw BAM records in page-locked host memory -> "
                       "ConsensusOutput bytes in host memory; records staged, shipped whole, rows built on the device)"})
    del pinned
    return res


def records_cpu_baseline(families: int, n_threads: int, depth: int = 8, seed: int = 42, min_seconds: float = 6.0):
    """The record-level CPU baseline: the PRODUCT's host code (group rules, source-read decisions, record
    assembly) over the CPU oracle's vote -- oracle/libfgb_cpu_caller.so (test infrastructure, labelled 'port')."""
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    so = os.path.join(root, "oracle", "libfgb_cpu_caller.so")
    os.environ["FGB_CPU_THREADS"] = str(n_threads)
    cpu = C.CDLL(so)
    vp, u64 = C.c_void_p, C.c_uint64
    cpu.fgb_caller_create.argtypes = [C.c_int, C.POINTER(_l.FgbCallerOptions), C.POINTER(vp)]
    cpu.fgb_caller_add_groups.argtypes = [vp, vp, vp, vp, u64]
    cpu.fgb_caller_flush.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    cpu.fgb_caller_destroy.argtypes = [vp]
    cpu.fgb_caller_last_error.argtypes = [vp, C.c_char_p, C.c_size_t]
    blob, off, grp = synth.record_families(int(families), depth, L, 1e-3, seed=seed)
    c = _Caller(cpu, 0, n_threads)
    try:
        c.process(blob.ctypes.data, off.ctypes.data, grp.ctypes.data, len(grp) - 1)
        reps, t0 = 0, time.perf_counter()
        while True:
            _, _, cnt = c.process(blob.ctypes.data, off.ctypes.data, grp.ctypes.data, len(grp) - 1)
            reps += 1
            dt = time.perf_counter() - t0
            if dt >= min_seconds or reps >= 200:
                break
    finally:
        c.close()
    return {"value": int(families) * reps / dt, "unit": UNIT_READS, "cores": n_threads, "kind": "port",
            "sample": f"{reps} batches of {int(families)} families x {depth} records, {dt:.1f} s; the product's host "
                      "code (caller_host.cpp) over the CPU oracle's vote (tests/native/mock_engine.cpp), "
                      "-O3 -march=x86-64-v3"}
