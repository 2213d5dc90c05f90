"""Where the general vote kernel's time goes, from inside the kernel (Nsight-free), and what the memory system gives
its byte mix.

  python scripts/pipe_trace.py --build-only         # cross-compile the diagnostic libraries into variants/
  python scripts/pipe_trace.py [--compare A.so ...]  # on a GPU

Diagnostic libraries (fgumi_b200/build.py build_variant, never the in-tree one):
  variants/pipe_trace.so   FGB_PIPE_TRACE=1: clock64 sums per CTA -- producer cycles waiting on `empty`, consumer-warp
                           cycles waiting on `full`, issue -> `full` cycles of the tiles that had not landed when the
                           consumers arrived, voting cycles (fast pass / slow pass), how long a stage is held (warp 0
                           passing `full` -> the last warp's release) and the spread of the eight warps' releases.
                           Loaded through FGUMI_B200_LIB.
  variants/pipe_novote.so  FGB_PIPE_NOVOTE=1: consumers store constant words for their items instead of voting; the
                           producer, the stage ring, the prefetch and the stores are unchanged.

Legs: BASELINE config 2 (10 M families, depth 8, 150 bp), the same at depth 3, and the first of the sixteen
read-balanced shards of the Zipf(1) depth-1..100 workload (config 5), families packed by depth.  Per leg it prints the
traced build's ms per launch beside the in-tree library's (the trace's own perturbation), the split as fractions of
the kernel's time, and -- for config 2 -- two ceilings on the bench's own device columns: a read-only torch pass, a
two-read one-write torch pass (bases XOR quals as int64 into a third buffer: 67 % reads, the kernel moves 71 %), and
the no-vote library.  `--compare` libraries (e.g. an A/B build, or another commit's library) are timed on the same
batch, alternating with the in-tree one round by round, and their outputs are compared with its outputs; the split of
a traced --compare library (another commit's pipe_trace.so) is printed beside the in-tree sources' one.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAR = os.path.join(ROOT, "variants")
TRACE_LIB = os.path.join(VAR, "pipe_trace.so")
NOVOTE_LIB = os.path.join(VAR, "pipe_novote.so")
INTREE_LIB = os.path.join(ROOT, "fgumi_b200", "libfgumi_b200.so")
TRACE_WORDS = 16


def build_libs(force: bool):
    sys.path.insert(0, ROOT)
    from fgumi_b200 import build as B
    for path, defs in ((TRACE_LIB, {"FGB_PIPE_TRACE": 1}), (NOVOTE_LIB, {"FGB_PIPE_NOVOTE": 1})):
        if force or not os.path.exists(path):
            B.build_variant(path, defs)
            print("built", os.path.relpath(path, ROOT), flush=True)


class Lib:
    """One libfgumi_b200.so loaded on its own (its own handle, its own tile plan)."""

    def __init__(self, path, l):
        self.path, self.name = path, os.path.basename(path)
        self.so = C.CDLL(path)
        vp, u64 = C.c_void_p, C.c_uint64
        self.so.fgb_create.argtypes = [C.c_int, C.POINTER(l.FgbParams), C.POINTER(vp)]
        self.so.fgb_vote_device.argtypes = [vp, C.POINTER(l.FgbBatch), C.POINTER(l.FgbColumns), vp]
        self.so.fgb_plan_tiles.argtypes = [vp, u64, vp, u64, vp, u64, C.POINTER(u64)]
        self.so.fgb_sort_tiles_by_class.argtypes = [vp, u64, vp]
        self.so.fgb_destroy.argtypes = [vp]
        self.h = vp()
        st = self.so.fgb_create(0, C.byref(l.FgbParams(45, 40, 2, 0, 1)), C.byref(self.h))
        if st != 0:
            raise RuntimeError(f"fgb_create({self.name}) = {st}")
        self.trace = hasattr(self.so, "fgb_pipe_trace")
        if self.trace:
            self.so.fgb_pipe_trace.argtypes = [vp]

    def tiles(self, torch, dev, host, np, tile_dtype):
        """This library's tile plan of the batch (the stage cap is a compile-time constant), class-sorted, on the device."""
        n = C.c_uint64(0)
        up, rp = host.units.ctypes.data_as(C.c_void_p), host.reads.ctypes.data_as(C.c_void_p)
        assert self.so.fgb_plan_tiles(up, host.n_units, rp, host.n_reads, None, 0, C.byref(n)) == 0
        t = np.zeros(int(n.value), dtype=tile_dtype)
        assert self.so.fgb_plan_tiles(up, host.n_units, rp, host.n_reads, t.ctypes.data_as(C.c_void_p), len(t), C.byref(n)) == 0
        counts = (C.c_uint64 * 3)()
        assert self.so.fgb_sort_tiles_by_class(t.ctypes.data_as(C.c_void_p), len(t), counts) == 0
        return torch.from_numpy(t.view(np.uint8).reshape(-1)).to(dev), len(t), tuple(int(c) for c in counts)

    def read_trace(self, np):
        buf = np.zeros(TRACE_WORDS, dtype=np.uint64)
        assert self.so.fgb_pipe_trace(buf.ctypes.data_as(C.c_void_p)) == 0
        return buf.astype(np.float64)

    def close(self):
        self.so.fgb_destroy(self.h)


def split(tr, t_ms, launches):
    """Fractions of the kernel's time from one traced round's counters (vote_kernel.cuh g_pipe_trace)."""
    cta, ctas, warp_cyc, tiles = tr[0], tr[10], tr[2], tr[9]
    clk_mhz = warp_cyc / (ctas * 8) / (t_ms * 1e-3) / 1e6     # ctas counts every launch's CTAs
    period = (warp_cyc / (ctas * 8)) / (tiles / ctas) if tiles else None     # cycles per tile per CTA
    return {
        "ctas": ctas / launches,
        "implied_sm_mhz": clk_mhz,
        "producer_wait_empty_frac": tr[1] / cta if cta else None,
        "consumer_wait_full_frac": tr[3] / warp_cyc,
        "consumer_vote_frac": tr[4] / warp_cyc,
        "consumer_fast_pass_frac": tr[5] / warp_cyc,
        "consumer_slow_pass_frac": tr[6] / warp_cyc,
        "consumer_other_frac": 1.0 - (tr[3] + tr[4]) / warp_cyc,
        "tiles_not_landed_on_arrival_frac": tr[7] / tiles if tiles else None,
        "issue_to_full_us_of_those": (tr[8] / tr[7]) / clk_mhz if tr[7] else None,
        "tile_period_us": period / clk_mhz if tiles else None,
        # warp 0 passing `full` -> the last warp's release of the stage, and last minus first release, per tile
        "stage_hold_us": tr[11] / tiles / clk_mhz if tiles else None,
        "release_skew_us": tr[12] / tiles / clk_mhz if tiles else None,
    }


def run(args):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import fgumi_b200 as fg
    from fgumi_b200 import synth
    from fgumi_b200.engine import TILE_DTYPE
    from fgumi_b200.shard import partition_by_reads
    l = fg.lib
    assert os.path.abspath(l.LIB_PATH) == TRACE_LIB, l.LIB_PATH
    dev = "cuda:0"
    torch.cuda.set_device(0)
    props = torch.cuda.get_device_properties(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": props.name, "sms": props.multi_processor_count, "nvidia_smi": smi}), flush=True)
    s = torch.cuda.current_stream().cuda_stream
    trace = Lib(TRACE_LIB, l)
    intree = Lib(INTREE_LIB, l)
    novote = Lib(NOVOTE_LIB, l)
    others = [Lib(p, l) for p in args.compare]

    def time_launches(lib, bs, cs, n):
        lib.so.fgb_vote_device(lib.h, C.byref(bs), C.byref(cs), C.c_void_p(s))       # warm
        torch.cuda.synchronize()
        if lib.trace:
            lib.read_trace(np)                                                        # zero the counters
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
        ev[0].record()
        for i in range(n):
            st = lib.so.fgb_vote_device(lib.h, C.byref(bs), C.byref(cs), C.c_void_p(s))
            assert st == 0, (lib.name, st)
            ev[i + 1].record()
        torch.cuda.synchronize()
        return [ev[i].elapsed_time(ev[i + 1]) for i in range(n)]

    def leg(name, depths, gbps_bytes):
        tb = synth.device_batch(torch, dev, depths, 150, 1e-3, seed=42)
        out = fg.DeviceColumns(tb.host.n_out, dev)
        plans = {}
        for lib in [trace, intree, novote] + others:
            tt, nt, cls = lib.tiles(torch, dev, tb.host, np, TILE_DTYPE)
            b = synth.TorchBatch(tb.bases, tb.quals, tb.reads, tb.units, tt, tb.host, cls)
            b.n_tiles = nt
            plans[lib.name] = (b, b.struct(), nt, cls)
        cs = out.struct()
        res = {"leg": name, "families": int(len(depths)), "tiles": plans[intree.name][2],
               "class_tiles": plans[intree.name][3]}
        # reference outputs: the in-tree library
        time_launches(intree, plans[intree.name][1], cs, 1)
        ref = [x.clone() for x in (out.base, out.qual, out.depth, out.errors)]
        ms = {lib.name: [] for lib in [intree, trace] + others}
        trs = {}
        same = {}
        for r in range(args.rounds):
            for lib in [intree, trace] + others:
                for x in (out.base, out.qual, out.depth, out.errors):
                    x.fill_(0x55)
                t = time_launches(lib, plans[lib.name][1], cs, args.launches)
                ms[lib.name].append(float(np.median(t)))
                if lib.trace:
                    trs[lib.name] = lib.read_trace(np)
                ok = all(torch.equal(a, b) for a, b in zip(ref, (out.base, out.qual, out.depth, out.errors)))
                same[lib.name] = same.get(lib.name, True) and ok
        del ref
        res["ms_per_launch"] = {k: {"median": float(np.median(v)), "min": min(v), "max": max(v), "rounds": v}
                                for k, v in ms.items()}
        res["outputs_equal_in_tree"] = same
        res["tb_s"] = {k: gbps_bytes / (float(np.median(v)) * 1e-3) / 1e12 for k, v in ms.items()}
        # the stall split of each traced build's last round (args.launches launches): the in-tree sources' and any
        # traced --compare library's
        res["trace"] = split(trs[trace.name], ms[trace.name][-1], args.launches)
        res["trace_compare"] = {k: split(v, ms[k][-1], args.launches) for k, v in trs.items() if k != trace.name}
        if name == "config2":
            # data movement alone: the no-vote build on the same tiles (outputs are constants, not compared)
            nv = [float(np.median(time_launches(novote, plans[novote.name][1], cs, args.launches)))
                  for _ in range(args.rounds)]
            res["ceiling_novote_ms"] = {"median": float(np.median(nv)), "min": min(nv), "max": max(nv),
                                        "tb_s": gbps_bytes / (float(np.median(nv)) * 1e-3) / 1e12}
            del out, cs
            torch.cuda.empty_cache()
            nb = tb.host.n_bytes // 8 * 8
            b64 = tb.bases[:nb].view(torch.int64)
            q64 = tb.quals[:nb].view(torch.int64)
            o64 = torch.empty_like(b64)

            def ev_ms(fn):
                fn(); torch.cuda.synchronize()
                e = [torch.cuda.Event(enable_timing=True) for _ in range(args.launches + 1)]
                e[0].record()
                for i in range(args.launches):
                    fn(); e[i + 1].record()
                torch.cuda.synchronize()
                return float(np.median([e[i].elapsed_time(e[i + 1]) for i in range(args.launches)]))
            r_ms = ev_ms(lambda: torch.sum(b64))
            x_ms = ev_ms(lambda: torch.bitwise_xor(b64, q64, out=o64))
            res["ceiling_torch_read_only"] = {"ms": r_ms, "bytes": nb, "tb_s": nb / (r_ms * 1e-3) / 1e12}
            res["ceiling_torch_2r1w"] = {"ms": x_ms, "bytes": 3 * nb, "tb_s": 3 * nb / (x_ms * 1e-3) / 1e12}
            del o64, b64, q64
        print(json.dumps(res), flush=True)
        del tb
        torch.cuda.empty_cache()

    def vbytes(d):
        return 2 * int(d.sum()) * 150 + 6 * len(d) * 150 + 8 * (int(d.sum()) + len(d)) + 8 * len(d)

    for name in args.legs.split(","):
        if name == "config2":
            d = np.full(args.units, 8, np.int64)
        elif name == "depth3":
            d = np.full(args.units, 3, np.int64)
        elif name == "zipf":
            all_d = synth.zipf_depths(100_000_000, 1, 100, 1.0, seed=42).astype(np.int64)
            lo, hi = partition_by_reads(all_d, 16)[0]
            d = np.sort(all_d[lo:hi], kind="stable")
            del all_d
        else:
            raise SystemExit(f"unknown leg {name}")
        leg(name, d, vbytes(d))
    for lib in [trace, intree, novote] + others:
        lib.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="store_true", help="rebuild the diagnostic libraries")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--compare", nargs="*", default=[], help="more libraries to time against the in-tree one")
    ap.add_argument("--legs", default="config2,depth3,zipf")
    ap.add_argument("--units", type=int, default=10_000_000)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    args.compare = [os.path.abspath(p) for p in args.compare]
    os.environ["FGUMI_B200_LIB"] = TRACE_LIB          # before the package is first imported (build_libs imports it)
    build_libs(args.build or args.build_only)
    if not args.build_only:
        run(args)


if __name__ == "__main__":
    main()
