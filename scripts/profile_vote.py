"""Profiling driver: build one synthetic batch in device memory and launch the vote kernel a few
times, timed with CUDA events (usage: python scripts/profile_vote.py [units] [depth|zipf] [launches])."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
import fgumi_b200 as fg
from fgumi_b200 import synth

units = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
depth = sys.argv[2] if len(sys.argv) > 2 else "8"
launches = int(sys.argv[3]) if len(sys.argv) > 3 else 5
eng = fg.Engine(0, 45, 40, 1, 2)
if depth.startswith("zipf"):        # BASELINE config 5: P(d) ~ 1/d on 1..100
    w = 1.0 / np.arange(1, 101)
    depths = np.random.default_rng(2).choice(np.arange(1, 101), size=units, p=w / w.sum()).astype(np.int64)
else:
    depths = np.full(units, int(depth), np.int64)
tb = synth.device_batch(torch, "cuda:0", depths, 150, 1e-3, seed=42)
out = fg.DeviceColumns(tb.host.n_out, "cuda:0")
b, c = tb.struct(), out.struct()
lib = fg.lib.load()
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(launches + 1)]
ev[0].record()
for i in range(launches):
    assert lib.fgb_vote_device(eng._h, C.byref(b), C.byref(c), C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    ev[i + 1].record()
torch.cuda.synchronize()
print("units", units, "depth", depth, "ms per launch", [round(ev[i].elapsed_time(ev[i + 1]), 3) for i in range(launches)])
print(eng.stats())
