"""Where a group trip of the packed-lanes kernel spends its time (needs a lib_ab build with -DPACK_STAGES, BF_LIB=...):
clock() deltas per warp, summed over all warps of a CUDA graph of pipelined passes, split into the regions of a trip —
ticket + barrier wait; planes + stages G / B / I / D-prep; stage C; the walk (with the issue of the next group's second
link); load_cut + cond fix-up + stage E; the issue of the next group's copies.  Prints SM cycles per trip and per warp and
pass for each region, and each region's share.  The probe's own clock reads slow the pass; the split, not the time, is
what it is for."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A, Frontier, synth  # noqa: E402
from bobrapet_b200.records import make_layout  # noqa: E402

REGIONS = ("wait", "planes + G/B/I/D-prep", "stage C", "walk", "load_cut + E", "issue")
cfg = int(os.environ.get("CFG", "3"))
n = int(os.environ.get("RUNS", "100000"))
passes = int(os.environ.get("PASSES", "60"))
S = 256
fr = Frontier(0)
dev = torch.device("cuda", 0)
try:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    gpu = "unknown"
L = make_layout(S, 0, (A.F_COND | A.F_DECISION) if cfg == 4 else 0)
sets = []
for k in range(3):
    ts = synth.topologies(cfg, k * 10_000_019, n, S)
    slots = fr.put_topologies(ts)
    st = synth.state(cfg, k * 10_000_019, n, L, slots, ts)
    sets.append((torch.from_numpy(st).to(dev), torch.zeros((n, L.result_stride), dtype=torch.uint8, device=dev),
                 torch.zeros(4, dtype=torch.int64, device=dev)))
ws = torch.cuda.Stream()


def one(k):
    d_state, d_result, d_counts = sets[k % 3]
    fr.eval_device(L, n, d_state.data_ptr(), d_result.data_ptr(), d_counts.data_ptr(), ws.cuda_stream,
                   flags=A.EVAL_COUNTS_SET | A.EVAL_PIPELINED)


lib = fr._lib
tot = np.zeros(8, dtype=np.uint64)
with torch.cuda.stream(ws):
    for k in range(6):
        one(k)
torch.cuda.synchronize()
gr = torch.cuda.CUDAGraph()
with torch.cuda.graph(gr, stream=ws, capture_error_mode="thread_local"):
    for k in range(passes):
        one(k)
with torch.cuda.stream(ws):
    gr.replay()
torch.cuda.synchronize()
assert lib.bf_debug_pack_stages(tot.ctypes.data_as(C.c_void_p)) == 0   # zeroes the totals of the warm-up
with torch.cuda.stream(ws):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ws)
    gr.replay()
    e1.record(ws)
torch.cuda.synchronize()
assert lib.bf_debug_pack_stages(tot.ctypes.data_as(C.c_void_p)) == 0
st = fr.stats()
warps = int(st["last_grid"]) * int(st["last_block"]) // 32
trips = int(tot[6])
cyc = tot[:6].astype(np.float64)
print("stage_probe: cfg%d, %d runs x %d steps, graph of %d pipelined passes; gpu: %s" % (cfg, n, S, passes, gpu))
print("launch: %d CTAs x %d warps, %d slot groups; %.2f us / pass with the probe; %.1f trips per warp and pass" % (
    int(st["last_grid"]), warps // int(st["last_grid"]), int(st["last_stages"]), e0.elapsed_time(e1) * 1e3 / passes,
    trips / warps / passes))
print("%-24s %14s %18s %8s" % ("region", "cycles / trip", "cycles / warp-pass", "share"))
for name, c in zip(REGIONS, cyc):
    print("%-24s %14.1f %18.0f %7.1f%%" % (name, c / trips, c / warps / passes, 100.0 * c / cyc.sum()))
print("%-24s %14.1f %18.0f" % ("total", cyc.sum() / trips, cyc.sum() / warps / passes))
fr.close()
