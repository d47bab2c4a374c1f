"""tools/transfer_probe.py: what moving live runs between resident batches costs on the device (bf_resident_transfer) against the
path a batcher has without it, and what a run pays for the width class it lives in.

A 100 000-run batch of cfg3-shaped Stories (200 to 256 steps, random DAGs, progress-shaped phases, phase planes only) at
steps_max 256, and a destination batch at steps_max 1024 (the class a Story edit past 256 steps moves a run to).
  - transfer: k = 1, 1 000 and 10 000 random runs moved from the source (freshly uploaded, first touched tick done, untimed) into
    the destination, against the host path: bf_resident_download of the source, re-packing the k runs at 1024 steps (numpy),
    bf_resident_upload into the destination and bf_resident_retire of the k runs from the source.  Host clock around calls that
    end in a synchronise; medians of --reps samples.  Both paths' records are byte-compared.
  - class: the same 100 000 runs held at steps_max 256 and at steps_max 1024, a dense tick (pass + download of the result
    records) and a full compact tick of each, alternated in one loop, medians of --ticks samples after --warmup; pass_us: the
    frontier kernels alone per dense tick, from torch.profiler over --prof-ticks ticks in a run of its own.  R: runs per warp
    trip of the pass (bf_stats.last_runs_per_trip; 1 = the one-run-per-warp kernel).  The results of both are byte-compared.
Prints the card and its power limit.

    python tools/transfer_probe.py [--runs 100000] [--reps 5] [--ticks 30] [--warmup 5]
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200.frontier import Frontier  # noqa: E402
from bobrapet_b200.records import make_layout  # noqa: E402
from tests import randgen  # noqa: E402
from tests import reshape as RS  # noqa: E402
from tests.transfer import relay_result, relay_state  # noqa: E402
from tools.narrow_probe import card, pass_kernel_us  # noqa: E402

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
KS = (1, 1000, 10000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5, help="samples per transfer size")
    ap.add_argument("--ticks", type=int, default=30, help="timed ticks per batch and kind")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-ticks", type=int, default=20, help="dense ticks per batch under the profiler")
    a = ap.parse_args()
    n = a.runs
    rng = np.random.default_rng(3)
    fr = Frontier(0)
    ts = randgen.random_topologies(rng, 64, 200, 256, max_deg=4, parallel=False, fill=0.5)
    slots = fr.put_topologies(ts)
    L0, st0, _ = randgen.random_state(rng, ts, slots, n, 0, phase_mix="progress", run_flag_mix=False)
    Ls, Ld = make_layout(256, 0, 0), make_layout(1024, 0, 0)
    st = RS.reshape_state(L0, Ls, st0, n)
    cap_ev = 64 * n
    kmax = max(k for k in KS if k <= n)
    print("card: %s" % card())
    print("source: %d runs of Stories of %d to %d steps at steps_max 256; destination: steps_max 1024; medians in us" % (
        n, int(ts.S.min()), int(ts.S.max())))
    import torch
    torch.cuda.init()

    def source():
        h = fr.resident_create(Ls, n)
        fr.resident_upload(h, 0, st)
        fr.resident_tick_touched(h, n, NONE, n, cap_ev)
        return h
    h, g = source(), fr.resident_create(Ld, kmax)   # warm-up, untimed: every call of both paths once
    fr.resident_transfer(h, g, n, 0, np.arange(kmax, dtype=np.uint32))
    fr.resident_download(h, 0, n - kmax, Ls.state_stride)
    fr.resident_upload(g, 0, relay_state(Ls, Ld, st[:kmax]))
    fr.resident_retire(h, n - kmax, np.arange(kmax, dtype=np.uint32))
    fr.resident_destroy(h)
    fr.resident_destroy(g)
    ok = True
    rows = []
    for k in KS:
        if k > n:
            continue
        t = {x: [] for x in ("dev", "down", "repack", "upload", "retire")}
        for _ in range(a.reps):
            runs = rng.choice(n, size=k, replace=False).astype(np.uint32)
            h, g = source(), fr.resident_create(Ld, kmax)
            t0 = time.perf_counter()
            fr.resident_transfer(h, g, n, 0, runs)
            t["dev"].append((time.perf_counter() - t0) * 1e6)
            h2, g2 = source(), fr.resident_create(Ld, kmax)
            t0 = time.perf_counter()
            recs = fr.resident_download(h2, 0, n, Ls.state_stride)
            t1 = time.perf_counter()
            moved = relay_state(Ls, Ld, recs[runs])
            t2 = time.perf_counter()
            fr.resident_upload(g2, 0, moved)
            t3 = time.perf_counter()
            fr.resident_retire(h2, n, runs)
            t4 = time.perf_counter()
            t["down"].append((t1 - t0) * 1e6); t["repack"].append((t2 - t1) * 1e6)
            t["upload"].append((t3 - t2) * 1e6); t["retire"].append((t4 - t3) * 1e6)
            ok &= np.array_equal(fr.resident_download(g, 0, k, Ld.state_stride), fr.resident_download(g2, 0, k, Ld.state_stride))
            ok &= np.array_equal(fr.resident_download(h, 0, n, Ls.state_stride), fr.resident_download(h2, 0, n, Ls.state_stride))
            for x in (h, g, h2, g2):
                fr.resident_destroy(x)
        rows.append((k, {x: float(np.median(v)) for x, v in t.items()}))
    print("%-8s %11s | %9s %9s %9s %9s %9s %7s" % ("runs", "transfer_us", "down_us", "repack_us", "upload_us", "retire_us",
                                                  "host_sum", "ratio"))
    for k, m in rows:
        hs = m["down"] + m["repack"] + m["upload"] + m["retire"]
        print("%-8d %11.1f | %9.1f %9.1f %9.1f %9.1f %9.1f %6.1fx" % (k, m["dev"], m["down"], m["repack"], m["upload"], m["retire"],
                                                                     hs, hs / m["dev"]))
    # the class: the same runs at 256 and at 1024 steps
    h256, h1024 = fr.resident_create(Ls, n), fr.resident_create(Ld, n)
    fr.resident_upload(h256, 0, st)
    fr.resident_upload(h1024, 0, relay_state(Ls, Ld, st))
    r256, _ = fr.resident_tick(h256, Ls, n, NONE)
    r1024, _ = fr.resident_tick(h1024, Ld, n, NONE)
    ok &= np.array_equal(relay_result(Ls, Ld, r256), r1024)
    p = {x: [] for x in ("d256", "d1024", "c256", "c1024")}
    R = {}
    for i in range(a.warmup + a.ticks):
        for h, L, x in ((h256, Ls, "256"), (h1024, Ld, "1024")):
            t0 = time.perf_counter()
            fr.resident_tick(h, L, n, NONE)
            if i >= a.warmup:
                p["d" + x].append((time.perf_counter() - t0) * 1e6)
            R[x] = fr.stats()["last_runs_per_trip"]
            t0 = time.perf_counter()
            fr.resident_tick_compact(h, n, NONE, cap_ev)
            if i >= a.warmup:
                p["c" + x].append((time.perf_counter() - t0) * 1e6)
    q = {x: float(np.median(v)) for x, v in p.items()}
    k256, k1024 = pass_kernel_us(fr, h256, Ls, n, a.prof_ticks), pass_kernel_us(fr, h1024, Ld, n, a.prof_ticks)
    print("%-6s %4s | %9s | %9s | %9s" % ("class", "R", "pass_us", "dense_us", "compact_us"))
    print("%-6s %4d | %9.1f | %9.1f | %9.1f" % ("256", R["256"], k256, q["d256"], q["c256"]))
    print("%-6s %4d | %9.1f | %9.1f | %9.1f" % ("1024", R["1024"], k1024, q["d1024"], q["c1024"]))
    print("1024 / 256: pass %.2fx, dense %.2fx, compact %.2fx" % (k1024 / max(k256, 1e-9), q["d1024"] / q["d256"], q["c1024"] / q["c256"]))
    fr.resident_destroy(h256)
    fr.resident_destroy(h1024)
    print("records of both transfer paths and results of both classes byte-identical" if ok else "RESULTS DIFFER")
    fr.close()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
