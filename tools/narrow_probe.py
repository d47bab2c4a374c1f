"""tools/narrow_probe.py: what narrowing a live resident batch costs on the device (bf_resident_narrow) against the path a batcher
has without it, and what it buys every pass after it.

A 100 000-run batch of Stories of at most 32 steps (random DAGs, progress-shaped phases), held in a layout a wider Story once
needed.  Legs: steps_max 256 -> 32; 224 -> 32 (7 words per run -> 1); 32 steps with all-PASS cond and all-PENDING decision
planes -> without them.
  - narrow: the call on a freshly uploaded batch that has had its first tick (untimed), against the host path of re-packing
    every run at the narrow layout (numpy), bf_resident_create, uploading the whole batch and the full touched tick a new batch
    needs.  Host clock around calls that end in a synchronise; medians of --reps samples.
    extent_us: bf_resident_extent alone on the same batch.
  - the gain: a dense tick (pass + download of the result records), a full compact tick (pass + compaction, no deltas) and a
    touched tick with 1 % of the runs touched by phase deltas, on the wide batch and on its narrowed twin, alternated in one
    loop; medians of --ticks samples each after --warmup.  R: runs per warp trip of the pass (bf_stats.last_runs_per_trip).
    pass_us: the pass kernels alone (the frontier kernels of a dense tick), their device time per tick from torch.profiler over
    --prof-ticks dense ticks of each batch, taken in a run of its own after the timed ticks.
  Before the first leg, one untimed round of every tick kind on a throwaway batch loads the kernels and sizes the buffers.
The device records of both paths are byte-compared, and so are the results of the wide and the narrowed batch where the narrow
keeps them (dropped decision planes change them: zero planes are PENDING, which a pass applies).  Prints the card and its power
limit.

    python tools/narrow_probe.py [--runs 100000] [--reps 5] [--ticks 40] [--warmup 5]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200.frontier import Frontier  # noqa: E402
from bobrapet_b200.records import make_layout  # noqa: E402
from tests import randgen  # noqa: E402
from tests import reshape as RS  # noqa: E402

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
# name, wide steps_max, wide input fields (all planes zero), narrow steps_max
LEGS = [("256->32", 256, 0, 32), ("224->32", 224, 0, 32), ("-cond-dec", 32, A.F_COND | A.F_DECISION, 32)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def touch(rng, n, share, steps):
    """one phase delta on each of share * n runs"""
    k = max(1, int(n * share))
    d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
    d["run"] = np.sort(rng.choice(n, size=k, replace=False))
    d["index"], d["field"], d["code"] = rng.integers(0, steps, size=k), A.DELTA_PHASE, 3
    return d


def pass_kernel_us(fr, h, L, n, ticks):
    """device time of the frontier kernels per dense tick, from torch.profiler (CUDA activities of the whole process)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(ticks):
            fr.resident_tick(h, L, n, NONE)
    tot = 0.0
    for ev in prof.key_averages():
        if "frontier" in ev.key:
            tot += float(getattr(ev, "device_time_total", 0) or getattr(ev, "cuda_time_total", 0))
    return tot / ticks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5, help="samples per narrow leg")
    ap.add_argument("--ticks", type=int, default=40, help="timed ticks per batch and kind")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-ticks", type=int, default=20, help="dense ticks per batch under the profiler")
    a = ap.parse_args()
    n = a.runs
    rng = np.random.default_rng(1)
    fr = Frontier(0)
    ts = randgen.random_topologies(rng, 64, 16, 32, max_deg=4, parallel=False, fill=0.5)
    slots = fr.put_topologies(ts)
    L0, st0, _ = randgen.random_state(rng, ts, slots, n, 0, phase_mix="progress", run_flag_mix=False)
    cap_ev = 64 * n
    print("card: %s" % card())
    print("batch: %d runs of Stories of at most %d steps; medians in us (narrow: %d samples, ticks: %d each)" % (
        n, int(ts.S.max()), a.reps, a.ticks))
    ok = True
    cost, gain = [], []
    import torch
    torch.cuda.init()
    Lx = make_layout(256, 0, 0)   # warm-up: every tick kind once, untimed
    hx = fr.resident_create(Lx, n)
    fr.resident_upload(hx, 0, RS.reshape_state(L0, Lx, st0, n))
    fr.resident_tick_touched(hx, n, NONE, n, cap_ev)
    fr.resident_tick_compact(hx, n, NONE, cap_ev)
    fr.resident_tick(hx, Lx, n, NONE)
    fr.resident_tick_touched(hx, n, touch(rng, n, 0.01, 32), n, cap_ev)
    fr.resident_destroy(hx)
    for name, s_w, f_w, s_n in LEGS:
        Lw = make_layout(s_w, 0, f_w)
        Ln = make_layout(s_n, 0, 0)
        host = RS.reshape_state(L0, Lw, st0, n)   # the batcher's records at the wide layout

        def source():
            h = fr.resident_create(Lw, n)
            fr.resident_upload(h, 0, host)
            fr.resident_tick_touched(h, n, NONE, n, cap_ev)
            return h
        t = {k: [] for k in ("dev", "extent", "repack", "create", "upload", "full")}
        for _ in range(a.reps):
            h = source()
            t0 = time.perf_counter()
            fr.resident_extent(h, n)
            t1 = time.perf_counter()
            fr.resident_narrow(h, Ln, n)
            t["extent"].append((t1 - t0) * 1e6)
            t["dev"].append((time.perf_counter() - t1) * 1e6)
            t0 = time.perf_counter()
            rec = RS.reshape_state(L0, Ln, st0, n)
            t1 = time.perf_counter()
            g = fr.resident_create(Ln, n)
            t2 = time.perf_counter()
            fr.resident_upload(g, 0, rec)
            t3 = time.perf_counter()
            o = fr.resident_tick_touched(g, n, NONE, n, cap_ev)
            t4 = time.perf_counter()
            assert o["full"] == 1
            t["repack"].append((t1 - t0) * 1e6); t["create"].append((t2 - t1) * 1e6); t["upload"].append((t3 - t2) * 1e6)
            t["full"].append((t4 - t3) * 1e6)
            ok &= np.array_equal(fr.resident_download(h, 0, n, Ln.state_stride), fr.resident_download(g, 0, n, Ln.state_stride))
            fr.resident_destroy(h)
            fr.resident_destroy(g)
        cost.append((name, {k: float(np.median(v)) for k, v in t.items()}))
        # the gain: the wide batch and its narrowed twin, ticked alternately
        hw, hn = source(), source()
        fr.resident_narrow(hn, Ln, n)
        same_results = not (f_w & A.F_DECISION)
        head_w, ev_w, _, _, _ = fr.resident_tick_compact(hw, n, NONE, cap_ev)
        head_n, ev_n, _, _, _ = fr.resident_tick_compact(hn, n, NONE, cap_ev)
        if same_results:
            ok &= np.array_equal(head_w, head_n) and np.array_equal(ev_w, ev_n)
        p = {k: [] for k in ("dw", "dn", "pw", "pn", "tw", "tn")}
        R = {}
        for i in range(a.warmup + a.ticks):
            for h, L, k in ((hw, Lw, "dw"), (hn, Ln, "dn")):
                t0 = time.perf_counter()
                fr.resident_tick(h, L, n, NONE)
                if i >= a.warmup:
                    p[k].append((time.perf_counter() - t0) * 1e6)
                R[k] = fr.stats()["last_runs_per_trip"]
            for h, k in ((hw, "pw"), (hn, "pn")):
                t0 = time.perf_counter()
                fr.resident_tick_compact(h, n, NONE, cap_ev)
                if i >= a.warmup:
                    p[k].append((time.perf_counter() - t0) * 1e6)
            d = touch(rng, n, 0.01, s_n)
            for h, k in ((hw, "tw"), (hn, "tn")):
                t0 = time.perf_counter()
                fr.resident_tick_touched(h, n, d, n, cap_ev)
                if i >= a.warmup:
                    p[k].append((time.perf_counter() - t0) * 1e6)
        ow = fr.resident_tick_touched(hw, n, NONE, n, cap_ev)
        on = fr.resident_tick_touched(hn, n, NONE, n, cap_ev)
        if same_results:
            ok &= np.array_equal(ow["head"], on["head"]) and np.array_equal(ow["events"], on["events"])
        q = {k: float(np.median(v)) for k, v in p.items()}
        q["kw"], q["kn"] = pass_kernel_us(fr, hw, Lw, n, a.prof_ticks), pass_kernel_us(fr, hn, Ln, n, a.prof_ticks)
        gain.append((name, R, q))
        fr.resident_destroy(hw)
        fr.resident_destroy(hn)
    print("%-10s %9s %9s | %9s %9s %9s %9s %9s" % ("leg", "narrow_us", "extent_us", "repack_us", "create_us", "upload_us",
                                                 "fulltk_us", "host_sum"))
    for name, m in cost:
        print("%-10s %9.1f %9.1f | %9.1f %9.1f %9.1f %9.1f %9.1f" % (
            name, m["dev"], m["extent"], m["repack"], m["create"], m["upload"], m["full"],
            m["repack"] + m["create"] + m["upload"] + m["full"]))
    print("%-10s %7s | %9s %9s %6s | %9s %9s %6s | %9s %9s %6s | %9s %9s %6s" % (
        "leg", "R w->n", "pass_w", "pass_n", "gain", "dense_w", "dense_n", "gain", "compact_w", "compact_n", "gain", "t1%_w", "t1%_n",
        "gain"))
    for name, R, q in gain:
        print("%-10s %3d->%-3d | %9.1f %9.1f %5.2fx | %9.1f %9.1f %5.2fx | %9.1f %9.1f %5.2fx | %9.1f %9.1f %5.2fx" % (
            name, R["dw"], R["dn"], q["kw"], q["kn"], q["kw"] / max(q["kn"], 1e-9), q["dw"], q["dn"], q["dw"] / q["dn"],
            q["pw"], q["pn"], q["pw"] / q["pn"], q["tw"], q["tn"], q["tw"] / q["tn"]))
    print("records of both paths and results of the wide and narrowed batches byte-identical" if ok else "RESULTS DIFFER")
    fr.close()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
