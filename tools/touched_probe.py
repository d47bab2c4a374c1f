"""tools/touched_probe.py: what a touched tick (bf_resident_tick_touched) costs against a changed-only compact tick
(bf_resident_tick_compact with BF_EVAL_CHANGED_ONLY) as the share of touched runs grows.

A 100 000 x 256 resident batch (BASELINE configs[2] shape, synth cfg 3) is uploaded twice; every tick sends the same deltas,
about 3 phase deltas per touched run, to both batches, from pinned buffers, and the two tick kinds alternate.  Each call is
synchronous (it ends with a device synchronise), so the host clock around it is the time of the whole tick.  The deltas of a
share are generated before its ticks, and the kind that goes first alternates from tick to tick: the call that follows the
host's copy of the next deltas (the GPU idle meanwhile) is not always the same kind.  The listed
runs, head words and events of the two are byte-compared at every tick.  Prints the card, its power limit, and per share the
median us per tick of each.

    python tools/touched_probe.py [--runs 100000] [--ticks 30]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200 import Frontier, synth  # noqa: E402
from bobrapet_b200.records import make_layout  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--ticks", type=int, default=30, help="timed ticks of each kind per share")
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    n, S = a.runs, a.steps
    fr = Frontier(0)
    print("card: %s" % card())
    ts = synth.topologies(3, 0, n, S)
    slots = fr.put_topologies(ts)
    L = make_layout(S, 0, 0)
    state = synth.state(3, 0, n, L, slots, ts)
    hT, hC = fr.resident_create(L, n), fr.resident_create(L, n)
    fr.resident_upload(hT, 0, state)
    fr.resident_upload(hC, 0, state)
    max_d = 3 * n
    ev_cap = 64 * n
    p_d = fr.alloc_pinned(max_d * 8).view(Frontier.DELTA_DTYPE)
    bufs = {"runs": fr.alloc_pinned(n * 4).view(np.uint32), "head": fr.alloc_pinned(n * 4).view(np.uint32),
            "events": fr.alloc_pinned(ev_cap * 2).view(np.uint16)}
    c_head = fr.alloc_pinned(n * 4).view(np.uint32)
    c_ev = fr.alloc_pinned(ev_cap * 2).view(np.uint16)
    rng = np.random.default_rng(12345)
    none = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
    fr.resident_tick_touched(hT, n, none, n, ev_cap, **bufs)          # the first tick of each kind evaluates every run
    fr.resident_tick_compact(hC, n, none, ev_cap, flags=A.EVAL_CHANGED_ONLY, head=c_head, events=c_ev)
    print("%8s %8s %12s %16s %8s %10s %22s" % ("share", "runs", "touched_us", "changed_only_us", "ratio", "listed", "touched first/second"))
    for share in (0.0001, 0.001, 0.01, 0.1, 1.0):
        k = max(1, int(round(n * share)))
        tt, tc, listed = [], [], 0
        first = {True: [], False: []}   # touched-tick times when it went first / second
        ticks = []
        for it in range(a.warmup + a.ticks):
            runs = rng.choice(n, size=k, replace=False) if k < n else np.arange(n)
            d = np.zeros(3 * k, dtype=Frontier.DELTA_DTYPE)
            d["run"] = np.repeat(runs, 3)
            d["index"] = (np.repeat(rng.integers(0, S - 3, size=k), 3) + np.tile(np.arange(3), k)).astype(np.uint16)
            d["field"] = A.DELTA_PHASE
            d["code"] = rng.choice([0, 1, 2, 3, 3, 3, 4, 13], size=3 * k)
            ticks.append(d)
        for it, d in enumerate(ticks):
            dd = p_d[:3 * k]
            dd[:] = d

            def touched():
                t0 = time.perf_counter()
                o = fr.resident_tick_touched(hT, n, dd, n, ev_cap, **bufs)
                return o, time.perf_counter() - t0

            def changed():
                t0 = time.perf_counter()
                r = fr.resident_tick_compact(hC, n, dd, ev_cap, flags=A.EVAL_CHANGED_ONLY, head=c_head, events=c_ev)
                return r, time.perf_counter() - t0

            if it % 2:
                (head, ev, n_ev, _, n_listed), dc = changed()
                out, dt = touched()
            else:
                out, dt = touched()
                (head, ev, n_ev, _, n_listed), dc = changed()
            lr = np.nonzero(head & A.HEAD_LISTED)[0]
            if out["full"] or not (np.array_equal(out["runs"], lr) and np.array_equal(out["head"], head[lr]) and np.array_equal(out["events"], ev)):
                print("MISMATCH at share %g tick %d: full=%d listed %d / %d" % (share, it, out["full"], out["n_listed"], n_listed))
                return 1
            if it >= a.warmup:
                tt.append(dt * 1e6)
                first[it % 2 == 0].append(dt * 1e6)
                tc.append(dc * 1e6)
                listed += out["n_listed"]
        mt, mc = float(np.median(tt)), float(np.median(tc))
        print("%7.2f%% %8d %12.1f %16.1f %8.2f %10d %11.1f / %.1f" % (share * 100, k, mt, mc, mt / mc, listed // a.ticks,
                                                                     float(np.median(first[True])), float(np.median(first[False]))))
    print("outputs byte-identical at every tick")
    fr.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
