"""Touched ticks of three width classes: one bf_resident_tick_touched_many call against three bf_resident_tick_touched calls.

Two twin sets of batches (80 000 runs x 256 steps, 15 000 x 512 with cond and decision planes, 5 000 x 1024 with a child area)
take the same deltas, 1 % of the runs with a changed phase code per batch and tick.  The sets alternate tick by tick in one
process; each tick is timed with a host clock around calls that end in a synchronisation.  Prints the median and range of each
form over the timed ticks, with the card's name and power limit, and checks that both forms listed the same runs.

    python tools/tick_many_probe.py [--ticks 30] [--warmup 5]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200 import Frontier  # noqa: E402
from tests import randgen  # noqa: E402

SHAPES = [("80000x256", 80_000, 128, 256, False, 0), ("15000x512+dec", 15_000, 300, 512, False, A.F_COND | A.F_DECISION | A.F_ALL_OUT),
          ("5000x1024+child", 5_000, 600, 1000, True, A.F_ALL_OUT)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    fr = Frontier(0)
    batches = []   # (name, n, L, handle of set M, handle of set S)
    for name, n, s_lo, s_hi, par, fields in SHAPES:
        ts = randgen.random_topologies(rng, 16, s_lo, s_hi, max_deg=4, parallel=par, fill=0.5)
        slots = fr.put_topologies(ts)
        L, state, _ = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
        hm, hs = fr.resident_create(L, n), fr.resident_create(L, n)
        fr.resident_upload(hm, 0, state)
        fr.resident_upload(hs, 0, state)
        batches.append((name, n, L, hm, hs))
    caps = [(n, 64 * n) for _, n, _, _, _ in batches]
    bufs = [{k: fr.alloc_pinned(4 * rc if k != "events" else 2 * ec).view(np.uint32 if k != "events" else np.uint16)
             for k in ("runs", "head", "events")} for rc, ec in caps]

    def deltas(n, L):
        k = max(1, n // 100)
        d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
        d["run"] = rng.choice(n, size=k, replace=False)
        d["index"] = rng.integers(0, 32 * L.words, size=k)
        d["field"] = A.DELTA_PHASE
        d["code"] = rng.choice([0, 2, 3, 4, 14], size=k)
        return d

    t_many, t_single = [], []
    for t in range(args.warmup + args.ticks):
        ds = [deltas(n, L) for _, n, L, _, _ in batches]
        for form in ((0, 1) if t % 2 == 0 else (1, 0)):
            if form == 0:
                parts = [dict(handle=hm, n_runs=n, deltas=d, runs_cap=rc, events_cap=ec, **b)
                         for (_, n, _, hm, _), d, (rc, ec), b in zip(batches, ds, caps, bufs)]
                t0 = time.perf_counter()
                got = fr.resident_tick_touched_many(parts)
                dt = time.perf_counter() - t0
                lm = [g["runs"].copy() for g in got]
            else:
                t0 = time.perf_counter()
                got = [fr.resident_tick_touched(hs, n, d, rc, ec, **b) for (_, n, _, _, hs), d, (rc, ec), b in zip(batches, ds, caps, bufs)]
                dt = time.perf_counter() - t0
                ls = [g["runs"].copy() for g in got]
            if t >= args.warmup:
                (t_many if form == 0 else t_single).append(dt * 1e3)
        assert all(np.array_equal(a, b) for a, b in zip(lm, ls)), "the two forms listed different runs"
    print("card: %s" % card())
    print("batches: %s; 1%% of runs with a changed phase code per batch and tick; %d ticks after %d warm-up, forms alternating" %
          (", ".join(b[0] for b in batches), args.ticks, args.warmup))
    for name, v in (("bf_resident_tick_touched_many (1 call)", t_many), ("bf_resident_tick_touched x3", t_single)):
        v = np.array(v)
        print("%-40s median %.3f ms  range %.3f .. %.3f ms" % (name, np.median(v), v.min(), v.max()))
    print("median saving: %.3f ms per tick" % (np.median(t_single) - np.median(t_many)))
    for b in bufs:
        for a in b.values():
            fr.free_pinned(a)
    fr.close()


if __name__ == "__main__":
    main()
