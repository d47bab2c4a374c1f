"""Cost of the run-control pass of bf_resident_fire: two resident batches of 100 000 runs with K = 4 timer slots each, every slot
armed and 1 % of the timers due at `now`; one batch also has a run-control area with a story and a drain deadline armed for every
run (none due, so every repetition sees the same batch).  Repetitions alternate between the batches; each re-arms the fired timers
(not timed) and times one fire as the caller sees it (host wall clock around the synchronous call).  Prints one line per batch.

    python tools/runctl_probe.py [--runs 100000] [--k 4] [--due 0.01] [--reps 50]
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200 import Frontier  # noqa: E402
from bobrapet_b200.records import make_layout  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--due", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    fr = Frontier(0)
    L = make_layout(256, 0, A.F_DECISION)
    n, K = a.runs, a.k
    rng = np.random.default_rng(0)
    rq = np.zeros(n * K, dtype=Frontier.TIMER_DTYPE)
    rq["run"] = np.repeat(np.arange(n, dtype=np.uint32), K)
    rq["step"] = np.tile(np.arange(K, dtype=np.uint16) * 7, n)
    rq["code"] = A.DEC_PENDING   # wake-only: a fire changes no record
    due = rng.random(n * K) < a.due
    rq["deadline"] = np.where(due, 100, 1_000_000).astype(np.uint32)
    hs = {}
    for name in ("without the area", "with the area"):
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, np.zeros((n, L.state_stride), np.uint8))
        fr.resident_timers(h, K)
        fr.resident_timers_arm(h, rq)
        if name == "with the area":
            fr.resident_runctl(h)
            p = np.zeros(n, dtype=Frontier.RUNCTL_PUT_DTYPE)
            p["run"] = np.arange(n)
            p["story_deadline"] = 2_000_000
            p["drain_deadline"] = 3_000_000
            fr.resident_runctl_put(h, p)
        hs[name] = h
    fired = np.zeros(n * (K + 2), dtype=Frontier.FIRED_DTYPE)
    times = {k: [] for k in hs}
    for rep in range(a.reps + 5):
        for name, h in hs.items():
            t0 = time.perf_counter()
            out = fr.resident_fire(h, n, 100, fired=fired)
            dt = time.perf_counter() - t0
            assert out["n_fired"] == int(due.sum()) and out["next_deadline"] == 1_000_000
            if rep >= 5:
                times[name].append(dt)
            fr.resident_timers_arm(h, rq[due])   # the fired timers again
    for name, t in times.items():
        us = np.array(t) * 1e6
        print("runctl_probe: runs=%d K=%d due=%.3f %-16s bf_resident_fire wall us: median %.1f  p10 %.1f  p90 %.1f  (%d reps)" %
              (n, K, a.due, name, np.median(us), np.percentile(us, 10), np.percentile(us, 90), a.reps))
    fr.close()


if __name__ == "__main__":
    main()
