"""Cost of bf_resident_fire: a resident batch of 100 000 runs with K = 4 timer slots each, every slot armed, 1 % of the timers due
at `now`.  Each repetition re-arms the fired timers (not timed) and times one fire as the caller sees it (host wall clock around
the synchronous call: two launches, the D2H copies and the synchronisation).  Prints one line per batch size.

    python tools/timer_probe.py [--runs 100000] [--k 4] [--due 0.01] [--reps 50]
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
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, np.zeros((n, L.state_stride), np.uint8))
    fr.resident_timers(h, K)
    rng = np.random.default_rng(0)
    rq = np.zeros(n * K, dtype=Frontier.TIMER_DTYPE)
    rq["run"] = np.repeat(np.arange(n, dtype=np.uint32), K)
    rq["step"] = np.tile(np.arange(K, dtype=np.uint16) * 7, n)
    rq["code"] = A.DEC_PENDING   # wake-only: a fire changes no record, so every repetition sees the same batch
    due = rng.random(n * K) < a.due
    rq["deadline"] = np.where(due, 100, 1_000_000).astype(np.uint32)
    fr.resident_timers_arm(h, rq)
    fired = np.zeros(n * K, dtype=Frontier.FIRED_DTYPE)
    times = []
    for rep in range(a.reps + 5):
        t0 = time.perf_counter()
        out = fr.resident_fire(h, n, 100, fired=fired)
        dt = time.perf_counter() - t0
        assert out["n_fired"] == int(due.sum()) and out["next_deadline"] == 1_000_000
        if rep >= 5:
            times.append(dt)
        fr.resident_timers_arm(h, rq[due])   # the fired timers again
    us = np.array(times) * 1e6
    print("timer_probe: runs=%d K=%d due=%.3f fired=%d  bf_resident_fire wall us: median %.1f  p10 %.1f  p90 %.1f  (%d reps)" %
          (n, K, a.due, int(due.sum()), np.median(us), np.percentile(us, 10), np.percentile(us, 90), a.reps))
    fr.close()


if __name__ == "__main__":
    main()
