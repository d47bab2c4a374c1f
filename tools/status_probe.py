"""Cost of bf_resident_status on a resident batch of 100 000 runs x 256 steps (parallel steps, so the batch has a child area),
for 1 % of the runs (a touched tick's DONE runs, or a commit's written runs) and for all of them, next to a touched tick that
changed 1 % of the phase codes.  Times are host clocks around calls that end in a device synchronise; each figure is the median
and the min-max range over the rounds.

usage: python tools/status_probe.py [--runs N] [--rounds K] [--warmup W] [--out FILE]"""
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

S = 256


def timed(f):
    t = time.perf_counter()
    f()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    fr = Frontier(0)
    rng = np.random.default_rng(1)
    ts = randgen.random_topologies(rng, 16, S // 2, S, max_deg=4, parallel=True, fill=0.5)
    slots = fr.put_topologies(ts)
    n = a.runs
    L, st, _ = randgen.random_state(rng, ts, slots, n, A.F_DECISION | A.F_ALL_OUT, phase_mix="progress")
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    fr.resident_tick_touched(h, n, np.zeros(0, dtype=Frontier.DELTA_DTYPE), n, n * S)
    few = np.sort(rng.choice(n, size=n // 100, replace=False)).astype(np.uint32)
    t_few, t_all, t_tick = [], [], []
    for k in range(a.warmup + a.rounds):
        d = np.zeros(n * S // 100 // 8, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"] = rng.integers(0, n, d.size), rng.integers(0, 128, d.size)
        d["field"], d["code"] = A.DELTA_PHASE, rng.choice([2, 3, 4, 13], d.size)
        _, ui = np.unique(d[["run", "index"]], return_index=True)
        d = np.ascontiguousarray(d[np.sort(ui)])
        tt = timed(lambda: fr.resident_tick_touched(h, n, d, n, n * S))
        tf = timed(lambda: fr.resident_status(h, n, few, events_cap=few.size * S))
        ta = timed(lambda: fr.resident_status(h, n, events_cap=n * S))
        if k >= a.warmup:
            t_tick.append(tt); t_few.append(tf); t_all.append(ta)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    fmt = lambda t: "median %.1f us (%.1f - %.1f)" % (np.median(t) * 1e6, np.min(t) * 1e6, np.max(t) * 1e6)  # noqa: E731
    text = "\n".join(["status_probe: %d runs x %d steps, %d rounds; %s" % (n, S, a.rounds, gpu),
                      "touched tick (1 %% of the codes changed): %s" % fmt(t_tick),
                      "status, 1 %% of the runs (%d):         %s" % (few.size, fmt(t_few)),
                      "status, every run:                    %s" % fmt(t_all)])
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    fr.close()


if __name__ == "__main__":
    main()
