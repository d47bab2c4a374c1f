"""Steady-state limiter cost of a resident batch: touched tick + bf_schedule against touched tick + bf_resident_schedule.

A 100 000-run batch of up to 256 steps; each tick 1 % of the runs get a phase delta and a new limiter input.  The two loops
alternate within each round, so both see the same machine; each round reports the median per-tick time of each loop.  Bytes
across PCIe per tick are computed from the record sizes and the lists the calls return.  Then one schedule over two batches
(256 and 1024 steps) in one call.  The card's name and power limit are read in the same run.

    python tools/sched_probe.py [--runs 100000] [--ticks 20] [--rounds 5] > tools/sched_probe_h100.txt"""
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
from tests import sched_resident as SRM  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:   # the figure is reported either way, with what is known of the card
        return "unknown (%s)" % e


def batch(rng, fr, n, smin, smax):
    ts = randgen.random_topologies(rng, 64, smin, smax)
    slots = fr.put_topologies(ts)
    L, state, topo = randgen.random_state(rng, ts, slots, n, A.F_COND | A.F_DECISION, phase_mix="progress")
    return ts, L, state, topo


def inputs(rng, runs, now):
    p = SRM.defaults(runs.size)
    p["run"] = runs
    p["story_key"] = rng.integers(0, 500, size=runs.size)
    p["queue_key"] = rng.integers(0, 8, size=runs.size)
    p["priority"] = rng.integers(0, 5, size=runs.size)
    p["queued_since"] = np.where(rng.random(runs.size) < 0.5, SRM.NONE, rng.integers(0, now, size=runs.size))
    p["run_phase"] = A.PHASE_RUNNING
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--ticks", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    fr = Frontier(0)
    n = a.runs
    ts, L, state, topo = batch(rng, fr, n, 200, 256)
    tables = dict(story_limit=rng.choice([0, 2, 5, 50], size=500).astype(np.int32), queue_limit=np.array([0, 100, 1000, 5000] * 2, np.int32),
                  queue_aging_s=np.array([60] * 8, np.int32), global_limit=50_000)
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, state)
    fr.resident_sched(h)
    now = 1_000_000
    inp = inputs(rng, np.arange(n, dtype=np.uint32), now)
    fr.resident_sched_put(h, inp)
    k = n // 100
    stride = A.sched_stride(L.words)

    def deltas():
        runs = rng.choice(n, size=k, replace=False)
        d = np.zeros(k, Frontier.DELTA_DTYPE)
        d["run"] = runs
        d["index"] = [int(rng.integers(0, int(ts.S[int(topo[r])]))) for r in runs]
        d["field"] = A.DELTA_PHASE
        d["code"] = rng.choice([0, 1, 2, 3, 14], size=k)
        return d, runs

    fr.resident_tick_touched(h, n, np.zeros(0, Frontier.DELTA_DTYPE), n, 1 << 24)
    fr.resident_schedule([dict(handle=h, n_runs=n)], tables, now)   # the first schedule lists every run
    times = {"bf_schedule": [], "bf_resident_schedule": []}
    bytes_ = {"bf_schedule": [], "bf_resident_schedule": []}
    for _ in range(a.rounds):
        for which in ("bf_schedule", "bf_resident_schedule"):
            per = []
            for _ in range(a.ticks):
                d, runs = deltas()
                p = inputs(rng, np.sort(runs).astype(np.uint32), now)
                now += 1
                inp[p["run"]] = p
                t0 = time.perf_counter()
                fr.resident_tick_touched(h, n, d, n, 1 << 24)
                if which == "bf_schedule":
                    host_sched = SRM.sched_runs(inp, now)   # every queued run's elapsed time moved: the host rewrites them all
                    fr.schedule(L, n, host_sched, **tables)
                    b = n * 32 + n * stride
                else:
                    fr.resident_sched_put(h, p)
                    got = fr.resident_schedule([dict(handle=h, n_runs=n, events_cap=1 << 22)], tables, now)["parts"][0]
                    b = p.nbytes + got["n_listed"] * (4 + 16) + got["n_events"] * 2 + 16
                per.append(time.perf_counter() - t0)
                bytes_[which].append(b)
            times[which].append(float(np.median(per)))
    print("card: %s" % card())
    print("batch: %d runs x up to %d steps (%d words), %d deltas and %d limiter-input puts per tick, %d ticks x %d rounds per loop"
          % (n, L.steps_max, L.words, k, k, a.ticks, a.rounds))
    for which in times:
        t = np.array(times[which]) * 1e3
        print("touched tick + %-21s median %.3f ms per tick (round medians %s ms); %.2f MB across PCIe per tick (schedule part)"
              % (which, float(np.median(t)), " ".join("%.3f" % x for x in t), float(np.mean(bytes_[which])) / 1e6))
    # two batches of different widths in one call
    ts2, L2, state2, topo2 = batch(rng, fr, 20_000, 900, 1024)
    h2 = fr.resident_create(L2, 20_000)
    fr.resident_upload(h2, 0, state2)
    fr.resident_sched(h2)
    fr.resident_sched_put(h2, inputs(rng, np.arange(20_000, dtype=np.uint32), now))
    fr.resident_tick_touched(h2, 20_000, np.zeros(0, Frontier.DELTA_DTYPE), 20_000, 1 << 24)
    per = []
    for i in range(a.ticks):
        t0 = time.perf_counter()
        got = fr.resident_schedule([dict(handle=h, n_runs=n, events_cap=1 << 22), dict(handle=h2, n_runs=20_000, events_cap=1 << 22)],
                                   tables, now + i)
        per.append(time.perf_counter() - t0)
    print("two batches (%d x 256 and 20000 x 1024 steps) in one bf_resident_schedule: median %.3f ms, min %.3f, max %.3f ms "
          "(no state change between calls: %d + %d runs listed in the last)" % (n, float(np.median(per)) * 1e3, min(per) * 1e3,
                                                                             max(per) * 1e3, got["parts"][0]["n_listed"],
                                                                             got["parts"][1]["n_listed"]))
    fr.close()


if __name__ == "__main__":
    main()
