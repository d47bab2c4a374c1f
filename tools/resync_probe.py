"""Cost of bf_resident_resync on a resident batch of 100 000 runs x 256 steps in the shape of BASELINE configs[2] (cfg3: phase
planes only), against what a batcher did before it: bf_resident_upload of every record, then the touched tick and the
bf_resident_schedule that follow.  Two twin batches with limiter inputs hold the same state; the caller's records (pinned) are
snapshots of it where 0 %, 0.1 % and 1 % of the runs drifted (one phase code each).  Each round restores both batches (untimed),
then times, on alternate batches in alternate order: the resync alone, the resync + touched tick + schedule, and the upload +
touched tick + schedule.  Times are host clocks around calls that end in a device synchronise: median and min-max over the
rounds.  Also reported: the runs each path lists (touched tick, schedule) and the resync's drifted runs.

usage: python tools/resync_probe.py [--runs N] [--rounds K] [--warmup W] [--out FILE]"""
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

S = 256
NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
TABLES = dict(story_limit=[3, 0, 0, 0], queue_limit=[0, 4, 0], queue_aging_s=[0, 60, 10], global_limit=0)


def timed(f):
    t = time.perf_counter()
    out = f()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.runs
    fr = Frontier(0)
    rng = np.random.default_rng(1)
    ts = synth.topologies(3, 0, n, S)
    slots = fr.put_topologies(ts)
    L = make_layout(S, 0, A.F_ALL_OUT)
    base = synth.state(3, 0, n, L, slots, ts)
    hs = [fr.resident_create(L, n) for _ in range(2)]
    q = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
    q["run"], q["story_key"], q["queue_key"] = np.arange(n), np.arange(n) % 4, np.arange(n) % 3
    q["priority"], q["queued_since"], q["run_phase"] = np.arange(n) % 5, A.SCHED_NONE, A.PHASE_RUNNING
    for h in hs:
        fr.resident_sched(h)
        fr.resident_sched_put(h, q)
    rec = fr.alloc_pinned(base.nbytes).view(np.uint8).reshape(base.shape)

    def restore(h):
        fr.resident_upload(h, 0, base)
        fr.resident_tick_touched(h, n, NONE, n, n * S)
        fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=n * S)], TABLES, 0)

    def tick_and_schedule(h):
        t = fr.resident_tick_touched(h, n, NONE, n, n * S)
        s = fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=n * S)], TABLES, 0)["parts"][0]
        return t["n_listed"], s["n_listed"]

    lines = []
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    lines.append("resync_probe: %d runs x %d steps (cfg3 shape), %d rounds; %s" % (n, S, a.rounds, gpu))
    fmt = lambda t: "median %8.1f us (%.1f - %.1f)" % (np.median(t) * 1e6, np.min(t) * 1e6, np.max(t) * 1e6)  # noqa: E731
    for share in (0.0, 0.001, 0.01):
        snap = base.copy()
        k = int(round(share * n))
        drift = rng.choice(n, size=k, replace=False)
        snap[drift, L.off_phase] ^= 1   # step 0's phase code, bit 0
        rec[:] = snap
        t_rs, t_rsts, t_up = [], [], []
        listed = {}
        for r in range(a.warmup + a.rounds):
            hr, hu = (hs[0], hs[1]) if r % 2 == 0 else (hs[1], hs[0])
            restore(hr)
            restore(hu)
            order = [("resync", hr), ("upload", hu)] if r % 4 < 2 else [("upload", hu), ("resync", hr)]
            for kind, h in order:
                if kind == "resync":
                    t1, out = timed(lambda: fr.resident_resync(h, n, rec, items_cap=max(k, 1)))
                    t2, ls = timed(lambda: tick_and_schedule(h))
                    if r >= a.warmup:
                        t_rs.append(t1); t_rsts.append(t1 + t2)
                    listed["resync"] = (out["n_drifted"],) + ls
                else:
                    t1, _ = timed(lambda: fr.resident_upload(h, 0, rec))
                    t2, ls = timed(lambda: tick_and_schedule(h))
                    if r >= a.warmup:
                        t_up.append(t1 + t2)
                    listed["upload"] = ls
        lines.append("%.1f %% of the runs drifted (%d):" % (share * 100, k))
        lines.append("  resync alone:                          %s; drifted %d" % (fmt(t_rs), listed["resync"][0]))
        lines.append("  resync + touched tick + schedule:      %s; listed %d by the tick, %d by the schedule"
                     % ((fmt(t_rsts),) + listed["resync"][1:]))
        lines.append("  upload + touched tick + schedule:      %s; listed %d by the tick, %d by the schedule"
                     % ((fmt(t_up),) + listed["upload"]))
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    fr.free_pinned(rec)
    fr.close()


if __name__ == "__main__":
    main()
