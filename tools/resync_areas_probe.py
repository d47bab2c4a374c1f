"""Cost of bf_resident_resync_areas on a resident batch of 100 000 runs x 256 steps in the shape of BASELINE configs[2] (cfg3:
phase planes only) with all three side areas (K = 8 timer slots per run, four of them armed; limiter inputs; run control with a
story and a drain deadline), against what a batcher does without it: the three downloads (bf_resident_timers_download,
_sched_download, _runctl_download), a numpy compare of the raw rows, and the repairs of the drifted rows through
bf_resident_timers_arm, _sched_put and _runctl_put.  The host path compares bytes: it has no copy of the device's rules (terminal
steps, slots taken as fired), so it also lists and rewrites runs whose only difference is a slot at a terminal step, which the
device call leaves alone (the next fire prunes that slot).
Two twin batches hold the same areas; the caller's areas are a copy of them where 0 %, 0.1 % and 1 % of the runs drifted (one timer
deadline, one limiter input or one story deadline, in turn).  Each round restores both batches (untimed), then times, on alternate
batches in alternate order: the device call with BF_RESYNC_CHECK, the device call that repairs, and the host path; the two device
calls also take turns going first (between a repair and a check that follows it, an untimed device call back to the batch's own
areas undoes what the repair wrote).  Times are host
clocks around calls that end in a device synchronise: median and min-max over the rounds.

usage: python tools/resync_areas_probe.py [--runs N] [--rounds K] [--warmup W] [--out FILE]"""
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

S, K, ARMED = 256, 8, 4


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
    arms = np.zeros(n * ARMED, dtype=Frontier.TIMER_DTYPE)
    arms["run"] = np.repeat(np.arange(n), ARMED)
    arms["step"] = np.tile(np.arange(ARMED) * 50 + 20, n)
    arms["code"] = A.DEC_PENDING   # wake-only: the layout has no decision planes
    arms["deadline"] = 10_000 + rng.integers(0, 1000, n * ARMED)
    q = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
    q["run"], q["story_key"], q["queue_key"] = np.arange(n), np.arange(n) % 4, np.arange(n) % 3
    q["priority"], q["queued_since"], q["run_phase"] = np.arange(n) % 5, A.SCHED_NONE, A.PHASE_RUNNING
    c = np.zeros(n, dtype=Frontier.RUNCTL_PUT_DTYPE)
    c["run"], c["story_deadline"], c["drain_deadline"] = np.arange(n), 50_000 + np.arange(n) % 977, 90_000
    hs = [fr.resident_create(L, n) for _ in range(2)]
    for h in hs:
        fr.resident_upload(h, 0, base)
        fr.resident_timers(h, K)
        fr.resident_timers_arm(h, arms)
        fr.resident_sched(h)
        fr.resident_sched_put(h, q)
        fr.resident_runctl(h)
        fr.resident_runctl_put(h, c)
    own = (fr.resident_timers_download(hs[0], 0, n, K), fr.resident_sched_download(hs[0], 0, n),
           fr.resident_runctl_download(hs[0], 0, n))

    def device(h, areas, check):
        return fr.resident_resync_areas(h, n, timers=areas[0], sched=areas[1], runctl=areas[2], check=check,
                                        items_cap=max(n // 50, 1))

    def host(h, areas):
        """three downloads, a compare of the raw rows, the repairs through the put calls -> drifted runs"""
        t, s, r = (fr.resident_timers_download(h, 0, n, K), fr.resident_sched_download(h, 0, n),
                   fr.resident_runctl_download(h, 0, n))
        dt = np.nonzero((t.view(np.uint64) != areas[0].view(np.uint64)).any(axis=1))[0]
        ds = np.nonzero(s.view(np.uint8).reshape(n, -1).__ne__(areas[1].view(np.uint8).reshape(n, -1)).any(axis=1))[0]
        dr = np.nonzero(r.view(np.uint8).reshape(n, -1).__ne__(areas[2].view(np.uint8).reshape(n, -1)).any(axis=1))[0]
        req = []
        for run in dt:   # cancel the device's slots the caller lacks, arm the caller's
            want = {int(x["step"]): x for x in areas[0][run] if x["deadline"] != A.TIMER_NONE}
            for x in t[run]:
                if x["deadline"] != A.TIMER_NONE and int(x["step"]) not in want:
                    req.append((run, int(x["step"]), 0, 0, A.TIMER_NONE, 0))
            req += [(run, st, int(x["code"]), 0, int(x["deadline"]), 0) for st, x in want.items()]
        if req:
            fr.resident_timers_arm(h, np.array(req, dtype=Frontier.TIMER_DTYPE))
        if ds.size:
            fr.resident_sched_put(h, areas[1][ds])
        if dr.size:
            p = np.zeros(dr.size, dtype=Frontier.RUNCTL_PUT_DTYPE)
            p["run"] = dr
            for f in ("story_deadline", "drain_deadline", "stop"):
                p[f] = areas[2][f][dr]
            fr.resident_runctl_put(h, p)
        return np.union1d(np.union1d(dt, ds), dr).size

    lines = []
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    lines.append("resync_areas_probe: %d runs x %d steps (cfg3 shape), K = %d (%d armed), limiter inputs and run control, %d rounds; %s"
                 % (n, S, K, ARMED, a.rounds, gpu))
    fmt = lambda t: "median %8.1f us (%.1f - %.1f)" % (np.median(t) * 1e6, np.min(t) * 1e6, np.max(t) * 1e6)  # noqa: E731
    for share in (0.0, 0.001, 0.01):
        caller = tuple(x.copy() for x in own)
        k = int(round(share * n))
        for j, run in enumerate(rng.choice(n, size=k, replace=False)):
            if j % 3 == 0:
                caller[0]["deadline"][run, 0] += 7
            elif j % 3 == 1:
                caller[1]["priority"][run] += 1
            else:
                caller[2]["story_deadline"][run] += 11
        times = {"check": [], "repair": [], "host": []}
        found = {}
        for r in range(a.warmup + a.rounds):
            hd, hh = (hs[0], hs[1]) if r % 2 == 0 else (hs[1], hs[0])
            for h in hs:   # both batches back to their own areas, byte for byte (dormant slots too)
                host(h, own)
            order = [("device", hd), ("host", hh)] if r % 4 < 2 else [("host", hh), ("device", hd)]
            for kind, h in order:
                if kind == "device" and r % 4 in (0, 3):   # the device calls take turns going first (5 timed rounds each)
                    t1, out1 = timed(lambda: device(h, caller, True))
                    t2, out2 = timed(lambda: device(h, caller, False))
                elif kind == "device":
                    t2, out2 = timed(lambda: device(h, caller, False))
                    device(h, own, False)   # undoes exactly what the repair wrote, so the check follows a device call here too
                    t1, out1 = timed(lambda: device(h, caller, True))
                if kind == "device":
                    found["check"], found["repair"] = out1["n_drifted"], out2["n_written"]
                    if r >= a.warmup:
                        times["check"].append(t1)
                        times["repair"].append(t2)
                else:
                    t3, found["host"] = timed(lambda: host(h, caller))
                    if r >= a.warmup:
                        times["host"].append(t3)
        lines.append("%.1f %% of the runs drifted (%d):" % (share * 100, k))
        lines.append("  bf_resident_resync_areas, BF_RESYNC_CHECK:   %s; drifted %d" % (fmt(times["check"]), found["check"]))
        lines.append("  bf_resident_resync_areas, repair:            %s; written %d" % (fmt(times["repair"]), found["repair"]))
        lines.append("  3 downloads + numpy compare + put repairs:   %s; drifted %d" % (fmt(times["host"]), found["host"]))
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    fr.close()


if __name__ == "__main__":
    main()
