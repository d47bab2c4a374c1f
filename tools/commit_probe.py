"""Per-tick cost of committing a tick's decisions on the device against echoing them back as deltas.

Two resident batches hold the same 100 000 runs x 256 steps with limiter inputs.  Each tick changes 1 % of the phase codes by
deltas (the StepRun events of a tick) and then, on each batch:
  commit: touched tick (with the deltas) + bf_resident_schedule + bf_resident_commit
  echo:   touched tick (with the deltas) + bf_resident_schedule + bf_resident_apply of the deltas the commit's writes amount to
The echo deltas are the difference of the commit batch's records across its commit, computed outside the timed sections; both
batches hold the same records after every tick.  Times are host clocks around calls that end in a device synchronise.

usage: python tools/commit_probe.py [--runs N] [--ticks K] [--warmup W] [--out FILE]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200 import Frontier  # noqa: E402
from bobrapet_b200.records import _unpack_planes  # noqa: E402
from tests import randgen  # noqa: E402

S = 256
TABLES = dict(story_limit=[50, 80, 1000, 20], queue_limit=[400, 100000, 700], queue_aging_s=[0, 60, 10], global_limit=200_000)


def codes(L, st):
    return _unpack_planes(st[:, L.off_phase:L.off_phase + 16 * L.words], L.words, 4, S)


def echo_deltas(L, before, after):
    cb, ca = codes(L, before), codes(L, after)
    r, s = np.nonzero(cb != ca)
    d = np.zeros(r.size, dtype=Frontier.DELTA_DTYPE)
    d["run"], d["index"], d["field"], d["code"] = r, s, A.DELTA_PHASE, ca[r, s]
    rb, ra = before[:, 8:16].copy().view("<u8")[:, 0], after[:, 8:16].copy().view("<u8")[:, 0]
    regs = []
    for run in np.nonzero(rb != ra)[0]:
        new = int(ra[run]) & ~int(rb[run])
        regs += [(int(run), q, A.DELTA_REGISTERED, 1) for q in range(64) if (new >> q) & 1]
    return np.concatenate([d, np.array(regs, dtype=Frontier.DELTA_DTYPE)]) if regs else d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--ticks", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    fr = Frontier(0)
    rng = np.random.default_rng(1)
    ts = randgen.random_topologies(rng, 16, S // 2, S, max_deg=4, parallel=False, fill=0.5)
    ts.step_flags[(ts.step_flags & A.SF_TYPE_MASK) == A.STEP_STOP] &= ~np.uint8(A.SF_TYPE_MASK)   # no stop entries needed
    slots = fr.put_topologies(ts)
    n = a.runs
    L, st, _ = randgen.random_state(rng, ts, slots, n, A.F_DECISION | A.F_ALL_OUT, phase_mix="progress")
    q = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
    q["run"] = np.arange(n)
    q["story_key"], q["queue_key"], q["priority"] = rng.integers(0, 4, n), rng.integers(0, 3, n), rng.integers(0, 5, n)
    q["queued_since"], q["run_phase"] = A.SCHED_NONE, A.PHASE_RUNNING
    hs = []
    for _ in range(2):
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, st)
        fr.resident_sched(h)
        fr.resident_sched_put(h, q)
        fr.resident_tick_touched(h, n, np.zeros(0, Frontier.DELTA_DTYPE), n, 1 << 24)
        hs.append(h)
    hc, he = hs
    part = lambda h: [dict(handle=h, n_runs=n, runs_cap=n, events_cap=1 << 24)]  # noqa: E731
    t_commit, t_echo, n_echo, n_written = [], [], [], []
    for tick in range(a.warmup + a.ticks):
        k = n * S // 100
        d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"], d["field"] = rng.integers(0, n, k), rng.integers(0, S, k), A.DELTA_PHASE
        d["code"] = rng.choice([2, 3, 3, 3, 4, 13], k)
        _, first = np.unique(d["run"].astype(np.int64) * S + d["index"], return_index=True)
        d = d[first]   # at most one delta per (run, step)
        t0 = time.perf_counter()
        fr.resident_tick_touched(hc, n, d, n, 1 << 24)
        fr.resident_schedule(part(hc), TABLES, 100 + tick)
        t1 = time.perf_counter()
        before = fr.resident_download(hc, 0, n, L.state_stride)
        t2 = time.perf_counter()
        c = fr.resident_commit(hc, n)
        t3 = time.perf_counter()
        after = fr.resident_download(hc, 0, n, L.state_stride)
        echo = echo_deltas(L, before, after)
        t4 = time.perf_counter()
        fr.resident_tick_touched(he, n, d, n, 1 << 24)
        fr.resident_schedule(part(he), TABLES, 100 + tick)
        fr.resident_apply(he, echo)
        t5 = time.perf_counter()
        assert np.array_equal(fr.resident_download(he, 0, n, L.state_stride), after), "the echo batch differs"
        if tick >= a.warmup:
            t_commit.append((t1 - t0) + (t3 - t2))
            t_echo.append(t5 - t4)
            n_echo.append(echo.shape[0])
            n_written.append(c["n_runs_written"])
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    lines = ["commit_probe: %d runs x %d steps, 1 %% of codes changed per tick, %d ticks after %d warm-up" % (n, S, a.ticks, a.warmup),
             "gpu: %s" % gpu,
             "commit (touched tick + schedule + commit): median %.1f us, min %.1f us" % (np.median(t_commit) * 1e6, np.min(t_commit) * 1e6),
             "echo   (touched tick + schedule + apply):  median %.1f us, min %.1f us" % (np.median(t_echo) * 1e6, np.min(t_echo) * 1e6),
             "echo deltas per tick: median %d; runs written per commit: median %d" % (np.median(n_echo), np.median(n_written))]
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    fr.close()


if __name__ == "__main__":
    main()
