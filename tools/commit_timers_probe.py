"""Per-tick cost of arming the launched steps' timers in the tick commit against a commit followed by bf_resident_timers_arm.

Two resident batches hold the same 100 000 runs x 256 steps, a quarter of the steps gates (cfg4's 256-step runs carry condition or
gate codes on half their steps), at most 64 per Story so that no run overflows, each gate with a timeout timing of 8 clock
units, and a timer area of 64 slots per run.  Each tick changes 1 % of the phase codes by
deltas and runs, on each batch, Fire(now) and a touched tick with the deltas, and then:
  timed:   bf_resident_commit_timed(now)
  two:     bf_resident_commit + bf_resident_timers_arm of the slots the timed commit armed
The arm requests are the difference of the timed batch's slots across its commit, taken outside the timed sections, so the timed
form runs first in each tick and the two forms alternate tick by tick in one process; both batches hold the same records and
slots after every tick.  Times are host clocks around calls that end in a device synchronise.

usage: python tools/commit_timers_probe.py [--runs N] [--ticks K] [--warmup W] [--out FILE]"""
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

S, K, DELAY = 256, 64, 8
NONE_D = np.zeros(0, Frontier.DELTA_DTYPE)


def new_arms(before, after):
    """the slots of `after` that `before` does not hold, as bf_timer requests"""
    n = before.shape[0]
    key = lambda a: a["step"].astype(np.int64) | np.arange(n, dtype=np.int64)[:, None] << 16  # noqa: E731
    b, a = key(before)[before["deadline"] != A.TIMER_NONE], after["deadline"] != A.TIMER_NONE
    r, k = np.nonzero(a)
    fresh = ~np.isin(key(after)[r, k], b)
    r, k = r[fresh], k[fresh]
    req = np.zeros(r.size, dtype=Frontier.TIMER_DTYPE)
    req["run"], req["step"], req["code"], req["deadline"] = r, after["step"][r, k], after["code"][r, k], after["deadline"][r, k]
    return req


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--ticks", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    fr = Frontier(0)
    rng = np.random.default_rng(4)
    ts = randgen.random_topologies(rng, 16, S // 2, S, max_deg=4, parallel=False, fill=0.5)
    gate = rng.random(ts.step_flags.shape[0]) < 0.25
    s0 = 0
    for i in range(ts.count):   # at most K gates per Story: every launched gate of a run fits its slots
        g = np.nonzero(gate[s0:s0 + int(ts.S[i])])[0]
        gate[s0 + g[K:]] = False
        s0 += int(ts.S[i])
    ts.step_flags[:] = np.where(gate, A.STEP_GATE, A.STEP_ENGRAM).astype(np.uint8) | (ts.step_flags & ~np.uint8(A.SF_TYPE_MASK))
    slots = fr.put_topologies(ts)
    s0 = 0
    for i in range(ts.count):
        n_s = int(ts.S[i])
        fr.put_timings(int(slots[i]), [(s, A.DEC_TIMED_OUT, DELAY) for s in np.nonzero(gate[s0:s0 + n_s])[0]])
        s0 += n_s
    n = a.runs
    L, st, _ = randgen.random_state(rng, ts, slots, n, A.F_DECISION | A.F_ALL_OUT, phase_mix="progress")
    hs = []
    for _ in range(2):
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, st)
        fr.resident_timers(h, K)
        fr.resident_tick_touched(h, n, NONE_D, n, 1 << 24)
        hs.append(h)
    ht, h2 = hs
    t_timed, t_two, armed, written = [], [], [], []
    for tick in range(a.warmup + a.ticks):
        now = 1000 + tick
        k = n * S // 100
        d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"], d["field"] = rng.integers(0, n, k), rng.integers(0, S, k), A.DELTA_PHASE
        d["code"] = rng.choice([2, 3, 3, 3, 4, 13], k)
        _, first = np.unique(d["run"].astype(np.int64) * S + d["index"], return_index=True)
        d = d[first]   # at most one delta per (run, step)
        for h in hs:
            fr.resident_fire(h, n, now, fired_cap=0)
            fr.resident_tick_touched(h, n, d, n, 1 << 24)
        before = fr.resident_timers_download(ht, 0, n, K)
        t0 = time.perf_counter()
        c = fr.resident_commit(ht, n, now=now)
        t1 = time.perf_counter()
        req = new_arms(before, fr.resident_timers_download(ht, 0, n, K))
        t2 = time.perf_counter()
        fr.resident_commit(h2, n)
        fr.resident_timers_arm(h2, req)
        t3 = time.perf_counter()
        assert np.array_equal(fr.resident_download(ht, 0, n, L.state_stride), fr.resident_download(h2, 0, n, L.state_stride))
        assert np.array_equal(fr.resident_timers_download(ht, 0, n, K), fr.resident_timers_download(h2, 0, n, K))
        if tick >= a.warmup:
            t_timed.append(t1 - t0)
            t_two.append(t3 - t2)
            armed.append(c["n_armed"])
            written.append(c["n_runs_written"])
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    q = lambda t: (np.median(t) * 1e6, np.percentile(t, 25) * 1e6, np.percentile(t, 75) * 1e6, np.min(t) * 1e6)  # noqa: E731
    lines = ["commit_timers_probe: %d runs x %d steps (a quarter gates, each with a timing), K = %d, 1 %% of codes changed per tick, "
             "%d ticks after %d warm-up" % (n, S, K, a.ticks, a.warmup),
             "gpu: %s" % gpu,
             "timed (bf_resident_commit_timed):                   median %.1f us, p25 %.1f, p75 %.1f, min %.1f (%d ticks)" % (q(t_timed) + (len(t_timed),)),
             "two   (bf_resident_commit + bf_resident_timers_arm): median %.1f us, p25 %.1f, p75 %.1f, min %.1f (%d ticks)" % (q(t_two) + (len(t_two),)),
             "slots armed per tick: median %d; runs written per commit: median %d" % (np.median(armed), np.median(written))]
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    fr.close()


if __name__ == "__main__":
    main()
