"""tools/ctx_span_probe.py: what spanning resident batches over several ctxs costs on one H100, with two ctxs on device 0.

  - schedule: a 100 000-run batch at steps_max 256 and a 20 000-run batch at steps_max 1024 (random Stories of 200 to 256 and 600
    to 1000 steps, limiter inputs on every run), held in one ctx (A) and spread over two ctxs, one batch each (B).  Each tick
    changes 1 % of the runs of each batch (a phase delta of step 0), ticks every batch touched, then times one schedule:
    bf_resident_schedule over both batches of A, bf_resident_schedule_ctxs over both of B, alternated in one loop.  Host clock
    around the calls (they end in a synchronise); median, p25 and p75 of --ticks samples after --warmup.  Both schedules' lists
    and totals are compared.
  - transfer: k = 1 000 and 10 000 random runs moved from the 256-step batch into a 1024-step batch, in one ctx
    (bf_resident_transfer) and between two ctxs (bf_resident_transfer_ctx), alternated, medians of --reps samples.  Both
    destinations' state records are compared at the end.
Peer copies between two devices and spans over more than one GPU are not measured here (one GPU).  Prints the card and its
power limit.

    python tools/ctx_span_probe.py [--ticks 30] [--warmup 5] [--reps 5]
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200.frontier import Frontier, resident_schedule_ctxs  # noqa: E402
from bobrapet_b200.records import make_layout  # noqa: E402
from tests import randgen  # noqa: E402
from tests import reshape as RS  # noqa: E402
from tools.narrow_probe import card  # noqa: E402

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
N_STORIES, N_QUEUES = 128, 4


def pct(xs):
    return np.percentile(np.asarray(xs) * 1e6, [50, 25, 75])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    rng = np.random.default_rng(5)
    ts = [randgen.random_topologies(rng, 64, 200, 256, max_deg=4, parallel=False, fill=0.5),
          randgen.random_topologies(rng, 64, 600, 1000, max_deg=4, parallel=False, fill=0.5)]
    sizes, widths = (100_000, 20_000), (256, 1024)
    fa, fb = Frontier(0), [Frontier(0), Frontier(0)]
    for fr in [fa] + fb:   # the same Stories in the same order everywhere: the slot map is the identity
        slots = [fr.put_topologies(t) for t in ts]
    layouts, states = [], []
    for t, s, n, w in zip(ts, slots, sizes, widths):
        L0, st0, _ = randgen.random_state(rng, t, s, n, 0, phase_mix="progress", run_flag_mix=False)
        L = make_layout(w, 0, 0)
        layouts.append(L)
        states.append(RS.reshape_state(L0, L, st0, n))
    tables = {"story_limit": rng.integers(0, 400, N_STORIES).astype(np.int32),
              "queue_limit": np.array([0, 5000, 20000, 900], np.int32), "queue_aging_s": np.array([0, 30, 60, 5], np.int32),
              "global_limit": 60000}
    ha, hb = [], []
    for b, (L, st, n) in enumerate(zip(layouts, states, sizes)):
        q = np.zeros(n, Frontier.SCHED_PUT_DTYPE)
        q["run"] = np.arange(n)
        q["story_key"] = rng.integers(0, N_STORIES, n)
        q["queue_key"] = rng.integers(0, N_QUEUES, n)
        q["priority"] = rng.integers(0, 8, n)
        q["queued_since"] = A.TIMER_NONE
        q["run_phase"] = 2
        for fr, hs in ((fa, ha), (fb[b], hb)):
            h = fr.resident_create(L, n)
            fr.resident_upload(h, 0, st)
            fr.resident_sched(h)
            fr.resident_sched_put(h, q)
            hs.append(h)
    print("card: %s" % card())
    print("schedule: batches of %d x 256 and %d x 1024 steps, 1 %% of runs changed per tick; A: one ctx, B: two ctxs on device 0"
          % sizes)

    def tick(deltas):
        for b in range(2):
            for fr, h in ((fa, ha[b]), (fb[b], hb[b])):
                fr.resident_tick_touched(h, sizes[b], deltas[b], sizes[b], sizes[b] * 64)

    def deltas():
        out = []
        for n in sizes:
            k = n // 100
            d = np.zeros(k, Frontier.DELTA_DTYPE)
            d["run"] = rng.choice(n, size=k, replace=False)
            d["index"] = 0
            d["field"] = A.DELTA_PHASE
            d["code"] = rng.choice([2, 3, 0], size=k)
            out.append(d)
        return out

    parts_a = [{"handle": ha[b], "n_runs": sizes[b]} for b in range(2)]
    parts_b = [(fb[b], {"handle": hb[b], "n_runs": sizes[b]}) for b in range(2)]
    ta, tb = [], []
    same = True
    for i in range(a.warmup + a.ticks):
        tick(deltas())
        now = 1000 + i
        t0 = time.perf_counter()
        ra = fa.resident_schedule(parts_a, tables, now)
        t1 = time.perf_counter()
        rb = resident_schedule_ctxs(parts_b, tables, now)
        t2 = time.perf_counter()
        same &= all(pa["n_listed"] == pb["n_listed"] and pa["runs"].tobytes() == pb["runs"].tobytes() and
                    pa["events"].tobytes() == pb["events"].tobytes() for pa, pb in zip(ra["parts"], rb["parts"]))
        same &= ra["story_running"].tobytes() == rb["story_running"].tobytes() and ra["global_running"] == rb["global_running"]
        if i >= a.warmup:
            ta.append(t1 - t0)
            tb.append(t2 - t1)
    listed = sum(p["n_listed"] for p in ra["parts"])
    print("form               median_us   p25_us   p75_us   (last tick: %d runs listed)" % listed)
    for name, xs in (("one ctx", ta), ("two ctxs (span)", tb)):
        m, p25, p75 = pct(xs)
        print("%-17s %10.1f %8.1f %8.1f" % (name, m, p25, p75))
    print("span / one ctx: %.2fx (medians)" % (np.median(tb) / np.median(ta)))
    print("schedules of both forms identical: %s" % same)

    # transfers: a fresh 256-step source and a 1024-step destination in A, and in B one in each ctx
    n = sizes[0]
    Ld = make_layout(1024, 0, 0)
    kmax = 10_000
    cap = kmax * (a.reps + 1) + 1000 * (a.reps + 1)
    src_a, dst_a = fa.resident_create(layouts[0], n), fa.resident_create(Ld, cap)
    src_b, dst_b = fb[0].resident_create(layouts[0], n), fb[1].resident_create(Ld, cap)
    for fr, h in ((fa, src_a), (fb[0], src_b)):
        fr.resident_upload(h, 0, states[0])
        fr.resident_tick_touched(h, n, NONE, n, n * 64)
    smap = np.arange(ts[0].count, dtype=np.uint32)   # the slots of the 256-step Stories, which the moved runs hold
    na = nb = n
    da = db = 0
    print("transfer: runs of the %d x 256 batch into a 1024-step batch; medians of %d in us" % (n, a.reps))
    print("runs     in_ctx_us  cross_ctx_us   ratio")
    for k in (1000, kmax):
        xa, xb = [], []
        for _ in range(a.reps + 1):   # the first of each size warms it up
            runs = rng.choice(min(na, nb), size=k, replace=False).astype(np.uint32)
            t0 = time.perf_counter()
            fa.resident_transfer(src_a, dst_a, na, da, runs)
            t1 = time.perf_counter()
            fb[0].resident_transfer_ctx(fb[1], src_b, dst_b, nb, db, runs, smap)
            t2 = time.perf_counter()
            na -= k; nb -= k; da += k; db += k
            xa.append(t1 - t0)
            xb.append(t2 - t1)
        ma, mb = np.median(xa[1:]) * 1e6, np.median(xb[1:]) * 1e6
        print("%-8d %9.1f %13.1f %6.2fx" % (k, ma, mb, mb / ma))
    ra = fa.resident_download(dst_a, 0, da, Ld.state_stride)
    rb = fb[1].resident_download(dst_b, 0, db, Ld.state_stride)
    print("destinations of both transfer forms identical: %s" % (ra.tobytes() == rb.tobytes()))
    for fr in [fa] + fb:
        fr.close()


if __name__ == "__main__":
    main()
