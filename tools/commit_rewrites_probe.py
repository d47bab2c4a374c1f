"""Per-tick cost of storing a pass's stage G / H / I rewrites: bf_resident_commit_rewrites against bf_resident_commit_journal.

Two resident batches start from the same 100 000 runs x 256 steps of random topologies with parallel steps (a child area), a
quarter of the steps gates with a timeout timing of 8 clock units (at most 64 per Story), a timer area of 64 slots per run and
random run flags (fail-fast, realtime, terminated topologies among them).  Each tick changes 1 % of the phase codes by deltas and
runs, on each batch, Fire(now) (timed-out gates are rewritten by stage G), a touched tick with the deltas, and then one commit:
  journal:   bf_resident_commit_journal(now) into pinned items and runs buffers
  rewrites:  bf_resident_commit_rewrites(now) into pinned items and runs buffers
The order of the two commits alternates tick by tick.  The batches diverge after the first commit (the rewriting one stores what
the other recomputes), so the items listed differ; both are reported.  Times are host clocks around calls that end in a device
synchronise.

usage: python tools/commit_rewrites_probe.py [--runs N] [--ticks K] [--warmup W] [--out FILE]"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200 import Frontier  # noqa: E402
from tests import randgen  # noqa: E402
from tests.test_host_commit import no_stops  # noqa: E402

S, K, DELAY = 256, 64, 8
NONE_D = np.zeros(0, Frontier.DELTA_DTYPE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--ticks", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    fr = Frontier(0)
    rng = np.random.default_rng(4)
    # no stop steps: a launched stop step needs a BF_COMMIT_PHASE entry, and the probe commits none
    ts = no_stops(randgen.random_topologies(rng, 16, S // 2, S, max_deg=4, parallel=True, fill=0.5))
    types = ts.step_flags & np.uint8(A.SF_TYPE_MASK)
    gate = (rng.random(ts.step_flags.shape[0]) < 0.25) & (types == A.STEP_ENGRAM)
    s0 = 0
    for i in range(ts.count):   # at most K gates per Story: every launched gate of a run fits its slots
        g = np.nonzero(gate[s0:s0 + int(ts.S[i])])[0]
        gate[s0 + g[K:]] = False
        s0 += int(ts.S[i])
    ts.step_flags[:] = np.where(gate, np.uint8(A.STEP_GATE) | (ts.step_flags & ~np.uint8(A.SF_TYPE_MASK)), ts.step_flags)
    slots = fr.put_topologies(ts)
    s0 = 0
    for i in range(ts.count):
        n_s = int(ts.S[i])
        fr.put_timings(int(slots[i]), [(s, A.DEC_TIMED_OUT, DELAY) for s in np.nonzero(gate[s0:s0 + n_s])[0]])
        s0 += n_s
    n = a.runs
    L, st, _ = randgen.random_state(rng, ts, slots, n, A.F_DECISION | A.F_ALL_OUT, phase_mix="progress")
    assert L.off_child != A.OFF_NONE
    hs = []
    for _ in range(2):
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, st)
        fr.resident_timers(h, K)
        fr.resident_tick_touched(h, n, NONE_D, n, 1 << 24)
        hs.append(h)
    cap = n * 64   # items: far above what a tick of this workload lists (n_items is checked against it below)
    bufs = [(fr.alloc_pinned(cap * 16), fr.alloc_pinned(n * 4)) for _ in range(2)]
    names = ("journal", "rewrites")
    times = {k: [] for k in names}
    items = {k: [] for k in names}
    rewritten = []

    def commit(form, h, now):
        out = A.CommitOut(struct_size=C.sizeof(A.CommitOut))
        arm = A.CommitArm(struct_size=C.sizeof(A.CommitArm), now=now)
        ib, rb = bufs[form]
        j = A.CommitJournal(struct_size=C.sizeof(A.CommitJournal), items=ib.ctypes.data, items_cap=cap, runs=rb.ctypes.data,
                            runs_cap=n)
        nrw = C.c_uint32(0)
        if form == 0:
            rc = fr._lib.bf_resident_commit_journal(fr._ctx, h, n, None, 0, C.byref(out), C.byref(arm), C.byref(j))
        else:
            rc = fr._lib.bf_resident_commit_rewrites(fr._ctx, h, n, None, 0, C.byref(out), C.byref(arm), C.byref(j), C.byref(nrw))
        assert rc == 0, fr._lib.bf_last_error(fr._ctx)
        assert j.n_items <= cap
        return int(j.n_items), int(nrw.value)

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
        for j in range(2):
            form = (tick + j) % 2
            t0 = time.perf_counter()
            m, nrw = commit(form, hs[form], now)
            t1 = time.perf_counter()
            if tick >= a.warmup:
                times[names[form]].append(t1 - t0)
                items[names[form]].append(m)
                if form == 1:
                    rewritten.append(nrw)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    q = lambda t: (np.median(t) * 1e6, np.percentile(t, 25) * 1e6, np.percentile(t, 75) * 1e6, np.min(t) * 1e6, np.max(t) * 1e6, len(t))  # noqa: E731
    lines = ["commit_rewrites_probe: %d runs x %d steps (parallel steps with a child area, a quarter of the engram steps gates "
             "with a timing), K = %d, 1 %% of codes changed per tick, %d ticks after %d warm-up, the two forms alternating"
             % (n, S, K, a.ticks, a.warmup), "gpu: %s" % gpu]
    for k, label in zip(names, ("bf_resident_commit_journal, pinned buffers", "bf_resident_commit_rewrites, pinned buffers")):
        lines.append("%-8s (%s): median %.1f us, p25 %.1f, p75 %.1f, range %.1f .. %.1f (%d ticks); items per tick median %d"
                     % ((k, label) + q(times[k]) + (np.median(items[k]),)))
    lines.append("steps rewritten per rewriting commit: median %d (min %d, max %d)" % (np.median(rewritten), min(rewritten), max(rewritten)))
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    for ib, rb in bufs:
        fr.free_pinned(ib)
        fr.free_pinned(rb)
    fr.close()


if __name__ == "__main__":
    main()
