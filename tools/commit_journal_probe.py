"""Per-tick cost of listing a tick commit's writes: bf_resident_commit_journal against bf_resident_commit_timed.

Three resident batches hold the same 100 000 runs x 256 steps, a quarter of the steps gates with a timeout timing of 8 clock
units (at most 64 per Story, so that no run overflows), and a timer area of 64 slots per run: the workload of
tools/commit_timers_probe.py.  Each tick changes 1 % of the phase codes by deltas and runs, on each batch, Fire(now) and a touched
tick with the deltas, and then one commit per batch:
  timed:     bf_resident_commit_timed(now)
  pinned:    bf_resident_commit_journal(now) into items and runs buffers in pinned memory (written in place)
  pageable:  bf_resident_commit_journal(now) into numpy buffers (staged in the device scratch and copied back)
The journal buffers are allocated once, sized to what the workload's commits can list.  The order of the three commits rotates
tick by tick, and the three batches hold the same records and timer slots after every tick.  Times are host clocks around calls
that end in a device synchronise.

usage: python tools/commit_journal_probe.py [--runs N] [--ticks K] [--warmup W] [--out FILE]"""
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
    for _ in range(3):
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, st)
        fr.resident_timers(h, K)
        fr.resident_tick_touched(h, n, NONE_D, n, 1 << 24)
        hs.append(h)
    cap = n * 64   # items: far above what a tick of this workload lists (n_items is checked against it below)
    pin_items, pin_runs = fr.alloc_pinned(cap * 16), fr.alloc_pinned(n * 4)
    page_items, page_runs = np.zeros(cap, Frontier.COMMIT_WRITE_DTYPE), np.zeros(n, np.uint32)
    bufs = {1: (pin_items.ctypes.data, pin_runs.ctypes.data), 2: (page_items.ctypes.data, page_runs.ctypes.data)}
    names = ("timed", "pinned", "pageable")
    times = {k: [] for k in names}
    items_per_tick, written = [], []

    def commit(form, h, now):
        out = A.CommitOut(struct_size=C.sizeof(A.CommitOut))
        arm = A.CommitArm(struct_size=C.sizeof(A.CommitArm), now=now)
        if form == 0:
            rc = fr._lib.bf_resident_commit_timed(fr._ctx, h, n, None, 0, C.byref(out), C.byref(arm))
            j = None
        else:
            ip, rp = bufs[form]
            j = A.CommitJournal(struct_size=C.sizeof(A.CommitJournal), items=ip, items_cap=cap, runs=rp, runs_cap=n)
            rc = fr._lib.bf_resident_commit_journal(fr._ctx, h, n, None, 0, C.byref(out), C.byref(arm), C.byref(j))
        assert rc == 0, fr._lib.bf_last_error(fr._ctx)
        return out, j

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
        got = {}
        for j in range(3):
            form = (tick + j) % 3
            t0 = time.perf_counter()
            got[form] = commit(form, hs[form], now)
            t1 = time.perf_counter()
            if tick >= a.warmup:
                times[names[form]].append(t1 - t0)
        o0, (o1, j1), (o2, j2) = got[0][0], got[1], got[2]
        assert bytes(o0) == bytes(o1) == bytes(o2) and j1.n_items == j2.n_items <= cap and j1.n_runs_listed == o0.n_runs_written
        m = int(j1.n_items)
        assert np.array_equal(pin_items.view(Frontier.COMMIT_WRITE_DTYPE)[:m], page_items[:m])
        ref = fr.resident_download(hs[0], 0, n, L.state_stride)
        for h in hs[1:]:
            assert np.array_equal(ref, fr.resident_download(h, 0, n, L.state_stride))
        if tick >= a.warmup:
            items_per_tick.append(m)
            written.append(o0.n_runs_written)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    q = lambda t: (np.median(t) * 1e6, np.percentile(t, 25) * 1e6, np.percentile(t, 75) * 1e6, np.min(t) * 1e6, np.max(t) * 1e6,  # noqa: E731
                   len(t))
    lines = ["commit_journal_probe: %d runs x %d steps (a quarter gates, each with a timing), K = %d, 1 %% of codes changed per tick, "
             "%d ticks after %d warm-up, the three forms rotating" % (n, S, K, a.ticks, a.warmup),
             "gpu: %s" % gpu]
    for k, label in zip(names, ("bf_resident_commit_timed", "bf_resident_commit_journal, pinned buffers",
                                "bf_resident_commit_journal, pageable buffers")):
        lines.append("%-8s (%s): median %.1f us, p25 %.1f, p75 %.1f, range %.1f .. %.1f (%d ticks)" % ((k, label) + q(times[k])))
    lines.append("items per tick: median %d; runs written per commit: median %d" % (np.median(items_per_tick), np.median(written)))
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    fr.free_pinned(pin_items)
    fr.free_pinned(pin_runs)
    fr.close()


if __name__ == "__main__":
    main()
