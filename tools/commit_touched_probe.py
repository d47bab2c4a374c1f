"""Per-tick cost of a touched commit (bf_resident_commit_touched) against the full form it matches.

Two resident batches hold the same runs x 256 steps, a quarter of the steps gates with a timeout timing, and a timer area of 64
slots per run (the workload of tools/commit_journal_probe.py); batch B has the commit-due bits.  Each tick changes a phase code
in 1 % of the runs by deltas and runs, on both batches, Fire(now) and a touched tick with the deltas; then A commits with the
full form and B with the touched call of the same form, the order alternating tick by tick.  The forms are measured one after
the other (a form change makes the next touched commit full, which the warm-up ticks absorb):
  timed:     bf_resident_commit_timed(now)
  journal:   bf_resident_commit_journal(now) into pinned items and runs buffers
  rewrites:  bf_resident_commit_rewrites(now) into pinned items and runs buffers
Times are host clocks around calls that end in a device synchronise.  Every pair of commits must return the same outs and
journals, and the two batches' records and timer slots are compared after each form.

usage: python tools/commit_touched_probe.py [--runs N[,N...]] [--ticks K] [--warmup W] [--out FILE]"""
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
FORMS = ("timed", "journal", "rewrites")


def probe(fr, n, ticks, warmup, seed):
    rng = np.random.default_rng(seed)
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
    L, st, _ = randgen.random_state(rng, ts, slots, n, A.F_DECISION | A.F_ALL_OUT, phase_mix="progress")
    hs = []
    for _ in range(2):
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, st)
        fr.resident_timers(h, K)
        fr.resident_tick_touched(h, n, NONE_D, n, 1 << 24)
        hs.append(h)
    del st
    fr.resident_commit_marks(hs[1])
    cap = n * 64
    bufs = [(fr.alloc_pinned(cap * 16), fr.alloc_pinned(n * 4)) for _ in range(2)]
    res = {}
    tick_no = 0
    for form in FORMS:
        times = {"full": [], "touched": []}
        considered, full_ticks = [], 0

        def commit(b, now):
            out = A.CommitOut(struct_size=C.sizeof(A.CommitOut))
            arm = A.CommitArm(struct_size=C.sizeof(A.CommitArm), now=now)
            scope = A.CommitScope(struct_size=C.sizeof(A.CommitScope), flags=A.COMMIT_SCOPE_REWRITES if form == "rewrites" else 0)
            nrw = C.c_uint32(0)
            j = None
            if form != "timed":
                ip, rp = bufs[b]
                j = A.CommitJournal(struct_size=C.sizeof(A.CommitJournal), items=ip.ctypes.data, items_cap=cap, runs=rp.ctypes.data,
                                    runs_cap=n)
            t0 = time.perf_counter()
            if b == 1:
                rc = fr._lib.bf_resident_commit_touched(fr._ctx, hs[1], n, None, 0, C.byref(out), C.byref(arm),
                                                        None if j is None else C.byref(j), C.byref(nrw), C.byref(scope))
            elif form == "timed":
                rc = fr._lib.bf_resident_commit_timed(fr._ctx, hs[0], n, None, 0, C.byref(out), C.byref(arm))
            elif form == "journal":
                rc = fr._lib.bf_resident_commit_journal(fr._ctx, hs[0], n, None, 0, C.byref(out), C.byref(arm), C.byref(j))
            else:
                rc = fr._lib.bf_resident_commit_rewrites(fr._ctx, hs[0], n, None, 0, C.byref(out), C.byref(arm), C.byref(j),
                                                         C.byref(nrw))
            t1 = time.perf_counter()
            assert rc == 0, fr._lib.bf_last_error(fr._ctx)
            return t1 - t0, out, arm, j, nrw.value, scope

        for tick in range(warmup + ticks):
            now = 1000 + tick_no
            tick_no += 1
            k = max(n // 100, 1)
            d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
            d["run"] = rng.choice(n, size=k, replace=False)
            d["index"], d["field"] = rng.integers(0, S, k), A.DELTA_PHASE
            d["code"] = rng.choice([2, 3, 3, 3, 4, 13], k)
            for h in hs:
                fr.resident_fire(h, n, now, fired_cap=0)
                fr.resident_tick_touched(h, n, d, n, 1 << 24)
            got = {}
            for b in ((0, 1) if tick % 2 == 0 else (1, 0)):
                got[b] = commit(b, now)
            (ta, oa, aa, ja, ra, _), (tb, ob, ab, jb, rb, sc) = got[0], got[1]
            assert bytes(oa) == bytes(ob) and bytes(aa) == bytes(ab) and ra == rb
            if ja is not None:
                m = int(ja.n_items)
                assert (ja.n_items, ja.n_runs_listed) == (jb.n_items, jb.n_runs_listed) and m <= cap
                assert np.array_equal(bufs[0][0][:16 * m], bufs[1][0][:16 * m])
                assert np.array_equal(bufs[0][1][:4 * ja.n_runs_listed], bufs[1][1][:4 * ja.n_runs_listed])
            if tick >= warmup:
                times["full"].append(ta)
                times["touched"].append(tb)
                considered.append(sc.n_considered)
                full_ticks += sc.full
        a, b = (fr.resident_download(h, 0, n, L.state_stride) for h in hs)
        assert np.array_equal(a, b)
        del a, b
        ta, tb = (fr.resident_timers_download(h, 0, n, K) for h in hs)
        assert np.array_equal(ta, tb)
        del ta, tb
        res[form] = (times, int(np.median(considered)), full_ticks)
    for p in bufs:
        for x in p:
            fr.free_pinned(x)
    for h in hs:
        fr.resident_destroy(h)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", default="100000,1000000")
    ap.add_argument("--ticks", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    fr = Frontier(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    q = lambda t: (np.median(t) * 1e6, np.percentile(t, 25) * 1e6, np.percentile(t, 75) * 1e6, np.min(t) * 1e6,  # noqa: E731
                   np.max(t) * 1e6)
    lines = ["commit_touched_probe: runs x %d steps (a quarter gates, each with a timing), K = %d, a phase code changed in 1 %% of "
             "the runs per tick, %d ticks per form after %d warm-up, full form and touched form alternating on twin batches"
             % (S, K, a.ticks, a.warmup), "gpu: %s" % gpu]
    for n in (int(x) for x in a.runs.split(",")):
        res = probe(fr, n, a.ticks, a.warmup, 5 + n)
        for form, (times, cons, nfull) in res.items():
            for kind in ("full", "touched"):
                lines.append("%8d runs %-8s %-7s: median %7.1f us, p25 %7.1f, p75 %7.1f, range %7.1f .. %7.1f" %
                             ((n, form, kind) + q(times[kind])))
            lines.append("%8d runs %-8s runs considered by the touched form: median %d, full calls %d" % (n, form, cons, nfull))
        print("\n".join(lines[-9:]), flush=True)
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    fr.close()


if __name__ == "__main__":
    main()
