"""tools/retire_probe.py: what taking runs out of a live resident batch costs on the device (bf_resident_retire) against the path a
batcher has without it: re-pack the surviving runs on the host (numpy), bf_resident_create, upload them and the full touched tick
that follows (a new batch has no touched-tick bookkeeping).  And what the compaction buys: a full compact tick and a changed-only
tick over the un-compacted batch (every index, retired runs included) against the compacted one.

A 100 000 x 256 cfg3-shaped batch with phase planes only, its records held on the host as a batcher's mirror holds them.  Three
legs retire 1 %, 10 % and 50 % of the runs, scattered.  The device path is timed with the capacity kept and with it shrunk to
the surviving runs.  Each sample starts from a freshly uploaded batch that has had its first tick (untimed); each call is timed
on the host around calls that end in a synchronise, and each timed full or changed-only tick follows an untimed one of the same
kind over the same runs; medians of --reps samples.  The device records both paths leave are
byte-compared.  Prints the card and its power limit.

    python tools/retire_probe.py [--runs 100000] [--reps 10]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200 import synth  # noqa: E402
from bobrapet_b200.frontier import Frontier  # noqa: E402
from bobrapet_b200.records import make_layout  # noqa: E402
from tests import retire as RT  # noqa: E402

S = 256
NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
SHARES = (0.01, 0.10, 0.50)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(f, *args, **kw):
    t0 = time.perf_counter()
    out = f(*args, **kw)
    return (time.perf_counter() - t0) * 1e6, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=10, help="samples per leg")
    a = ap.parse_args()
    n = a.runs
    rng = np.random.default_rng(1)
    fr = Frontier(0)
    ts = synth.topologies(3, 0, n, S)
    slots = fr.put_topologies(ts)
    L = make_layout(S, 0, 0)
    host = synth.state(3, 0, n, L, slots, ts)   # the batcher's records
    cap_ev = 64 * n

    def source():
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, host)
        fr.resident_tick_touched(h, n, NONE, n, cap_ev)
        return h

    def full_tick(h, k):
        return timed(fr.resident_tick_compact, h, k, NONE, cap_ev)[0]

    def changed_tick(h, k):
        return timed(fr.resident_tick_compact, h, k, NONE, cap_ev, flags=A.EVAL_CHANGED_ONLY)[0]

    print("card: %s" % card())
    print("batch: %d runs x %d steps, cfg3, phase planes only; %d samples per leg, medians in us" % (n, S, a.reps))
    print("%-7s %7s %8s %9s %9s | %9s %9s %9s %9s %9s | %9s %9s %9s %9s" % (
        "retire", "moves", "keep_us", "shrink_us", "tick_us", "repack_us", "create_us", "upload_us", "fulltk_us", "host_sum",
        "full_n_us", "full_m_us", "chg_n_us", "chg_m_us"))
    all_same = True
    for share in SHARES:
        k = int(n * share)
        t = {x: [] for x in ("keep", "shrink", "tick", "repack", "create", "upload", "full", "full_n", "full_m", "chg_n", "chg_m")}
        n_moves = 0
        for _ in range(a.reps):
            runs = rng.choice(n, size=k, replace=False).astype(np.uint32)
            m = n - k
            # device path, capacity kept; then ticks over the un-compacted and the compacted batch
            h = source()
            full_tick(h, n)
            t["full_n"].append(full_tick(h, n))
            changed_tick(h, n)
            t["chg_n"].append(changed_tick(h, n))
            us, (_, mf, _) = timed(fr.resident_retire, h, n, runs)
            t["keep"].append(us)
            n_moves = mf.size
            t["tick"].append(timed(fr.resident_tick_touched, h, m, NONE, m, cap_ev)[0])   # lists the moved runs
            full_tick(h, m)
            t["full_m"].append(full_tick(h, m))
            changed_tick(h, m)
            t["chg_m"].append(changed_tick(h, m))
            # device path, capacity shrunk to the survivors
            g = source()
            t["shrink"].append(timed(fr.resident_retire, g, n, runs, m)[0])
            # host path
            t0 = time.perf_counter()
            rec = np.ascontiguousarray(host[RT.order(n, runs)])
            t1 = time.perf_counter()
            f = fr.resident_create(L, m)
            t2 = time.perf_counter()
            fr.resident_upload(f, 0, rec)
            t3 = time.perf_counter()
            us_full, o = timed(fr.resident_tick_touched, f, m, NONE, m, cap_ev)
            assert o["full"] == 1
            t["repack"].append((t1 - t0) * 1e6); t["create"].append((t2 - t1) * 1e6); t["upload"].append((t3 - t2) * 1e6)
            t["full"].append(us_full)
            want = fr.resident_download(f, 0, m, L.state_stride)
            all_same &= np.array_equal(fr.resident_download(h, 0, m, L.state_stride), want)
            all_same &= np.array_equal(fr.resident_download(g, 0, m, L.state_stride), want)
            for x in (h, g, f):
                fr.resident_destroy(x)
        md = {x: float(np.median(v)) for x, v in t.items()}
        host_sum = md["repack"] + md["create"] + md["upload"] + md["full"]
        print("%-7s %7d %8.1f %9.1f %9.1f | %9.1f %9.1f %9.1f %9.1f %9.1f | %9.1f %9.1f %9.1f %9.1f" % (
            "%g %%" % (share * 100), n_moves, md["keep"], md["shrink"], md["tick"], md["repack"], md["create"], md["upload"],
            md["full"], host_sum, md["full_n"], md["full_m"], md["chg_n"], md["chg_m"]))
    print("device records of both paths byte-identical" if all_same else "DEVICE RECORDS DIFFER")
    fr.close()
    return 0 if all_same else 1


if __name__ == "__main__":
    sys.exit(main())
