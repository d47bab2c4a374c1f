"""tools/reshape_probe.py: what growing a live resident batch costs on the device (bf_resident_reshape) against the path a batcher
has without it: re-pack every run at the new layout on the host (numpy), bf_resident_create, upload the whole batch, and the full
touched tick that follows (a new batch has no touched-tick bookkeeping).

A 100 000 x 256 cfg3-shaped batch with phase planes only, its records held on the host as a batcher's mirror holds them.  Four
reshapes: capacity x 2 only; + cond and decision planes; steps_max 256 -> 288; + a child area.  Each sample starts from a freshly
uploaded source batch that has had its first tick (untimed); each leg is timed on the host around calls that end in a
synchronise; medians of --reps samples.  Also reported: the first touched tick after each path with 1 % of the runs touched by
phase deltas (after the host path that is the tick following its full one).  The device records both paths leave are
byte-compared.  Prints the card and its power limit.

    python tools/reshape_probe.py [--runs 100000] [--reps 10]
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
from tests import reshape as RS  # noqa: E402

S = 256
NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
LEGS = [("cap x2", S, 0, 0, 2), ("+cond+dec", S, 0, A.F_COND | A.F_DECISION, 1), ("steps 288", 288, 0, 0, 1),
        ("+child", S, 64, A.F_CHILD, 1)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def touch(rng, L, n, share):
    """one phase delta on each of share * n runs"""
    k = max(1, int(n * share))
    d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
    d["run"] = np.sort(rng.choice(n, size=k, replace=False))
    d["index"], d["field"], d["code"] = rng.integers(0, S, size=k), A.DELTA_PHASE, 3
    return d


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
    Lo = make_layout(S, 0, 0)
    host = synth.state(3, 0, n, Lo, slots, ts)   # the batcher's records
    cap_ev = 64 * n

    def source():
        h = fr.resident_create(Lo, n)
        fr.resident_upload(h, 0, host)
        fr.resident_tick_touched(h, n, NONE, n, cap_ev)
        return h

    def tick(h, d):
        t0 = time.perf_counter()
        o = fr.resident_tick_touched(h, n, d, n, cap_ev)
        return (time.perf_counter() - t0) * 1e6, o

    print("card: %s" % card())
    print("batch: %d runs x %d steps, cfg3, phase planes only; %d samples per leg, medians in us" % (n, S, a.reps))
    print("%-10s %9s %9s | %9s %9s %9s %9s %9s | %9s %9s" % ("reshape", "dev_us", "tick1%_us", "repack_us", "create_us", "upload_us",
                                                            "fulltk_us", "host_sum", "tick1%_us", "upload_MB"))
    all_same = True
    for name, steps, child, add, mult in LEGS:
        Ln = make_layout(steps, child, Lo.fields | add)
        cap = n * mult
        t = {k: [] for k in ("dev", "dtick", "repack", "create", "upload", "full", "htick")}
        for _ in range(a.reps):
            d = touch(rng, Ln, n, 0.01)
            # device path
            h = source()
            t0 = time.perf_counter()
            fr.resident_reshape(h, Ln, cap)
            t["dev"].append((time.perf_counter() - t0) * 1e6)
            us, o = tick(h, d)
            assert o["full"] == int(bool(add & A.F_DECISION))   # added decision planes make the next touched tick a full one
            t["dtick"].append(us)
            # host path
            t0 = time.perf_counter()
            rec = RS.reshape_state(Lo, Ln, host, cap)
            t1 = time.perf_counter()
            g = fr.resident_create(Ln, cap)
            t2 = time.perf_counter()
            fr.resident_upload(g, 0, rec)
            t3 = time.perf_counter()
            us_full, o = tick(g, NONE)
            assert o["full"] == 1
            us, o = tick(g, d)
            t["repack"].append((t1 - t0) * 1e6); t["create"].append((t2 - t1) * 1e6); t["upload"].append((t3 - t2) * 1e6)
            t["full"].append(us_full); t["htick"].append(us)
            same = np.array_equal(fr.resident_download(h, 0, cap, Ln.state_stride), fr.resident_download(g, 0, cap, Ln.state_stride))
            all_same &= same
            fr.resident_destroy(h)
            fr.resident_destroy(g)
        m = {k: float(np.median(v)) for k, v in t.items()}
        host_sum = m["repack"] + m["create"] + m["upload"] + m["full"]
        print("%-10s %9.1f %9.1f | %9.1f %9.1f %9.1f %9.1f %9.1f | %9.1f %9.1f" % (
            name, m["dev"], m["dtick"], m["repack"], m["create"], m["upload"], m["full"], host_sum, m["htick"],
            cap * Ln.state_stride / 1e6))
    print("device records of both paths byte-identical" if all_same else "DEVICE RECORDS DIFFER")
    fr.close()
    return 0 if all_same else 1


if __name__ == "__main__":
    sys.exit(main())
