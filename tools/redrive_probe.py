"""tools/redrive_probe.py: what an operator redrive of live runs costs on the device (bf_resident_redrive) against the delta path a
batcher has without it (bf_topology_closure, then one coalesced delta per reset step field, child nibble, registered bit and
run-flags byte through bf_resident_apply from pinned memory).

A 100 000 x 256 resident batch holds runs of eight Stories (all three groups, `if` steps), with cond and decision planes; the
second leg adds parallel steps and a child area.  Per leg, 1 %, 10 % and 50 % of the runs are redriven from a random step of
their Story, and 10 % are redriven whole.  Each call is synchronous, so the host clock around it is its whole time; the batch is
re-uploaded (untimed) before each one.  The delta path is timed in its three parts: the closure call, building and coalescing
the deltas on the host (numpy, into pinned memory), and bf_resident_apply.  The records both paths leave are byte-compared.
Prints the card and its power limit, and per row the median of each time and the bytes each path sends to the device.

    python tools/redrive_probe.py [--runs 100000] [--reps 10]
    python tools/redrive_probe.py --bytes-only     (no GPU: the bytes, with the closures computed on the host)
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200.frontier import Frontier  # noqa: E402
from bobrapet_b200.records import layout_py, pack_state  # noqa: E402
from tests import redrive as RD  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def host_closure(packed_of_slot):
    def closure(slots, steps, words):
        return np.stack([RD.closure_mask(packed_of_slot[int(s)], int(t), words) for s, t in zip(slots, steps)])
    return closure


def batch(rng, L, packed, slots, n):
    """random records: codes of every field, registered bits and child nibbles of the runs' Stories, TopologyTerminated on half"""
    story = rng.integers(0, len(packed), n)
    W32 = L.words * 32
    phase = rng.integers(0, 15, size=(n, W32), dtype=np.uint8)
    cond = rng.integers(0, 4, size=(n, W32), dtype=np.uint8)
    dec = rng.integers(0, 4, size=(n, W32), dtype=np.uint8)
    for s, ps in enumerate(packed):
        for a in (phase, cond, dec):
            a[story == s, ps.S:] = 0
    child = rng.integers(0, 15, size=(n, max(L.child_nibbles, 1)), dtype=np.uint8) if L.off_child != A.OFF_NONE else None
    reg = np.zeros(n, np.uint64)
    for s, ps in enumerate(packed):
        if ps.par_steps:
            on = story == s
            reg[on] = rng.integers(0, 1 << len(ps.par_steps), size=int(on.sum()), dtype=np.uint64)
    flags = np.where(rng.random(n) < 0.5, A.RF_TOPOLOGY_TERMINATED, 0).astype(np.uint8) | A.RF_FAIL_FAST
    return story, flags, pack_state(L, np.asarray(slots, np.uint32)[story], flags, phase, cond, dec, child, reg)


def requests(rng, packed, slots, story, share, whole):
    n = story.shape[0]
    runs = np.sort(rng.choice(n, size=int(round(n * share)), replace=False))
    req = np.zeros(runs.size, Frontier.REDRIVE_DTYPE)
    req["run"], req["slot"] = runs, np.asarray(slots)[story[runs]]
    S = np.array([p.S for p in packed])[story[runs]]
    req["step"] = A.REDRIVE_ALL if whole else (rng.random(runs.size) * S).astype(np.uint32)
    return req


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=10, help="timed calls per row")
    ap.add_argument("--bytes-only", action="store_true")
    a = ap.parse_args()
    n = a.runs
    fr = None if a.bytes_only else Frontier(0)
    if fr:
        print("card: %s" % card())
    print("%-6s %-7s %7s %11s %11s %11s %11s %11s %12s %12s" % ("leg", "redrive", "runs", "redrive_us", "closure_us", "build_us",
                                                               "apply_us", "deltas", "redrive_B", "delta_B"))
    for leg, n_par in (("cond", 0), ("child", 10)):
        rng = np.random.default_rng(77 + n_par)
        gens = [RD.random_story(rng, "t%d-" % k, int(rng.integers(200, 257)), n_par) for k in range(8)]
        packed = [RD.packed_story(s) for s in gens]
        fields = A.F_COND | A.F_DECISION | (A.F_CHILD if n_par else 0)
        L = layout_py(max(p.S for p in packed), max(p.child_nibbles() for p in packed), fields)
        if fr:
            from tests import packing as P
            slots = [int(s) for s in fr.put_topologies(P.topology_set(packed))]
        else:
            slots = list(range(len(packed)))
        pos = {s: p for s, p in zip(slots, packed)}
        closure = fr.closure if fr else host_closure(pos)
        story, flags, state = batch(rng, L, packed, slots, n)
        hR = fr.resident_create(L, n) if fr else None
        hD = fr.resident_create(L, n) if fr else None
        for share, whole in ((0.01, False), (0.1, False), (0.5, False), (0.1, True)):
            req = requests(rng, packed, slots, story, share, whole)
            keys = len({(int(q["slot"]), int(q["step"])) for q in req if q["step"] != A.REDRIVE_ALL})
            deltas = RD.redrive_deltas(closure, L, pos, req, flags)
            rb = req.nbytes
            db = 8 * keys + 4 * L.words * keys + deltas.nbytes   # closure queries + masks back + deltas
            t_r, t_c, t_b, t_a = [], [], [], []
            if fr:
                pin = fr.alloc_pinned(max(deltas.nbytes, 8)).view(Frontier.DELTA_DTYPE)
                for rep in range(a.reps + 1):
                    fr.resident_upload(hR, 0, state)
                    t0 = time.perf_counter()
                    _, applied = fr.resident_redrive(hR, req)
                    t1 = time.perf_counter()
                    assert applied == req.shape[0]
                    fr.resident_upload(hD, 0, state)
                    named = req["step"] != A.REDRIVE_ALL
                    ks = sorted({(int(s), int(t)) for s, t in zip(req["slot"][named], req["step"][named])})
                    t2 = time.perf_counter()
                    masks = fr.closure([k[0] for k in ks], [k[1] for k in ks], L.words) if ks else None
                    t3 = time.perf_counter()
                    d = RD.redrive_deltas(lambda *_: masks, L, pos, req, flags)
                    pin[:d.shape[0]] = d
                    t4 = time.perf_counter()
                    fr.resident_apply(hD, pin[:d.shape[0]])
                    t5 = time.perf_counter()
                    if rep:
                        t_r.append((t1 - t0) * 1e6)
                        t_c.append((t3 - t2) * 1e6)
                        t_b.append((t4 - t3) * 1e6)
                        t_a.append((t5 - t4) * 1e6)
                assert np.array_equal(fr.resident_download(hR, 0, n, L.state_stride), fr.resident_download(hD, 0, n, L.state_stride))
                fr.free_pinned(pin.view(np.uint8))
            med = lambda t: "%11.1f" % np.median(t) if t else "%11s" % "-"
            print("%-6s %-7s %7d %s %s %s %s %11d %12d %12d" % (leg, "whole" if whole else "%g%%" % (share * 100), req.shape[0],
                                                               med(t_r), med(t_c), med(t_b), med(t_a), deltas.shape[0], rb, db))
        if fr:
            fr.resident_destroy(hR)
            fr.resident_destroy(hD)
    if fr:
        print("device records of both paths byte-identical")
        fr.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
