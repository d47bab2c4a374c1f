"""tools/migrate_probe.py: what moving the live runs of an edited Story to its new generation costs on the device
(bf_resident_migrate) against the host alternatives, as the share of the batch's runs on the edited Story grows.

A 100 000 x 256 resident batch (phase planes only) holds runs of eight Stories; a share of them (1 %, 10 %, 50 %) runs on Story 0,
scattered through the batch.  Story 0 is edited (steps removed, renamed, inserted, moved between groups, reordered) and its
new generation put.  Then, per share:
  migrate      bf_resident_migrate of the runs on the old slot (one launch, one synchronise);
  repack       the host re-pack of the same runs' records (numpy gather of the phase codes through the step map);
  per-run      repack + one bf_resident_upload per run (the runs are not contiguous);
  whole        repack + one bf_resident_upload of the whole batch.
Each call is synchronous, so the host clock around it is its whole time; the batch is re-uploaded (untimed) before each
migration.  The records the three paths leave on the device are byte-compared.  Prints the card and its power limit, and per
share the median of each.

    python tools/migrate_probe.py [--runs 100000] [--reps 10]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bobrapet_b200 import _abi as A  # noqa: E402
from bobrapet_b200 import Frontier  # noqa: E402
from bobrapet_b200.records import make_layout, pack_state  # noqa: E402
from tests import migration as M  # noqa: E402
from tests import packing as P  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=10, help="timed migrations per share")
    ap.add_argument("--per-run-reps", type=int, default=2, help="timed per-run upload passes per share")
    a = ap.parse_args()
    n = a.runs
    fr = Frontier(0)
    print("card: %s" % card())
    rng = np.random.default_rng(2024)
    gens = [M.random_story(rng, "t%d-" % k, 240, 0) for k in range(8)]
    gens.append(M.edit_story(rng, gens[0], "t0-e", parallel=False))
    packed = [M.story_from_steps(s) for s in gens]
    slots = fr.put_topologies(P.topology_set(packed))
    S = max(p.S for p in packed)
    L = make_layout(S, 0, 0)
    smap, _ = M.migration_map(packed[0], packed[8])
    inv = np.full(L.words * 32, A.MIGRATE_GONE, np.int64)
    keep = smap != A.MIGRATE_GONE
    inv[smap[keep].astype(np.int64)] = np.nonzero(keep)[0]
    hM, hU = fr.resident_create(L, n), fr.resident_create(L, n)
    print("%6s %8s %12s %12s %14s %12s" % ("share", "runs", "migrate_us", "repack_us", "per_run_ms", "whole_ms"))
    for share in (0.01, 0.1, 0.5):
        k = int(round(n * share))
        on = np.sort(rng.choice(n, size=k, replace=False))
        story = rng.integers(1, 8, n)
        story[on] = 0
        codes = rng.integers(0, 15, size=(n, L.words * 32), dtype=np.uint8)
        for s in range(8):
            codes[story == s, packed[s].S:] = 0
        flags = np.ones(n, np.uint8)
        state = pack_state(L, slots[story].astype(np.uint32), flags, codes)
        tm, tr, tp, tw = [], [], [], []
        want = None
        for rep in range(a.reps + 1):
            fr.resident_upload(hM, 0, state)
            t0 = time.perf_counter()
            got = fr.resident_migrate(hM, int(slots[0]), int(slots[8]), smap, n)
            dt = time.perf_counter() - t0
            assert got == k
            t0 = time.perf_counter()
            moved = codes[on][:, np.minimum(inv, codes.shape[1] - 1)] * (inv != A.MIGRATE_GONE)
            recs = pack_state(L, np.full(k, slots[8], np.uint32), flags[on], moved.astype(np.uint8))
            dr = time.perf_counter() - t0
            if rep:
                tm.append(dt * 1e6)
                tr.append(dr * 1e6)
            want = state.copy()
            want[on] = recs
        for rep in range(a.per_run_reps):
            fr.resident_upload(hU, 0, state)
            t0 = time.perf_counter()
            moved = codes[on][:, np.minimum(inv, codes.shape[1] - 1)] * (inv != A.MIGRATE_GONE)
            recs = pack_state(L, np.full(k, slots[8], np.uint32), flags[on], moved.astype(np.uint8))
            for i, r in enumerate(on):
                fr.resident_upload(hU, int(r), recs[i:i + 1])
            tp.append((time.perf_counter() - t0) * 1e3)
        assert np.array_equal(fr.resident_download(hU, 0, n, L.state_stride), want)
        for rep in range(3):
            t0 = time.perf_counter()
            moved = codes[on][:, np.minimum(inv, codes.shape[1] - 1)] * (inv != A.MIGRATE_GONE)
            full = state.copy()
            full[on] = pack_state(L, np.full(k, slots[8], np.uint32), flags[on], moved.astype(np.uint8))
            fr.resident_upload(hU, 0, full)
            tw.append((time.perf_counter() - t0) * 1e3)
        dev = fr.resident_download(hM, 0, n, L.state_stride)
        assert np.array_equal(dev, want) and np.array_equal(fr.resident_download(hU, 0, n, L.state_stride), want)
        print("%5.0f%% %8d %12.1f %12.1f %14.1f %12.1f" % (share * 100, k, np.median(tm), np.median(tr), np.median(tp), np.median(tw)))
    print("device records of the three paths byte-identical")
    fr.resident_destroy(hM)
    fr.resident_destroy(hU)
    fr.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
