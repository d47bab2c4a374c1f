#!/bin/bash
# tools/sanitize_resync_areas.sh: compute-sanitizer (memcheck, racecheck, synccheck) over bf_resident_resync_areas — its count and
# list launches and cta_scan<2> over a run list and over every run, a check and a repair of every area (re-armed slots, inputs,
# deadlines, a stop), pinned and pageable outputs with caps below the totals, K = 1 and K = 64, and a refusal.  Prints the tools'
# summaries.
cd "$(dirname "$0")/.."
cat > /tmp/san_resync_areas.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np
from bobrapet_b200 import _abi as A, Frontier
from tests import resync_areas as M
from tests.lifecycle import RUNCTL, SCHED, TIMERS
from tests.test_gpu_resync_areas import FIRED_NOW, Batch, perturb
from tests.test_gpu_run_areas import Env
rng = np.random.default_rng(5)
fr = Frontier(0)
env = Env(fr)
for K, n in ((1, 40), (64, 40), (4, 8 * 1025)):
    b = Batch(env, TIMERS | SCHED | RUNCTL, K, n, n)
    t, s, c = perturb(rng, b.m, np.arange(n))
    fr.resident_resync_areas(b.h, n, timers=t, sched=s, runctl=c, fired_now=FIRED_NOW, check=True, items_cap=7, drifted_cap=3)
    runs = np.arange(1, n, 3, dtype=np.uint32)
    fr.resident_resync_areas(b.h, n, runs=runs, timers=t[runs], sched=s[runs], runctl=c[runs], fired_now=FIRED_NOW)
    fr.resident_resync_areas(b.h, n, timers=t, sched=s, runctl=c, fired_now=FIRED_NOW)
    p_items = fr.alloc_pinned(16 * 64).view(Frontier.DRIFT_DTYPE)
    q = A.ResyncAreas(struct_size=__import__("ctypes").sizeof(A.ResyncAreas), n_runs=n, n=n, areas=A.RESYNC_AREA_SCHED,
                      fired_now=FIRED_NOW, sched=s.ctypes.data, items=p_items.ctypes.data, items_cap=64)
    fr._lib.bf_resident_resync_areas(fr._ctx, b.h, __import__("ctypes").byref(q))
    fr.free_pinned(p_items)
    bad = s.copy()
    bad["run"][0] = 1
    try:
        fr.resident_resync_areas(b.h, n, sched=bad)
    except A.FrontierError:
        pass
print("probe ok")
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python /tmp/san_resync_areas.py 2>&1 | tail -6
done
