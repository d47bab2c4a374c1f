#!/bin/bash
# tools/sanitize_runctl.sh: compute-sanitizer (memcheck, racecheck, synccheck) over the run-control kernels and the kernels that
# gained its re-keying — the put (with stops), the upload's re-stop, the delta scatter with RUN_FLAGS deltas of stopped runs, fires
# with story timeouts and drain deadlines over one and several CTAs with a capped list and without a timer area, redrives of both
# kinds (two requests of one run in one launch), retire (with a new capacity), transfer (a fit and a refusal into a batch without
# an area) and reshape.  Prints the tools' summaries.
cd "$(dirname "$0")/.."
cat > /tmp/san_runctl.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np
from bobrapet_b200 import _abi as A, Frontier
from bobrapet_b200.records import make_layout
from tests import randgen, reshape as RS
from tests.test_gpu_timers import requests
from tests.test_gpu_runctl import puts
rng = np.random.default_rng(3)
fr = Frontier(0)
ts = randgen.random_topologies(rng, 4, 40, 40, max_deg=3, parallel=False, fill=0.5)
slots = fr.put_topologies(ts)
L0, st0, _ = randgen.random_state(rng, ts, slots, 700, A.F_DECISION, phase_mix="progress")
L = make_layout(64, 0, A.F_DECISION | A.F_ALL_OUT)
st = RS.reshape_state(L0, L, st0, 700)
h = fr.resident_create(L, 720)
fr.resident_upload(h, 0, st)
fr.resident_timers(h, 3)
fr.resident_sched(h)
fr.resident_runctl(h)
fr.resident_timers_arm(h, requests(rng, L, 720, 600, step_hi=40))
fr.resident_runctl_put(h, puts(rng, 720, 500, p_stop=0.3, hi=400))
fr.resident_upload(h, 0, st[:300])
d = np.zeros(64, dtype=Frontier.DELTA_DTYPE)
d["run"] = np.arange(64) * 11
d["field"] = A.DELTA_RUN_FLAGS
d["code"] = 1
fr.resident_apply(h, d)
fr.resident_fire(h, 700, 200, fired_cap=17)
fr.resident_fire(h, 5, 600)
rq = np.zeros(12, dtype=Frontier.REDRIVE_DTYPE)
for i in range(12):
    r = i // 2
    rq[i] = (r, int(st[r, :4].view(np.uint32)[0]), A.REDRIVE_ALL if i % 2 else 3, 0)
fr.resident_redrive(h, rq)
fr.resident_retire(h, 700, np.arange(0, 700, 7, dtype=np.uint32), 650)
n = 700 - 100
g = fr.resident_create(L, 300)
fr.resident_timers(g, 3)
try:
    fr.resident_transfer(h, g, n, 0, np.arange(n, dtype=np.uint32)[:200])
except A.FrontierError:
    pass
fr.resident_runctl(g)
fr.resident_transfer(h, g, n, 0, np.array([r for r in range(n) if r % 50 == 1][:4], dtype=np.uint32))
fr.resident_reshape(h, make_layout(128, 0, L.fields), 900)
b = fr.resident_create(L, 50)
fr.resident_runctl(b)
fr.resident_upload(b, 0, st[:50])
fr.resident_runctl_put(b, puts(rng, 50, 50, p_stop=0.5, hi=10))
fr.resident_fire(b, 50, 5)
print("probe ok")
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python /tmp/san_runctl.py 2>&1 | tail -6
done
