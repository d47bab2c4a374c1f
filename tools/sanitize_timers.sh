#!/bin/bash
# tools/sanitize_timers.sh: compute-sanitizer (memcheck, racecheck, synccheck) over the step-timer kernels — the area's creation
# and growth (relay_timers), both arm launches with an overflow refusal, fires over one and several CTAs with a capped list, and
# the re-keying in retire (with a new capacity), redrive, migrate, transfer (a fit and a refusal), reshape and extent.  Prints the
# tools' summaries.
cd "$(dirname "$0")/.."
cat > /tmp/san_timers.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np
from bobrapet_b200 import _abi as A, Frontier
from bobrapet_b200.records import make_layout
from tests import randgen, reshape as RS
from tests.test_gpu_timers import requests
rng = np.random.default_rng(3)
fr = Frontier(0)
ts = randgen.random_topologies(rng, 4, 40, 40, max_deg=3, parallel=False, fill=0.5)
slots = fr.put_topologies(ts)
L0, st0, _ = randgen.random_state(rng, ts, slots, 700, A.F_DECISION, phase_mix="progress")
L = make_layout(64, 0, A.F_DECISION | A.F_ALL_OUT)
st = RS.reshape_state(L0, L, st0, 700)
h = fr.resident_create(L, 720)
fr.resident_upload(h, 0, st)
fr.resident_timers(h, 2)
fr.resident_timers(h, 5)
fr.resident_timers_arm(h, requests(rng, L, 720, 600, step_hi=40))
try:
    fr.resident_timers_arm(h, np.array([(9, s, 1, 0, 5, 0) for s in range(6)], dtype=Frontier.TIMER_DTYPE))
except A.FrontierError:
    pass
fr.resident_fire(h, 700, 300, fired_cap=17)
fr.resident_fire(h, 5, 600)
fr.resident_retire(h, 700, np.arange(0, 700, 7, dtype=np.uint32), 650)
n = 700 - 100
rq = np.zeros(10, dtype=Frontier.REDRIVE_DTYPE)
for i in range(10):
    rq[i] = (i, int(st[0, :4].view(np.uint32)[0]), A.REDRIVE_ALL if i % 2 else 3, 0)
fr.resident_redrive(h, rq)
fr.resident_migrate(h, int(slots[0]), int(slots[1]), rng.permutation(40).astype(np.uint16), n)
g = fr.resident_create(L, 300)
fr.resident_timers(g, 2)
try:
    fr.resident_transfer(h, g, n, 0, np.arange(n, dtype=np.uint32)[:200])
except A.FrontierError:
    pass
fr.resident_transfer(h, g, n, 0, np.array([r for r in range(n) if r % 50 == 1][:4], dtype=np.uint32))
fr.resident_reshape(h, make_layout(128, 0, L.fields), 900)
fr.resident_extent(h, n - 4)
fr.resident_fire(h, n - 4, 10_000)
print("probe ok")
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python /tmp/san_timers.py 2>&1 | tail -6
done
