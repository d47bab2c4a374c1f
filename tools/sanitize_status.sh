#!/bin/bash
# tools/sanitize_status.sh: compute-sanitizer (memcheck, racecheck, synccheck) over the run-status kernels — a batch with parallel
# steps (the shared stage of the join) and run control, every run and a subset with a short event buffer; a batch without a child
# area; several CTAs of the count, scan and list launches.  Prints the tools' summaries.
cd "$(dirname "$0")/.."
cat > /tmp/san_status.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np
from bobrapet_b200 import _abi as A, Frontier
from tests import randgen
rng = np.random.default_rng(3)
fr = Frontier(0)
for parallel, S in ((True, 200), (False, 40)):
    ts = randgen.random_topologies(rng, 6, S // 2, S, max_deg=3, parallel=parallel, fill=0.5)
    slots = fr.put_topologies(ts)
    L, st, _ = randgen.random_state(rng, ts, slots, 900, A.F_COND | A.F_DECISION | A.F_OUT_FAIL, phase_mix="progress")
    h = fr.resident_create(L, 900)
    fr.resident_upload(h, 0, st)
    fr.resident_runctl(h)
    req = np.zeros(50, dtype=Frontier.RUNCTL_PUT_DTYPE)
    req["run"], req["story_deadline"], req["drain_deadline"] = np.arange(50) * 17, A.TIMER_NONE, A.TIMER_NONE
    req["stop"] = np.arange(50) % 4
    fr.resident_runctl_put(h, req)
    fr.resident_status(h, 900)
    fr.resident_status(h, 900, np.arange(3, 900, 5, dtype=np.uint32), events_cap=40)
print("probe ok")
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python /tmp/san_status.py 2>&1 | tail -6
done
