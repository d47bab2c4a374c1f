#!/bin/bash
# tools/sanitize_sched.sh: compute-sanitizer (memcheck, racecheck, synccheck) over the resident limiter kernels — the inputs
# area's puts, schedules of one and of two batches (several CTAs, caps below the lists, n_runs = 0), and the re-keying in retire
# (with a new capacity), transfer, reshape (new words and capacity), narrow and migrate (a generation without parallel steps,
# so it goes through).  Prints the tools' summaries.
cd "$(dirname "$0")/.."
cat > /tmp/san_sched.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np
from bobrapet_b200 import _abi as A, Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import make_layout
from tests import randgen, sched_resident as SRM, schedref as SR
rng = np.random.default_rng(4)
fr = Frontier(0)
ts = randgen.random_topologies(rng, 6, 20, 60)
slots = fr.put_topologies(ts)
L, st, _ = randgen.random_state(rng, ts, slots, 900, A.F_COND | A.F_DECISION, phase_mix="progress")
none = np.zeros(0, Frontier.DELTA_DTYPE)
tables = SR.random_tables(rng, 20, 3, 900, maxprio_base=True)
hs = []
for n in (900, 300):
    h = fr.resident_create(L, 1000)
    fr.resident_upload(h, 0, st[:n])
    fr.resident_sched(h)
    p = SRM.defaults(n)
    p["run"] = np.arange(n)
    p["story_key"], p["queue_key"] = rng.integers(0, 22, size=n), rng.integers(0, 4, size=n)
    p["queued_since"] = rng.integers(0, 200, size=n)
    fr.resident_sched_put(h, p)
    fr.resident_tick_compact(h, n, none, 1 << 22)
    hs.append((h, n))
(a, na), (b, nb) = hs
fr.resident_schedule([dict(handle=a, n_runs=na, runs_cap=13, events_cap=99), dict(handle=b, n_runs=nb)], tables, 100)
fr.resident_schedule([dict(handle=a, n_runs=0), dict(handle=b, n_runs=nb)], tables, 150)
m, _, _ = fr.resident_retire(a, na, np.arange(0, na, 9, dtype=np.uint32), 950)
t = fr.resident_transfer(a, b, m, nb, np.arange(0, m, 11, dtype=np.uint32))
fr.resident_reshape(a, make_layout(128, L.child_nibbles, L.fields), 1200)
fr.resident_narrow(a, L, t["src_n_runs"])
slot = int(fr.resident_download(b, 0, 1, L.state_stride)[0, :4].view("<u4")[0])
S = int(ts.S[list(slots).index(slot)])
flat = TopologySet(S=[S], E=[0], row_ptr=np.zeros(S + 1, np.uint32), col_idx=np.zeros(0, np.uint16), step_flags=np.zeros(S, np.uint8))
assert fr.resident_migrate(b, slot, int(fr.put_topologies(flat)[0]), np.arange(S, dtype=np.uint16), t["dst_n_runs"]) > 0
for h, n in ((a, t["src_n_runs"]), (b, t["dst_n_runs"])):
    fr.resident_tick_compact(h, n, none, 1 << 22)
fr.resident_schedule([dict(handle=a, n_runs=t["src_n_runs"]), dict(handle=b, n_runs=t["dst_n_runs"])], tables, 200)
print("probe ok")
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python /tmp/san_sched.py 2>&1 | tail -6
done
