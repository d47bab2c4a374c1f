#!/bin/bash
# tools/sanitize_tick_many.sh: compute-sanitizer (memcheck, racecheck, synccheck) over bf_resident_tick_touched_many — three
# width classes (64, 512 with decision planes, 1024 with a child area) through a full first call, touched calls with pinned and
# pageable buffers and caps below the counts, a part whose tick is full between two that are not, a part without touched runs,
# a rejected delta and a refused call.  Prints the tools' summaries.
cd "$(dirname "$0")/.."
cat > /tmp/san_tick_many.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np
from bobrapet_b200 import _abi as A, Frontier
from tests import randgen
from tests.test_gpu_tick_many import deltas, NONE
rng = np.random.default_rng(5)
fr = Frontier(0)
class P: pass
parts = []
for s_lo, s_hi, par, fields, n in ((20, 64, False, 0, 3000), (300, 512, False, A.F_COND | A.F_DECISION | A.F_ALL_OUT, 900),
                                   (600, 1000, True, A.F_ALL_OUT, 400)):
    p = P()
    p.ts = randgen.random_topologies(rng, 6, s_lo, s_hi, max_deg=4, parallel=par, fill=0.5)
    p.slots = fr.put_topologies(p.ts)
    p.L, st, _ = randgen.random_state(rng, p.ts, p.slots, n, fields, phase_mix="progress")
    p.n, p.h = n, fr.resident_create(p.L, n + 20)
    fr.resident_upload(p.h, 0, st)
    parts.append(p)
def call(ds, caps=None, pinned=(False, False, False), n=None):
    q = []
    for p, d, (rc, ec), pn in zip(parts, ds, caps or [(p.n, 1 << 22) for p in parts], pinned):
        e = dict(handle=p.h, n_runs=n or p.n, deltas=d, runs_cap=rc, events_cap=ec)
        if pn:
            e.update(runs=fr.alloc_pinned(4 * max(rc, 1)).view(np.uint32), head=fr.alloc_pinned(4 * max(rc, 1)).view(np.uint32),
                     events=fr.alloc_pinned(2 * max(ec, 1)).view(np.uint16))
        q.append(e)
    try:
        fr.resident_tick_touched_many(q)
    except A.FrontierError as e:
        print("refused or rejected:", e.bad_part)
    for e in q:
        for k in ("runs", "head", "events"):
            if k in e:
                fr.free_pinned(e[k])
call([NONE] * 3)
call([deltas(rng, p, 200) for p in parts], caps=[(5, 7), (0, 0), (50, 1 << 20)], pinned=(True, False, True))
fr.resident_upload(parts[1].h, parts[1].n, np.zeros((20, parts[1].L.state_stride), np.uint8))
parts[1].n += 20
call([deltas(rng, parts[0], 30), NONE, NONE])
call([deltas(rng, p, 10, rejected=(i == 1)) for i, p in enumerate(parts)])
call([deltas(rng, p, 10) for p in parts], n=1 << 30)
print("probe ok")
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python /tmp/san_tick_many.py 2>&1 | tail -6
done
