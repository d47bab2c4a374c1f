#!/bin/bash
# tools/sanitize.sh: compute-sanitizer (memcheck, racecheck, synccheck) over small passes of every kernel shape — smoke() plus a
# wide (S = 1024, parallel joins, 10-bit rows) and a pipelined batch, the limiters over the latter (bf_schedule_device), and a
# resident batch that takes an extent, a narrow (the extent and re-layout kernels) and touched ticks on either side of it, then a
# transfer of some of its runs into a wider batch and a transfer the fit check refuses (the fit, transfer and retire kernels).
# Prints the tools' summaries.
cd "$(dirname "$0")/.."
cat > /tmp/san_probe.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np, torch
import __graft_entry__ as g
from bobrapet_b200 import _abi as A, Frontier, synth
from bobrapet_b200.records import make_layout
from oracle import packed as PK
g.smoke()
fr = Frontier(0)
ts = synth.topologies(5, 0, 96, 1024)
slots = fr.put_topologies(ts)
pt = PK.PackedTopologies(ts, slots)
child = pt.max_child_nibbles()
L = make_layout(1024, child, A.F_COND | A.F_DECISION | A.F_CHILD)
cf = fr.child_first(int(slots[0]))
st = synth.state(5, 0, 96, L, slots, ts, cf)
got, c = fr.eval(L, st)
want, wc = PK.evaluate(pt, L, st, threads=4)
assert np.array_equal(got, want) and c == wc
f2 = Frontier(0)
ts3 = synth.topologies(3, 0, 1500, 256)
s3 = f2.put_topologies(ts3)
L3 = make_layout(256, 0, 0)
st3 = synth.state(3, 0, 1500, L3, s3, ts3)
w3, wc3 = PK.evaluate(PK.PackedTopologies(ts3, s3), L3, st3, threads=4)
dev = torch.device("cuda", 0)
d_state = torch.from_numpy(st3).to(dev)
res = [torch.zeros((1500, L3.result_stride), dtype=torch.uint8, device=dev) for _ in range(3)]
cnt = [torch.full((4,), 9, dtype=torch.int64, device=dev) for _ in range(3)]
s = torch.cuda.Stream()
with torch.cuda.stream(s):
    for k in range(6):
        f2.eval_device(L3, 1500, d_state.data_ptr(), res[k % 3].data_ptr(), cnt[k % 3].data_ptr(), s.cuda_stream,
                       flags=A.EVAL_COUNTS_SET | A.EVAL_PIPELINED)
torch.cuda.synchronize()
for k in range(3):
    assert np.array_equal(res[k].cpu().numpy(), w3) and cnt[k].cpu().numpy().tolist() == [wc3["ready"], wc3["skip"], wc3["expansion"], wc3["evals"]]
# the limiters on the device path over the pipelined batch: tables that span several sched_init blocks, keys out of range
from tests import schedref as SR
rs = np.random.default_rng(6)
sched = SR.random_sched(rs, 1500, 700, 40, out_of_range=0.05)
tables = SR.random_tables(rs, 700, 40, 1500, maxprio_base=True)
got = SR.schedule_device(f2, L3, 1500, d_state, res[2], sched, tables, s)
SR.assert_schedule(got, SR.expected(L3, st3, w3, SR.from_topology_set(ts3, s3), sched, tables))
from tests import randgen
from tests import reshape as RS
rng = np.random.default_rng(5)
f3 = Frontier(0)
ts4 = randgen.random_topologies(rng, 16, 8, 32, max_deg=4, parallel=False, fill=0.5)
s4 = f3.put_topologies(ts4)
L0, st0, _ = randgen.random_state(rng, ts4, s4, 600, 0, phase_mix="progress")
Lw, Ln = make_layout(256, 0, A.F_COND | A.F_ALL_OUT), make_layout(32, 0, A.F_ALL_OUT)
h = f3.resident_create(Lw, 640)
f3.resident_upload(h, 0, RS.reshape_state(L0, Lw, st0, 600))
e = f3.resident_extent(h, 600)
assert e["steps_max"] <= 32 and e["fields"] == 0, e
f3.resident_tick_touched(h, 600, np.zeros(0, dtype=Frontier.DELTA_DTYPE), 600, 1 << 20)
f3.resident_narrow(h, Ln, 600)
d = np.zeros(50, dtype=Frontier.DELTA_DTYPE)
d["run"], d["index"], d["field"], d["code"] = np.arange(0, 600, 12), 0, A.DELTA_PHASE, 3
o = f3.resident_tick_touched(h, 600, d, 600, 1 << 20)
assert o["full"] == 0 and o["n_evaluated"] == 50
st4 = f3.resident_download(h, 0, 600, Ln.state_stride)
got, _ = f3.resident_tick(h, Ln, 600, np.zeros(0, dtype=Frontier.DELTA_DTYPE))
want, _ = PK.evaluate(PK.PackedTopologies(ts4, s4), Ln, st4, threads=4)
assert np.array_equal(got, want)
# a transfer into a wider batch with every field (the fit and transfer kernels, the source's retire), one refused by the fit
Lx = make_layout(1024, 16, A.F_COND | A.F_DECISION | A.F_CHILD | A.F_ALL_OUT)
hx = f3.resident_create(Lx, 64)
t = f3.resident_transfer(h, hx, 600, 0, np.arange(0, 600, 13, dtype=np.uint32))
assert t["dst_n_runs"] == 47 and t["src_n_runs"] == 553
o = f3.resident_tick_touched(hx, 47, np.zeros(0, dtype=Frontier.DELTA_DTYPE), 64, 1 << 20)
assert o["full"] == 1 and o["n_listed"] == 47   # the destination's first tick
hy = f3.resident_create(make_layout(8, 0, 0), 8)
try:
    f3.resident_transfer(hx, hy, 47, 0, np.arange(4, dtype=np.uint32))
    raise AssertionError("a transfer the destination cannot hold was accepted")
except A.FrontierError as err:
    assert err.unfit != A.EXTENT_NO_RUN
for x in (h, hx, hy):
    f3.resident_destroy(x)
print("probe ok")
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python /tmp/san_probe.py 2>&1 | grep -v "^smoke\|NCCL" | tail -6
done
