"""Random sequences over two resident batches with limiter inputs: puts, deltas under every tick kind, fires, uploads, retires
(with and without a new capacity), transfers, reshapes (new capacity, new words), narrows, migrations and redrives, each
followed by ticks of both batches and one bf_resident_schedule over both, compared with the host model (tests/sched_resident.py):
totals, listed runs, heads and events.  Every sequence must schedule after every kind of operation."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import make_layout
from tests import schedref as SR
from tests.test_gpu_sched_resident import NONE_D, Resident, _batch, _inputs, _schedule

pytestmark = pytest.mark.gpu

OPS = ("put", "deltas", "fire", "upload", "retire", "retire_cap", "transfer", "reshape", "reshape_words", "narrow", "migrate",
       "redrive")
TICKS = ("dense", "compact", "changed", "touched")


@pytest.fixture(scope="module")
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _slot_of(fr, b, r):
    return int(fr.resident_download(b.h, r, 1, b.L.state_stride)[0, :4].copy().view("<u4")[0])


@pytest.mark.parametrize("seed", range(3))
def test_random_sequences(fr, seed):
    rng = np.random.default_rng(7000 + seed)
    now = 1000
    tables = SR.random_tables(rng, 16, 3, 2000, maxprio_base=bool(seed % 2))
    ts_a, sl_a, L_a, st_a, topo_a = _batch(rng, fr, 500, 60, parallel=False, count=12)
    ts_b, sl_b, L_b, st_b, topo_b = _batch(rng, fr, 400, 250, smin=100, parallel=False, count=12)
    descs = {**SR.from_topology_set(ts_a, sl_a), **SR.from_topology_set(ts_b, sl_b)}
    S_of = {int(s): int(ts_a.S[i]) for i, s in enumerate(sl_a)}
    S_of.update({int(s): int(ts_b.S[i]) for i, s in enumerate(sl_b)})
    a = Resident(fr, L_a, st_a, 700, descs)
    b = Resident(fr, L_b, st_b, 700, descs)
    home = {a.h: L_a, b.h: L_b}
    done = set()
    try:
        for x in (a, b):
            x.put(_inputs(rng, x.n, 16, 3, now))
            fr.resident_timers(x.h, 2)
        order = list(OPS) + list(rng.choice(OPS, size=14))
        rng.shuffle(order)
        for step, op in enumerate(order):
            x = (a, b)[int(rng.integers(0, 2))]
            now += int(rng.integers(0, 40))
            if op == "put":
                runs = np.sort(rng.choice(x.n, size=min(x.n, 30), replace=False))
                p = _inputs(rng, runs.size, 16, 3, now)
                p["run"] = runs
                x.put(p)
            elif op == "deltas":
                st = fr.resident_download(x.h, 0, x.n, x.L.state_stride)
                sid = st[:, :4].copy().view("<u4")[:, 0]
                d = np.zeros(20, Frontier.DELTA_DTYPE)
                d["run"] = rng.choice(x.n, size=20, replace=False)
                d["index"] = [int(rng.integers(0, S_of[int(sid[r])])) for r in d["run"]]
                d["field"] = A.DELTA_PHASE
                d["code"] = rng.choice([0, 1, 2, 2, 3, 14], size=20)
                fr.resident_apply(x.h, d)
            elif op == "fire":
                r = int(rng.integers(0, x.n))
                fr.resident_apply(x.h, np.array([(r, 0, A.DELTA_PHASE, A.PHASE_RUNNING), (r, 0, A.DELTA_DECISION, A.DEC_PENDING)],
                                                Frontier.DELTA_DTYPE))
                fr.resident_timers_arm(x.h, np.array([(r, 0, A.DEC_SUCCEED, 0, now, 0)], Frontier.TIMER_DTYPE))
                assert fr.resident_fire(x.h, x.n, now)["n_written"] == 1
            elif op == "upload":
                st = fr.resident_download(x.h, 0, x.n, x.L.state_stride)
                first, k = int(rng.integers(0, x.n - 10)), 10
                fr.resident_upload(x.h, first, np.ascontiguousarray(st[rng.choice(x.n, size=k)]))
                x.model.upload(first, k)
            elif op in ("retire", "retire_cap"):
                gone = rng.choice(x.n, size=int(rng.integers(1, 25)), replace=False)
                m = x.n - gone.size
                cap = int(rng.integers(m, x.model.cap + 1)) if op == "retire_cap" else 0
                newn, mf, mt = fr.resident_retire(x.h, x.n, gone, cap)
                moves = x.model.retire(x.n, gone)
                assert sorted(moves) == sorted(zip(mf.tolist(), mt.tolist()))
                if cap:
                    x.model.resize(cap)
                x.n = newn
            elif op == "transfer":
                k = min(int(rng.integers(1, 20)), b.model.cap - b.n, a.n - 1)
                if k <= 0:   # no room: grow the destination first, as a batcher would
                    fr.resident_reshape(b.h, b.L, b.model.cap + 40)
                    b.model.resize(b.model.cap + 40)
                    k = 10
                runs = rng.choice(a.n, size=k, replace=False)
                arriving = a.model.inputs[runs].copy()
                t = fr.resident_transfer(a.h, b.h, a.n, b.n, runs)
                a.model.retire(a.n, runs)
                b.model.receive(b.n, arriving)
                a.n, b.n = t["src_n_runs"], t["dst_n_runs"]
            elif op in ("reshape", "reshape_words"):
                L2 = make_layout(min(1024, x.L.steps_max + 40), x.L.child_nibbles, x.L.fields) if op == "reshape_words" else x.L
                cap = x.model.cap + int(rng.integers(0, 60))
                fr.resident_reshape(x.h, L2, cap)
                x.model.resize(cap)
                x.model.relayout(L2)
                x.L = L2
            elif op == "narrow":
                L2 = home[x.h]
                fr.resident_narrow(x.h, L2, x.n)
                x.model.relayout(L2)
                x.L = L2
            elif op == "migrate":
                slot = _slot_of(fr, x, int(rng.integers(0, x.n)))
                S = S_of[slot]
                nt = TopologySet(S=[S], E=[0], row_ptr=np.zeros(S + 1, np.uint32), col_idx=np.zeros(0, np.uint16),
                                 step_flags=np.zeros(S, np.uint8))
                new = int(fr.put_topologies(nt)[0])
                S_of[new] = S
                for y in (a, b):
                    y.descs = {**y.descs, **SR.from_topology_set(nt, [new])}
                sid = fr.resident_download(x.h, 0, x.n, x.L.state_stride)[:, :4].copy().view("<u4")[:, 0]
                on = np.nonzero(sid == slot)[0]
                assert fr.resident_migrate(x.h, slot, new, np.arange(S, dtype=np.uint16), x.n) == on.size > 0
                x.model.lose_baseline(on)
            elif op == "redrive":
                r = int(rng.integers(0, x.n))
                req = np.array([(r, _slot_of(fr, x, r), A.REDRIVE_ALL, 0)], Frontier.REDRIVE_DTYPE)
                assert fr.resident_redrive(x.h, req)[1] == 1
            for y in (a, b):
                kind = TICKS[int(rng.integers(0, len(TICKS)))]
                if kind == "dense":
                    fr.resident_tick(y.h, y.L, y.n, NONE_D)
                elif kind == "compact":
                    fr.resident_tick_compact(y.h, y.n, NONE_D, 1 << 22)
                elif kind == "changed":
                    fr.resident_tick_compact(y.h, y.n, NONE_D, 1 << 22, flags=A.EVAL_CHANGED_ONLY)
                else:
                    fr.resident_tick_touched(y.h, y.n, NONE_D, y.n, 1 << 22)
            caps = [dict(runs_cap=int(rng.integers(0, 40)), events_cap=int(rng.integers(0, 300)))] * 2 if step % 5 == 4 else None
            _schedule(fr, [a, b], tables, now, caps=caps)
            done.add(op)
        assert done == set(OPS)
    finally:
        a.close()
        b.close()
