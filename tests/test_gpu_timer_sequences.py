"""Random interleavings of timer arms and fires with deltas, touched and compact ticks, retires, redrives, migrations, reshapes
and narrows on one resident batch, compared bit for bit with the host model (tests/timers.py) after every step: the timer slots
always, the state records through every call the model restates (arm, fire, phase / decision deltas, ticks, retire)."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import randgen
from tests import reshape as RS
from tests import timers as T
from tests.test_gpu_timers import NONE, BIG, Twin, requests, _slot_of

pytestmark = pytest.mark.gpu

OPS = ["arm", "arm", "fire", "fire", "deltas", "touched", "compact", "retire", "redrive", "migrate", "reshape", "narrow"]


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _deltas(rng, tw, n, k):
    """phase and decision deltas, at most one per (run, field, step), applied to the model's records as the scatter does"""
    L, recs = tw.L, {}
    for _ in range(k):
        r, s = int(rng.integers(0, n)), int(rng.integers(0, 48))
        if rng.random() < 0.5:
            recs[(r, A.DELTA_PHASE, s)] = int(rng.choice([1, 2, 2, 3, 4, 8, 13]))
        else:
            recs[(r, A.DELTA_DECISION, s)] = int(rng.integers(0, 4))
    d = np.zeros(len(recs), dtype=Frontier.DELTA_DTYPE)
    for i, ((r, f, s), c) in enumerate(recs.items()):
        d[i] = (r, s, f, c)
        if f == A.DELTA_PHASE:
            T._set(tw.state[r], L.off_phase, L.words, 4, s, c)
        else:
            T._set(tw.state[r], L.off_decision, L.words, 2, s, c)
    return d


@pytest.mark.parametrize("seed", range(4))
def test_random_timer_sequences(fr, seed):
    rng = np.random.default_rng(1000 + seed)
    ts = randgen.random_topologies(rng, 6, 40, 48, max_deg=3, parallel=False, fill=0.5)
    slots = fr.put_topologies(ts)
    n = 400
    L0, st0, _ = randgen.random_state(rng, ts, slots, n, A.F_DECISION | A.F_COND, phase_mix="progress")
    L = make_layout(64, 0, L0.fields | A.F_ALL_OUT)
    tw = Twin(fr, L, RS.reshape_state(L0, L, st0, n), n + 16, int(rng.integers(1, 6)))
    now, seen = 0, set()
    for step in range(40):
        op = OPS[int(rng.integers(0, len(OPS)))] if step >= 2 else "arm"
        seen.add(op)
        if op == "arm":
            tw.arm(requests(rng, tw.L, n, int(rng.integers(1, 300)), step_hi=48))
        elif op == "fire":
            now += int(rng.integers(0, 150))
            tw.fire(int(rng.integers(0, n + 1)), now, cap=int(rng.choice([0, 5, 4096])))
        elif op == "deltas":
            fr.resident_apply(tw.h, _deltas(rng, tw, n, 60))
        elif op == "touched":
            fr.resident_tick_touched(tw.h, n, NONE, n, BIG)
        elif op == "compact":
            fr.resident_tick_compact(tw.h, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        elif op == "retire" and n > 100:
            runs = rng.choice(n, size=int(rng.integers(1, 20)), replace=False).astype(np.uint32)
            capacity = 0 if rng.random() < 0.5 or tw.cap - 3 < n - runs.size else tw.cap - 3
            m, mf, mt = fr.resident_retire(tw.h, n, runs, capacity)
            moved = tw.state.copy()
            for a, b in zip(mf, mt):
                moved[b] = tw.state[a]
            moved[m:n] = 0
            tw.state = moved[:capacity] if capacity else moved
            tw.area = T.retire(tw.area, n, runs, capacity)
            n = m
        elif op == "redrive":
            live = sorted({_slot_of(tw.state, r) for r in range(n)})
            runs = rng.choice(n, size=20, replace=False)
            rq = np.zeros(20, dtype=Frontier.REDRIVE_DTYPE)
            for i, r in enumerate(runs):
                s = _slot_of(tw.state, int(r))
                if i % 4 == 0:
                    s = live[(live.index(s) + 1) % len(live)]
                rq[i] = (int(r), s, A.REDRIVE_ALL if i % 2 else int(rng.integers(0, 10)), 0)
            status, _ = fr.resident_redrive(tw.h, rq)
            tw.area = T.redrive(tw.area, rq, status)
            tw.state = fr.resident_download(tw.h, 0, tw.cap, tw.L.state_stride)   # the records: tests/test_gpu_redrive.py
        elif op == "migrate":
            a, b = (int(x) for x in rng.choice(len(slots), size=2, replace=False))
            perm = rng.permutation(int(ts.S[b]))[:int(ts.S[a])].astype(np.uint16)
            if perm.size < int(ts.S[a]):
                perm = np.concatenate([perm, np.full(int(ts.S[a]) - perm.size, T.MIGRATE_GONE, np.uint16)])
            perm[rng.random(perm.size) < 0.2] = T.MIGRATE_GONE
            migrated = [r for r in range(n) if _slot_of(tw.state, r) == int(slots[a])]
            assert fr.resident_migrate(tw.h, int(slots[a]), int(slots[b]), perm, n) == len(migrated)
            tw.area = T.migrate(tw.area, migrated, perm)
            tw.state = fr.resident_download(tw.h, 0, tw.cap, tw.L.state_stride)   # the records: tests/test_gpu_migrate.py
        elif op == "reshape":
            Lb = make_layout(128 if tw.L.steps_max == 64 else tw.L.steps_max, 0, tw.L.fields)
            fr.resident_reshape(tw.h, Lb, tw.cap + 8)
            tw.state = RS.reshape_state(tw.L, Lb, tw.state, tw.cap + 8)
            tw.L, tw.area = Lb, T.reshape(tw.area, tw.cap + 8)
        elif op == "narrow":
            Ln = make_layout(64, 0, tw.L.fields)
            if tw.L.steps_max != 64:
                fr.resident_narrow(tw.h, Ln, n)   # S <= 48, armed steps < 48: always fits
                tw.L = Ln
                tw.state = fr.resident_download(tw.h, 0, tw.cap, Ln.state_stride)   # the records: tests/test_gpu_narrow.py
            ext = fr.resident_extent(tw.h, n)
            steps, fields, _ = T.extent(tw.area)
            assert ext["steps_max"] >= steps and (ext["fields"] & fields) == fields
        tw.check()
    assert {"arm", "fire"} <= seen
