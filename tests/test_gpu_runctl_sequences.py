"""Random interleavings of run-control puts and fires with every resident call that moves, rewrites or re-lays runs (deltas,
upload, redrive of both kinds, retire, transfer into batches with and without a run-control area, reshape, narrow, migrate),
checked against the host model tests/runctl.py after every call: the run-control records of both batches, the flags byte of every
stopped run and the state records the model can follow.  Each sequence asserts that it exercised every kind of call."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import runctl as R
from tests import timers as T
from tests.test_gpu_reshape import _batch
from tests.test_gpu_runctl import Twin, puts

pytestmark = pytest.mark.gpu

KINDS = ("put", "fire", "deltas", "upload", "redrive_step", "redrive_all", "retire", "transfer", "transfer_bare", "reshape",
         "narrow", "migrate")


def _resync(tw):
    """after a call whose record effects lie outside the model (redrive, migrate, reshape, narrow): the stopped runs must still
    carry the stopped byte, then the model takes the device's records"""
    got = tw.fr.resident_download(tw.h, 0, tw.cap, tw.L.state_stride)
    stopped = np.nonzero(tw.area["stop"])[0]
    assert np.all(got[stopped, 4] == R.STOPPED_FLAGS)
    tw.state = got
    if tw.K:
        tw.timers = tw.fr.resident_timers_download(tw.h, 0, tw.cap, tw.K).view(np.uint64).reshape(tw.cap, tw.K).copy()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_sequences(seed):
    fr = Frontier(0)
    try:
        _sequence(fr, seed)
    finally:
        fr.close()


def _sequence(fr, seed):
    rng = np.random.default_rng(1000 + seed)
    n = 800
    S = 96
    pt, L, st = _batch(fr, rng, S, A.F_DECISION | A.F_ALL_OUT, False, n)
    slots = sorted(set(int(x) for x in np.ascontiguousarray(st[:, :4]).view("<u4")[:, 0]))
    assert pt.n_slots == pt.ts.count   # a fresh ctx: slot i holds topology i
    tw = Twin(fr, L, st, n + 200, K=2)
    N = n
    other = Twin(fr, L, st[:1], 2000, K=2)   # a second batch with an area
    other_n = 1
    bare = fr.resident_create(L, 2000)   # a batch without one
    bare_n = 0
    seen = set()
    now = 0
    for it in range(60):
        kind = KINDS[it % len(KINDS)] if it < len(KINDS) else str(rng.choice(KINDS))
        if kind == "put":
            tw.put(puts(rng, tw.cap, int(rng.integers(1, 200)), p_stop=0.3, hi=now + 300))
        elif kind == "fire":
            now += int(rng.integers(0, 120))
            tw.fire(N, now, cap=int(rng.choice([3, 100_000])))
        elif kind == "deltas":
            tw.flags_deltas(rng, 40)
        elif kind == "upload":
            first = int(rng.integers(0, N - 20))
            recs = tw.state[first:first + 20].copy()
            for r in range(20):   # a resync from a host that knows nothing of stops: the run's own flags byte
                if tw.area["stop"][first + r]:
                    recs[r][4] = int(rng.integers(0, 8))
            fr.resident_upload(tw.h, first, recs)
            R.upload(tw.area, tw.state, first, recs)
        elif kind in ("redrive_step", "redrive_all"):
            runs = rng.choice(N, size=30, replace=False)
            rq = np.zeros(30, dtype=Frontier.REDRIVE_DTYPE)
            for i, r in enumerate(runs):
                slot = int(tw.state[r][:4].view("<u4")[0])
                step = A.REDRIVE_ALL if kind == "redrive_all" else 0
                rq[i] = (int(r), slot if rng.random() < 0.9 else slots[0] if slot != slots[0] else slots[-1], step, 0)
            status, _ = fr.resident_redrive(tw.h, rq)
            before = tw.state.copy()
            R.redrive(tw.area, tw.state, rq, status)
            got = fr.resident_download(tw.h, 0, tw.cap, L.state_stride)
            for q, s_ in zip(rq, status):   # applied: the saved byte of a stopped run, without TOPOLOGY_TERMINATED
                r = int(q["run"])
                want = int(tw.state[r][4]) & ~R.RF_TOPOLOGY_TERMINATED & 0xFF if any(status[rq["run"] == r]) else before[r][4]
                assert got[r][4] == want, (r, got[r][4], want)
            _resync(tw)
        elif kind == "retire":
            runs = rng.choice(N, size=int(rng.integers(1, 30)), replace=False)
            r = fr.resident_retire(tw.h, N, runs)
            tw.area = R.retire(tw.area, N, runs)
            m, mv = T.retire_moves(N, runs)
            for s_, d_ in mv.items():
                tw.state[d_] = tw.state[s_]
            tw.state[m:N] = 0
            tw.timers = T.retire(tw.timers, N, runs)
            N = m
        elif kind in ("transfer", "transfer_bare"):
            runs = [int(x) for x in rng.choice(N, size=int(rng.integers(1, 10)), replace=False)]
            if kind == "transfer":
                fr.resident_transfer(tw.h, other.h, N, other_n, runs)
                _, other.area = R.transfer(tw.area, other.area, N, other_n, runs)
                _, other.timers = T.transfer(tw.timers, other.timers, N, other_n, runs)
                for i, r in enumerate(runs):
                    other.state[other_n + i] = tw.state[r]
                other_n += len(runs)
            else:
                runs = [r for r in runs if T.fits(tw.timers, r, 0)]   # no timer area either
                ok = all(R.fits(tw.area, None, r) for r in runs)
                if not ok:
                    before = fr.resident_download(bare, 0, 2000, L.state_stride)
                    with pytest.raises(A.FrontierError):
                        fr.resident_transfer(tw.h, bare, N, bare_n, runs)
                    assert np.array_equal(fr.resident_download(bare, 0, 2000, L.state_stride), before)
                    runs = [r for r in runs if R.fits(tw.area, None, r)][:3]
                if not runs:
                    seen.add(kind)
                    tw.check()
                    continue
                fr.resident_transfer(tw.h, bare, N, bare_n, runs)
                bare_n += len(runs)
            m, mv = T.retire_moves(N, runs)
            tw.area = R.retire(tw.area, N, runs)
            for s_, d_ in mv.items():
                tw.state[d_] = tw.state[s_]
            tw.state[m:N] = 0
            tw.timers = T.retire(tw.timers, N, runs)
            N = m
            other.check()
        elif kind == "reshape":
            cap = tw.cap + 16
            fr.resident_reshape(tw.h, L, cap)
            tw.area = R.reshape(tw.area, cap)
            tw.timers = T.reshape(tw.timers, cap)
            _resync(tw)
            if tw.sched is not None:
                tw.sched = fr.resident_sched_download(tw.h, 0, cap)
        elif kind == "narrow":   # drop an output field: the state records keep their layout, the area is kept
            out = L.fields & A.F_ALL_OUT
            T2 = make_layout(L.steps_max, L.child_nibbles, L.fields & ~(out & -out)) if out else L
            same_state = all(getattr(T2, f) == getattr(L, f) for f in ("state_stride", "off_phase", "off_decision"))
            fr.resident_narrow(tw.h, T2 if same_state else L, N)
            if same_state:
                tw.L = L = T2
            _resync(tw)
        elif kind == "migrate":   # the runs of one slot to another, keeping the step indices both have
            old = int(tw.state[0][:4].view("<u4")[0])
            new = [s_ for s_ in range(pt.ts.count) if s_ != old][0]
            so, sn = int(pt.ts.S[old]), int(pt.ts.S[new])
            step_map = np.array([i if i < sn else 0xFFFF for i in range(so)], dtype=np.uint16)
            fr.resident_migrate(tw.h, old, new, step_map, N)
            _resync(tw)
        seen.add(kind)
        tw.check()
    assert seen == set(KINDS), set(KINDS) - seen

