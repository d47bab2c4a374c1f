"""The run status of resident batches on the device (bf_resident_status) against the host model tests/runstatus.py, byte for byte:
random batches at several widths, with and without cond / decision / child planes, compensation and finally groups, host-group and
stopped runs, dead slots, subsets of the runs, short event buffers, pinned buffers and every refusal; that the call changes nothing
a later call reads; the status after random per-tick loops; and runs moved by retire, transfer, migrate and redrive."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import randgen
from tests import runstatus as M
from tests.test_gpu_commit import BIG, TABLES
from tests.test_host_commit import no_stops

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
PLANES = [0, A.F_COND | A.F_OUT_FAIL, A.F_DECISION, A.F_COND | A.F_DECISION | A.F_ALL_OUT]


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _batch(fr, rng, S, fields, parallel, n, dead=0.03, host_groups=0.1, stops=True, cap=None):
    """random topologies of at most S steps, n runs of them resident on the device (capacity cap, default n); a share of the runs
    hold a slot never put (dead) and a share have a host-set group; stops=False makes every stop step an engram step (a commit
    then needs no entries) -> (ts, slots, L, state, handle)"""
    ts = randgen.random_topologies(rng, 12, max(2, S // 2), S, max_deg=4, parallel=parallel, fill=0.5)
    ts = ts if stops else no_stops(ts)
    slots = fr.put_topologies(ts)
    L, st, _ = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
    hg = rng.random(n) < host_groups
    st[hg, 4] = (st[hg, 4] & 0x07) | A.RF_HOST_GROUP | (rng.integers(0, 4, int(hg.sum())) << A.RF_HOST_GROUP_SHIFT).astype(np.uint8)
    st[rng.random(n) < dead, 0:4] = np.frombuffer(np.uint32(0xFFFF).tobytes(), np.uint8)
    h = fr.resident_create(L, cap or n)
    fr.resident_upload(h, 0, st)
    return ts, slots, L, st, h


def _same(got, want):
    g, ge, gn = got
    w, we, wn = want
    assert gn == wn
    assert np.array_equal(ge, we), (ge[:20], we[:20])
    assert g.tobytes() == w.tobytes(), next((i, g[i], w[i]) for i in range(len(g)) if g[i].tobytes() != w[i].tobytes())


@pytest.mark.parametrize("fields", PLANES)
@pytest.mark.parametrize("S", [64, 256, 1024])
def test_random_batches(fr, S, fields):
    rng = np.random.default_rng(S * 31 + fields)
    n = 600 if S < 1024 else 200
    ts, slots, L, st, h = _batch(fr, rng, S, fields, parallel=True, n=n)
    _same(fr.resident_status(h, n), M.status(L, ts, slots, st, n))
    runs = np.sort(rng.choice(n, size=n // 7, replace=False)).astype(np.uint32)
    _same(fr.resident_status(h, n, runs), M.status(L, ts, slots, st, n, runs))
    full = M.status(L, ts, slots, st, n)
    cap = full[2] // 3
    _same(fr.resident_status(h, n, events_cap=cap), M.status(L, ts, slots, st, n, events_cap=cap))
    assert fr.resident_download(h, 0, n, L.state_stride).tobytes() == st.tobytes()


@pytest.mark.parametrize("parallel", [False, True])
def test_stopped_runs(fr, parallel):
    """runs stopped for each reason report it; the others of the batch are unaffected"""
    rng = np.random.default_rng(7 + parallel)
    n = 500
    ts, slots, L, st, h = _batch(fr, rng, 96, A.F_COND | A.F_DECISION | A.F_OUT_FAIL, parallel, n)
    fr.resident_runctl(h)
    stop = rng.choice(n, size=60, replace=False)
    req = np.zeros(stop.size, dtype=Frontier.RUNCTL_PUT_DTYPE)
    req["run"], req["story_deadline"], req["drain_deadline"] = stop, A.TIMER_NONE, A.TIMER_NONE
    req["stop"] = rng.integers(1, 4, stop.size)
    fr.resident_runctl_put(h, req)
    area = fr.resident_runctl_download(h, 0, n)
    state = fr.resident_download(h, 0, n, L.state_stride)
    got = fr.resident_status(h, n)
    _same(got, M.status(L, ts, slots, state, n, runctl=area))
    outcomes = set(got[0]["outcome"].tolist())
    assert {A.OUTCOME_TIMED_OUT, A.OUTCOME_CANCELED, A.OUTCOME_STOPPED, A.OUTCOME_DEAD} <= outcomes


def test_every_outcome_on_device(fr):
    """a batch large enough to reach every outcome a run without stops can have, with compensation and finally groups"""
    rng = np.random.default_rng(11)
    n = 4000
    ts, slots, L, st, h = _batch(fr, rng, 48, A.F_DECISION, True, n, host_groups=0.0)
    got = fr.resident_status(h, n)
    _same(got, M.status(L, ts, slots, st, n))
    seen = set(got[0]["outcome"].tolist())
    assert {A.OUTCOME_NONE, A.OUTCOME_SUCCEEDED, A.OUTCOME_DEPENDENCY_FAILED, A.OUTCOME_COMPENSATED,
            A.OUTCOME_COMPENSATION_FAILED, A.OUTCOME_CLEANUP_FAILED, A.OUTCOME_DEAD} <= seen, seen


def test_pinned_buffers(fr):
    """pinned runs, records and events are used in place and give the same report"""
    rng = np.random.default_rng(3)
    n = 700
    ts, slots, L, st, h = _batch(fr, rng, 128, A.F_COND | A.F_OUT_FAIL, True, n)
    runs = np.sort(rng.choice(n, size=300, replace=False)).astype(np.uint32)
    want = M.status(L, ts, slots, st, n, runs)
    p_runs = fr.alloc_pinned(4 * runs.size).view(np.uint32)
    p_recs = fr.alloc_pinned(32 * runs.size).view(Frontier.STATUS_DTYPE)
    p_ev = fr.alloc_pinned(2 * max(want[2], 1)).view(np.uint16)
    p_runs[:] = runs
    out = A.StatusOut(struct_size=ctypes.sizeof(A.StatusOut), records=p_recs.ctypes.data, events=p_ev.ctypes.data,
                      events_cap=want[2])
    assert fr._lib.bf_resident_status(fr._ctx, h, n, p_runs.ctypes.data, runs.size, ctypes.byref(out)) == A.BF_OK
    _same((p_recs.copy(), p_ev[:want[2]].copy(), int(out.n_events)), want)
    for a in (p_runs, p_recs, p_ev):
        fr.free_pinned(a)


def _with_areas(fr, h, n, rng):
    """timer slots, limiter inputs and run control on batch h, with armed timers, deadlines and a few stops"""
    fr.resident_timers(h, 2)
    fr.resident_sched(h)
    fr.resident_runctl(h)
    runs = np.sort(rng.choice(n, size=n // 4, replace=False))
    tq = np.zeros(runs.size, dtype=Frontier.TIMER_DTYPE)
    tq["run"], tq["step"], tq["code"], tq["deadline"] = runs, 0, A.DEC_PENDING, rng.integers(5, 50, runs.size)
    fr.resident_timers_arm(h, tq)
    q = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
    q["run"], q["story_key"], q["queue_key"] = np.arange(n), np.arange(n) % 4, np.arange(n) % 3
    q["priority"], q["queued_since"], q["run_phase"] = np.arange(n) % 5, A.SCHED_NONE, A.PHASE_RUNNING
    fr.resident_sched_put(h, q)
    c = np.zeros(runs.size, dtype=Frontier.RUNCTL_PUT_DTYPE)
    c["run"], c["story_deadline"], c["drain_deadline"] = runs, rng.integers(10, 60, runs.size), A.TIMER_NONE
    c["stop"] = np.where(np.arange(runs.size) % 9 == 0, A.STOP_HOST, A.STOP_NONE)
    fr.resident_runctl_put(h, c)


def _eq(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_eq(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.tobytes() == b.tobytes()
    return a == b


def test_read_only(fr):
    """Two copies of one batch with every side area take the same calls, one with status calls between them: the state records,
    the side areas, the stored results (a changed-only tick lists exactly the runs whose result differs from them), the stored
    schedules (a schedule lists the runs whose schedule changed) and the touched tick's lists stay the same"""
    rng = np.random.default_rng(5)
    n = 800
    ts, slots, L, st, h1 = _batch(fr, rng, 200, A.F_COND | A.F_DECISION | A.F_ALL_OUT, True, n, stops=False)
    h2 = fr.resident_create(L, n)
    fr.resident_upload(h2, 0, st)
    for h in (h1, h2):
        _with_areas(fr, h, n, np.random.default_rng(6))
    d = np.zeros(40, dtype=Frontier.DELTA_DTYPE)
    d["run"] = rng.choice(n, size=40, replace=False)
    d["field"], d["index"], d["code"] = A.DELTA_PHASE, 0, A.PHASE_SUCCEEDED

    def step(h, k, with_status):
        out = {"fire": fr.resident_fire(h, n, 20 * k)}
        if with_status:
            fr.resident_status(h, n)
        out["touched"] = fr.resident_tick_touched(h, n, d if k == 1 else NONE_D, n, n * 256)
        if with_status:
            fr.resident_status(h, n, np.arange(0, n, 3, dtype=np.uint32))
        out["schedule"] = fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], TABLES, 20 * k)
        if with_status:
            fr.resident_status(h, n)
        out["commit"] = fr.resident_commit(h, n)
        if with_status:
            fr.resident_status(h, n)
        out["changed"] = fr.resident_tick_compact(h, n, NONE_D, n * 256, flags=A.EVAL_CHANGED_ONLY)
        out["state"] = fr.resident_download(h, 0, n, L.state_stride)
        out["timers"] = fr.resident_timers_download(h, 0, n, 2)
        out["sched"] = fr.resident_sched_download(h, 0, n)
        out["runctl"] = fr.resident_runctl_download(h, 0, n)
        return out

    for k in range(3):
        a, b = step(h1, k, True), step(h2, k, False)
        for key in a:
            assert _eq(a[key], b[key]), (k, key)


def test_after_per_tick_loop(fr):
    """random per-tick loops (Fire -> touched tick with deltas -> schedule -> commit) over a batch with every side area: the status
    of the runs the tick listed as done and of every run matches the model over the records and run control the device holds,
    with commit writes, fired story timeouts and stops in them"""
    rng = np.random.default_rng(31)
    n = 700
    ts, slots, L, st, h = _batch(fr, rng, 96, A.F_COND | A.F_DECISION | A.F_ALL_OUT, True, n, dead=0.0, stops=False)
    _with_areas(fr, h, n, rng)
    outcomes = set()
    for k in range(10):
        fr.resident_fire(h, n, 6 * k)
        d = np.zeros(60, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"] = rng.choice(n, size=60, replace=False), rng.integers(0, 48, 60)
        d["field"], d["code"] = A.DELTA_PHASE, rng.choice([A.PHASE_RUNNING, A.PHASE_SUCCEEDED, A.PHASE_FAILED, A.PHASE_SKIPPED], 60)
        t = fr.resident_tick_touched(h, n, d, n, n * 256)
        fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], TABLES, 6 * k)
        fr.resident_commit(h, n)
        state = fr.resident_download(h, 0, n, L.state_stride)
        area = fr.resident_runctl_download(h, 0, n)
        done = np.asarray(t["runs"][(t["head"] & A.SUM_GROUP_MASK) == A.GROUP_DONE], np.uint32)
        _same(fr.resident_status(h, n, done), M.status(L, ts, slots, state, n, done, runctl=area))
        got = fr.resident_status(h, n)
        _same(got, M.status(L, ts, slots, state, n, runctl=area))
        outcomes |= set(got[0]["outcome"].tolist())
    assert {A.OUTCOME_NONE, A.OUTCOME_TIMED_OUT, A.OUTCOME_STOPPED} <= outcomes, outcomes


def _moved_same(before, got, moves_from, moves_to):
    """each moved run's record at its new index equals its record before the move, but for run and first_event"""
    by_from = {int(r["run"]): r for r in before[0]}
    for f, t in zip(moves_from, moves_to):
        a, b = by_from[int(f)].copy(), got[0][int(t)].copy()
        a["run"] = b["run"] = 0
        a["first_event"] = b["first_event"] = 0
        assert a.tobytes() == b.tobytes()


def test_after_retire(fr):
    """after a retire the moved runs report under their new indices"""
    rng = np.random.default_rng(9)
    n = 400
    ts, slots, L, st, h = _batch(fr, rng, 80, A.F_DECISION, True, n)
    gone = rng.choice(n, size=90, replace=False)
    m, mf, mt = fr.resident_retire(h, n, gone)
    state = fr.resident_download(h, 0, m, L.state_stride)
    got = fr.resident_status(h, m)
    _same(got, M.status(L, ts, slots, state, m))
    _moved_same(M.status(L, ts, slots, st, n, np.sort(mf)), got, mf, mt)


def test_after_transfer(fr):
    """runs moved to another batch report there under their new indices, and the source's compacted runs under theirs"""
    rng = np.random.default_rng(13)
    n = 300
    ts, slots, L, st, h = _batch(fr, rng, 80, A.F_DECISION, True, n)
    g = fr.resident_create(L, n)
    other = fr.resident_download(h, 0, 40, L.state_stride)
    fr.resident_upload(g, 0, other)
    runs = np.sort(rng.choice(n, size=70, replace=False)).astype(np.uint32)
    t = fr.resident_transfer(h, g, n, 40, runs)
    got = fr.resident_status(g, t["dst_n_runs"])
    dst_state = fr.resident_download(g, 0, t["dst_n_runs"], L.state_stride)
    _same(got, M.status(L, ts, slots, dst_state, t["dst_n_runs"]))
    before = M.status(L, ts, slots, st, n, runs)
    _moved_same(before, got, runs, np.arange(40, 40 + runs.size))
    src_state = fr.resident_download(h, 0, t["src_n_runs"], L.state_stride)
    _same(fr.resident_status(h, t["src_n_runs"]), M.status(L, ts, slots, src_state, t["src_n_runs"]))


def test_after_migrate_and_redrive(fr):
    """runs migrated to a new generation of their Story report on the new slot; redriven runs report their reset state"""
    rng = np.random.default_rng(17)
    n = 400
    ts, slots, L, st, h = _batch(fr, rng, 64, A.F_COND | A.F_DECISION | A.F_OUT_FAIL, True, n, dead=0.0)
    slots2 = fr.put_topologies(ts)   # the same Stories as new generations: every step keeps its index
    before = M.status(L, ts, slots, st, n)
    for i in range(ts.count):
        fr.resident_migrate(h, int(slots[i]), int(slots2[i]), np.arange(int(ts.S[i])), n)
    state = fr.resident_download(h, 0, n, L.state_stride)
    assert not np.isin(state[:, :4].copy().view("<u4")[:, 0], slots).any()
    got = fr.resident_status(h, n)
    _same(got, M.status(L, ts, slots2, state, n))
    _same(got, before)
    rq = np.zeros(60, dtype=Frontier.REDRIVE_DTYPE)
    rq["run"] = np.sort(rng.choice(n, size=60, replace=False))
    rq["slot"] = state[rq["run"], :4].copy().view("<u4")[:, 0]
    rq["step"] = np.where(np.arange(60) % 2 == 0, A.REDRIVE_ALL, 0)
    fr.resident_redrive(h, rq)
    state = fr.resident_download(h, 0, n, L.state_stride)
    _same(fr.resident_status(h, n), M.status(L, ts, slots2, state, n))


def test_refusals(fr):
    rng = np.random.default_rng(1)
    n = 50
    ts, slots, L, st, h = _batch(fr, rng, 40, 0, False, n)
    recs = np.zeros(n, dtype=Frontier.STATUS_DTYPE)
    ev = np.zeros(64, dtype=np.uint16)

    def call(handle=h, n_runs=n, runs=None, k=n, records=True, events=True, cap=64, size=None):
        rl = None if runs is None else np.ascontiguousarray(runs, dtype=np.uint32)
        out = A.StatusOut(struct_size=ctypes.sizeof(A.StatusOut) if size is None else size,
                          records=recs.ctypes.data if records else None, events=ev.ctypes.data if events else None, events_cap=cap)
        out.n_events = 12345
        rc = fr._lib.bf_resident_status(fr._ctx, handle, n_runs, None if rl is None else rl.ctypes.data, k, ctypes.byref(out))
        return rc, int(out.n_events)

    for kw in (dict(size=8), dict(handle=h + 5), dict(n_runs=n + 1, k=n + 1), dict(runs=[3, 2], k=2), dict(runs=[2, 2], k=2),
               dict(runs=[1, n], k=2), dict(k=n - 1), dict(records=False), dict(events=False)):
        rc, ne = call(**kw)
        assert rc == A.BF_EINVAL, kw
        assert ne == 12345 and not recs.view(np.uint8).any() and not ev.any(), kw
    assert call(events=False, cap=0)[0] == A.BF_OK
    assert call(runs=[], k=0, records=False)[0] == A.BF_OK
