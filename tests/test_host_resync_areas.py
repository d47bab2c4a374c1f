"""The host model of bf_resident_resync_areas (tests/resync_areas.py) against the rules of its header section: refusals, a lifecycle
resynced against what its batcher persisted, the taken-as-fired rule, and the stops a resync lists, keeps or applies."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import make_layout
from tests import lifecycle as LC
from tests import resync_areas as M
from tests import runctl as R
from tests import timers as T

NOW = 1000
S = (40, 24)


def _batch(subset=LC.TIMERS | LC.SCHED | LC.RUNCTL, K=4, n=24):
    L = make_layout(64, 0, A.F_COND | A.F_DECISION)
    recs = LC.records_of(LC.template_records(L, [0, 1], S), n)
    b, _ = LC.seeded(L, n + 4, subset, K, recs, S[1] - 1, NOW)
    return b


def _set_dec(b, r, s, code):
    T._set(b.state[r], b.L.off_decision, b.L.words, 2, s, code)


def _row(K, entries):
    """a canonical caller timer row from {step: (deadline, code)}"""
    return T.canonical(entries, K).view(M.SLOT_DTYPE)


def test_own_areas_list_nothing():
    b = _batch()
    n = b.n
    t, s, c = M.device_areas(b)
    got = M.resync(b, n, timers=t, sched=s, runctl=c, check=True)
    assert got["status"] == 0 and got["items"].size == 0 and got["drifted"].size == 0


@pytest.mark.parametrize("seed", range(4))
def test_lifecycle_against_what_the_batcher_persisted_lists_nothing(seed):
    """the batcher keeps a fired slot until its step is terminal and a fired drain deadline until it persists the force-delete,
    and persists the stops the fire listed: with fired_now the device's disarmed slots and deadlines are equal"""
    rng = np.random.default_rng(seed)
    b = _batch()
    n = b.n
    arms = []
    for r in range(n):
        for st in rng.choice(np.arange(5, 40), size=2, replace=False):
            arms.append((r, int(st), int(rng.integers(0, 4)), 0, NOW + int(rng.integers(0, 60)), 0))
    arms = np.array(arms, np.dtype([("run", "<u4"), ("step", "<u2"), ("code", "u1"), ("reserved", "u1"), ("deadline", "<u4"),
                                    ("reserved2", "<u4")]))
    T.arm(b.timers, b.L, [q for q in arms if len(T.armed(b.timers[int(q["run"])])) < b.K - 1])
    for now in (NOW + 20, NOW + 45):
        kept_t, _, kept_c = M.device_areas(b)
        R.fire(b.runctl, b.L, b.state, b.timers, n, now, b.inputs)
        _, s, c = M.device_areas(b)
        c["drain_deadline"] = kept_c["drain_deadline"]   # not yet persisted as fired
        got = M.resync(b, n, timers=kept_t, sched=s, runctl=c, fired_now=now, check=True)
        assert got["items"].size == 0, got["items"][:6]


def test_taken_as_fired():
    b = _batch()
    r, s, K = 0, 7, b.K
    b.timers[r] = T.canonical({}, K)
    _, sched, ctl = M.device_areas(b, runs=[r])
    for code in (A.DEC_SUCCEED, A.DEC_PENDING):
        row = _row(K, {s: (NOW, code)})[None, :]
        for dec in (A.DEC_PENDING, A.DEC_SUCCEED):
            _set_dec(b, r, s, dec)
            for fired_now, want in ((M.NONE, True), (NOW - 1, True), (NOW, code != A.DEC_PENDING and dec == A.DEC_PENDING)):
                got = M.resync(b, b.n, runs=[r], timers=row, fired_now=fired_now, check=True)
                assert (got["items"].size == 1) == want, (code, dec, fired_now, got["items"])
                if want:
                    assert got["items"][0].tolist() == (r, s, A.DRIFT_TIMER, 0, M.NONE, NOW)
    # the stuck step: repaired, the next fire fires it
    _set_dec(b, r, s, A.DEC_PENDING)
    row = _row(K, {s: (NOW, A.DEC_SUCCEED), 20: (NOW - 5, A.DEC_PENDING)})[None, :]
    got = M.resync(b, b.n, runs=[r], timers=row, fired_now=NOW)
    assert got["n_written"] == 1 and [int(x) for x in got["items"]["index"]] == [s]
    assert T.armed(b.timers[r]) == [(s, NOW, A.DEC_SUCCEED)]   # the wake-only slot taken as fired is not re-armed
    fired = T.fire(b.timers[r:r + 1], b.L, b.state[r:r + 1], 1, NOW)
    assert fired["fired"] == [(0, s, A.DEC_SUCCEED, 1)] and T.decision(b.L, b.state[r], s) == A.DEC_SUCCEED
    assert M.resync(b, b.n, runs=[r], timers=row, fired_now=NOW, check=True)["items"].size == 0


def test_terminal_steps_and_items_order():
    b = _batch()
    r, K = 1, b.K
    b.timers[r] = T.canonical({2: (5, 1), 9: (50, 1), 12: (60, 0)}, K)   # step 2 is Succeeded (terminal)
    row = _row(K, {3: (7, 0), 9: (51, 3), 12: (60, 1), 30: (70, 0)})[None, :]   # step 3 is terminal too
    got = M.resync(b, b.n, runs=[r], timers=row, check=True)
    want = [(r, 9, A.DRIFT_TIMER, 0, 50, 51), (r, 30, A.DRIFT_TIMER, 0, M.NONE, 70),
            (r, 9, A.DRIFT_TIMER_CODE, 0, 1, 3), (r, 12, A.DRIFT_TIMER_CODE, 0, 0, 1)]
    assert [x.tolist() for x in got["items"]] == want
    M.resync(b, b.n, runs=[r], timers=row)
    assert T.armed(b.timers[r]) == [(3, 7, 0), (9, 51, 3), (12, 60, 1), (30, 70, 0)]


def test_device_stop_is_listed_and_kept():
    b = _batch()
    r = 3   # seeded stopped (r % 4 == 3)
    assert b.runctl["stop"][r]
    t, s, c = M.device_areas(b, runs=[r])
    before = (b.state.copy(), b.runctl.copy(), b.timers.copy())
    for stop in (R.STOP_NONE, R.STOP_CANCEL if b.runctl["stop"][r] != R.STOP_CANCEL else R.STOP_HOST):
        c["stop"] = stop
        t2 = _row(b.K, {30: (NOW, 0)})[None, :]   # a stopped run compares no timers
        got = M.resync(b, b.n, runs=[r], timers=t2, sched=s, runctl=c)
        assert [x.tolist() for x in got["items"]] == [(r, 0, A.DRIFT_STOP, 0, int(before[1]["stop"][r]), stop)]
        assert got["n_written"] == 0 and got["stopped"] == []
        assert b.state.tobytes() == before[0].tobytes() and b.runctl.tobytes() == before[1].tobytes()
        assert b.timers.tobytes() == before[2].tobytes()


def test_caller_stop_empties_timers_and_writes_timeout():
    b = _batch()
    r = 5   # seeded with armed slots and a story deadline, not stopped
    assert not b.runctl["stop"][r] and T.armed(b.timers[r])
    t, s, c = M.device_areas(b, runs=[r])
    own = int(b.state[r][4])
    c["stop"] = R.STOP_TIMEOUT
    t[0] = _row(b.K, {30: (NOW, 0)})   # not compared: the caller's stop empties the timers
    got = M.resync(b, b.n, runs=[r], timers=t, sched=s, runctl=c)
    assert [x.tolist() for x in got["items"]] == [(r, 0, A.DRIFT_STOP, 0, 0, R.STOP_TIMEOUT)]
    assert got["n_written"] == 1 and got["stopped"] == [r]
    assert not T.armed(b.timers[r]) and b.inputs["run_phase"][r] == R.PHASE_TIMEOUT
    assert b.runctl["stop"][r] == R.STOP_TIMEOUT and b.runctl["saved_flags"][r] == own and b.state[r][4] == R.STOPPED_FLAGS


def test_sched_and_deadlines_repair():
    b = _batch()
    r = 8
    _, s, c = M.device_areas(b, runs=[r])
    s["priority"][0] = -7
    s["run_phase"][0] = A.PHASE_SUCCEEDED
    c["story_deadline"][0] = NOW + 3
    c["drain_deadline"][0] = NOW - 2   # the device has none: taken as fired at fired_now >= NOW - 2
    got = M.resync(b, b.n, runs=[r], sched=s, runctl=c, fired_now=NOW - 3, check=True)
    assert [int(x) for x in got["items"]["field"]] == [A.DRIFT_SCHED_PRIORITY, A.DRIFT_SCHED_RUN_PHASE, A.DRIFT_STORY_DEADLINE,
                                                       A.DRIFT_DRAIN_DEADLINE]
    assert got["items"][0]["record"] == 0xFFFFFFF9
    got = M.resync(b, b.n, runs=[r], sched=s, runctl=c, fired_now=NOW)
    assert [int(x) for x in got["items"]["field"]] == [A.DRIFT_SCHED_PRIORITY, A.DRIFT_SCHED_RUN_PHASE, A.DRIFT_STORY_DEADLINE]
    assert b.inputs["priority"][r] == -7 and b.runctl["story_deadline"][r] == NOW + 3 and b.runctl["drain_deadline"][r] == M.NONE


def _refusals(b):
    """(description, kwargs of M.resync / the call, expected bad_run) of every refusal the header names"""
    n, K = b.n, b.K
    t, s, c = M.device_areas(b)
    out = [("n_runs above the capacity", dict(n_runs=b.cap + 1, timers=None), M.NONE),
           ("runs not ascending", dict(runs=[3, 2], timers=t[:2]), M.NONE),
           ("a run at n_runs", dict(runs=[n], timers=t[:1]), M.NONE)]
    bad = t.copy()
    bad[4][0], bad[4][1] = bad[4][1], bad[4][0]
    if T.armed(b.timers[4])[1:]:
        out.append(("slots not ascending", dict(timers=bad), 4))
    for name, edit in (("a repeated step", lambda row: row.__setitem__(1, row[0])),
                       ("a step at steps_max", lambda row: row.__setitem__(0, (1, b.L.steps_max, 0, 0))),
                       ("a code above 3", lambda row: row.__setitem__(0, (1, 30, 4, 0))),
                       ("a reserved byte", lambda row: row.__setitem__(0, (1, 30, 0, 1))),
                       ("an empty slot's bytes", lambda row: row.__setitem__(K - 1, (M.NONE, 3, 0, 0))),
                       ("an armed slot after an empty one", lambda row: row.__setitem__(K - 1, (5, 63, 0, 0)))):
        bad = t.copy()
        row = bad[9]
        row[:] = _row(K, {30: (NOW, 0)})
        edit(row)
        out.append((name, dict(timers=bad), 9))
    bad = s.copy()
    bad["run"][6] = 7
    out.append(("a sched row of another run", dict(sched=bad), 6))
    bad = s.copy()
    bad["reserved"][11, 1] = 1
    out.append(("a sched reserved word", dict(sched=bad), 11))
    for name, field, val in (("a stop above HOST", "stop", 4), ("saved_flags", "saved_flags", 1)):
        bad = c.copy()
        bad[field][2] = val
        out.append((name, dict(runctl=bad), 2))
    bad = c.copy()
    bad["reserved"][13, 5] = 1
    out.append(("a run-control reserved byte", dict(runctl=bad), 13))
    return out


def test_refusals_change_nothing():
    b = _batch()
    snap = (b.state.copy(), b.timers.copy(), b.inputs.copy(), b.runctl.copy())
    for name, kw, want in _refusals(b):
        kw = dict(kw)
        n_runs = kw.pop("n_runs", b.n)
        got = M.resync(b, n_runs, **kw)
        assert got["status"] == M.EINVAL and got["bad_run"] == want, name
    L = make_layout(64, 0, A.F_COND)
    no_decision = LC.AreaBatch(L, 8, LC.TIMERS, 4)
    no_decision.upload(0, LC.records_of(LC.template_records(L, [0, 1], S), 6))
    t, _, _ = M.device_areas(no_decision)
    t[0] = _row(no_decision.K, {30: (NOW, A.DEC_SUCCEED)})
    assert M.resync(no_decision, no_decision.n, timers=t)["bad_run"] == 0
    for subset in (LC.SCHED | LC.RUNCTL, LC.TIMERS | LC.RUNCTL, LC.TIMERS | LC.SCHED):   # a selected area the batch lacks
        lack = _batch(subset)
        own = _batch()
        t, s, c = M.device_areas(own)
        assert M.resync(lack, lack.n, timers=t, sched=s, runctl=c)["bad_run"] == M.NONE
    assert M.refusal(b, b.n, None, b.n, 0x8, 0) == M.NONE
    assert M.refusal(b, b.n, None, b.n, 0, 0x2) == M.NONE
    assert M.refusal(b, b.n, None, b.n, A.RESYNC_AREA_TIMERS, 0) == M.NONE   # a NULL array of a selected area
    assert M.refusal(b, b.n, None, b.n - 1, 0, 0) == M.NONE                   # runs == NULL needs n == n_runs
    assert (b.state.tobytes(), b.timers.tobytes(), b.inputs.tobytes(), b.runctl.tobytes()) == tuple(x.tobytes() for x in snap)
