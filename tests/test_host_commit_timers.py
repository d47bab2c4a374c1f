"""The packing rules of step timings (tests/step_timings.py) on the reference's own inputs and the edge cases of `with`, and the
host model of the arming commit (tests/commit_timers.py) on hand cases.  No GPU."""
import json

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from tests import commit as M
from tests import commit_timers as CT
from tests import timers as T
from tests.step_timings import DurationError, parse_duration, step_timing
from tests.test_host_commit import COND, E, GATE, SLEEP, STOP, WAIT, batch, phases, result

S_NS = 1_000_000_000


def w(**kw):
    return json.dumps(kw)


# ---- packing rules --------------------------------------------------------------------------------------------------------------
def test_reference_inputs():
    """dag_test.go:1322 / 1367 (wait, timeout 1s, onTimeout skip), 1416 / 1480 (sleep 1s), 1447 (sleep 10s)"""
    wait = w(until="{{ inputs.ready }}", timeout="1s", onTimeout="skip")
    assert step_timing(A.STEP_WAIT, wait) == (A.DEC_TIMED_OUT, 1)
    assert step_timing(A.STEP_SLEEP, w(duration="1s")) == (A.DEC_SUCCEED, 1)
    assert step_timing(A.STEP_SLEEP, w(duration="10s")) == (A.DEC_SUCCEED, 10)
    assert step_timing(A.STEP_SLEEP, w(duration="10s"), unit_ns=1_000_000) == (A.DEC_SUCCEED, 10_000)


@pytest.mark.parametrize("raw,ns", [("0", 0), ("0s", 0), ("1500ms", 1_500_000_000), ("1h2m3.5s", 3_723_500_000_000),
                                    ("2µs", 2_000), ("2μs", 2_000), ("2us", 2_000), ("-1s", -S_NS), ("+3m", 180 * S_NS),
                                    (".5s", S_NS // 2), ("1.s", S_NS), ("1.0000000001s", S_NS), ("3ns", 3)])
def test_parse_duration_as_go(raw, ns):
    assert parse_duration(raw) == ns


@pytest.mark.parametrize("raw", ["", "1", "s", ".s", "1x", " 1s", "1s ", "1.2.3s", "-", "9999999999999999999s", "3000000h"])
def test_parse_duration_refuses_as_go(raw):
    with pytest.raises(DurationError):
        parse_duration(raw)


def test_sleep_rules():
    assert step_timing(A.STEP_SLEEP, None) == (A.DEC_SUCCEED, 0)                  # absent: completes on its next sync
    assert step_timing(A.STEP_SLEEP, "") == (A.DEC_SUCCEED, 0)
    assert step_timing(A.STEP_SLEEP, w()) == (A.DEC_SUCCEED, 0)                   # no duration
    assert step_timing(A.STEP_SLEEP, w(duration="  ")) == (A.DEC_SUCCEED, 0)      # blank
    assert step_timing(A.STEP_SLEEP, w(duration="0s")) == (A.DEC_FAIL, 0)         # d <= 0: invalid
    assert step_timing(A.STEP_SLEEP, w(duration="-5s")) == (A.DEC_FAIL, 0)
    assert step_timing(A.STEP_SLEEP, w(duration="1500ms")) == (A.DEC_SUCCEED, 2)  # rounded up: never early
    assert step_timing(A.STEP_SLEEP, w(duration="1h2m3.5s")) == (A.DEC_SUCCEED, 3724)
    assert step_timing(A.STEP_SLEEP, w(duration="2µs")) == (A.DEC_SUCCEED, 1)
    assert step_timing(A.STEP_SLEEP, w(duration="2µs"), unit_ns=1) == (A.DEC_SUCCEED, 2000)
    assert step_timing(A.STEP_SLEEP, w(duration="soon")) == (A.DEC_FAIL, 0)
    assert step_timing(A.STEP_SLEEP, w(duration=5)) == (A.DEC_FAIL, 0)            # not a string: bad JSON for the struct
    assert step_timing(A.STEP_SLEEP, "{") == (A.DEC_FAIL, 0)
    assert step_timing(A.STEP_SLEEP, '{"Duration": "3s"}') == (A.DEC_SUCCEED, 3)  # encoding/json matches keys case-insensitively


def test_gate_rules():
    assert step_timing(A.STEP_GATE, None) is None                                 # the decision arrives as a delta
    assert step_timing(A.STEP_GATE, w()) is None
    assert step_timing(A.STEP_GATE, w(pollInterval="5s")) is None
    assert step_timing(A.STEP_GATE, w(timeout="30s", onTimeout="SKIP")) == (A.DEC_TIMED_OUT, 30)
    assert step_timing(A.STEP_GATE, w(timeout="1500ms")) == (A.DEC_TIMED_OUT, 2)
    for bad in ('{"timeout": 3}', "[1]", w(timeout="0s"), w(timeout="-1s"), w(timeout="x"), w(timeout="1s", pollInterval="0s"),
                w(timeout="1s", onTimeout="retry"), ""):
        assert step_timing(A.STEP_GATE, bad) == (A.DEC_FAIL, 0), bad


def test_wait_rules():
    assert step_timing(A.STEP_WAIT, None) == (A.DEC_FAIL, 0)                       # a wait needs `with`
    assert step_timing(A.STEP_WAIT, w(timeout="5s")) == (A.DEC_FAIL, 0)             # and with.until
    assert step_timing(A.STEP_WAIT, w(until=" ", timeout="5s")) == (A.DEC_FAIL, 0)
    assert step_timing(A.STEP_WAIT, w(until="x", timeout="5s", pollInterval="1s")) == (A.DEC_TIMED_OUT, 5)
    assert step_timing(A.STEP_WAIT, w(until="x", pollInterval="1500ms")) == (A.DEC_PENDING, 2)   # wake-only
    assert step_timing(A.STEP_WAIT, w(until="x")) is None
    for bad in (w(until="x", timeout=""), ):
        assert step_timing(A.STEP_WAIT, bad) is None                                  # an empty timeout is no timeout
    for bad in (w(until="x", timeout="0"), w(until="x", pollInterval="-2s"), w(until="x", onTimeout="later"), "nope"):
        assert step_timing(A.STEP_WAIT, bad) == (A.DEC_FAIL, 0), bad


def test_other_types_have_no_timing():
    for t in (A.STEP_ENGRAM, A.STEP_CONDITION, A.STEP_PARALLEL, A.STEP_STOP, A.STEP_EXECUTE_STORY):
        assert step_timing(t, w(duration="1s", timeout="1s")) is None


# ---- the arming commit --------------------------------------------------------------------------------------------------------------
def setup(types, ph, K=2, fields=A.F_ALL_OUT | A.F_DECISION):
    t, L, st = batch(types, ph, fields)
    return t, L, st, T.empty_area(st.shape[0], K)


def test_a_launched_sleep_pauses_and_arms():
    t, L, st, area = setup([SLEEP, E], [[0, 0]])
    rc, _, _, counts, touched, n, nxt = CT.commit_timed(L, t, {0: {0: (A.DEC_SUCCEED, 7)}}, st, result(L, 1, ready=[0, 1]), None,
                                                        1, (), area, 100, True)
    assert rc == 0 and touched == {0} and counts["n_launched"] == 2 and (n, nxt) == (1, 107)
    assert phases(L, st, 2)[0].tolist() == [A.PHASE_PAUSED, A.PHASE_RUNNING]
    assert T.armed(area[0]) == [(0, 107, A.DEC_SUCCEED)]


def test_arms_merge_in_step_order_and_a_stored_slot_wins():
    t, L, st, area = setup([E, SLEEP, GATE, WAIT, SLEEP], [[0] * 5], K=4)
    area[0] = T.canonical({2: (50, A.DEC_TIMED_OUT), 4: (60, A.DEC_FAIL)}, 4)
    tim = {0: {1: (A.DEC_SUCCEED, 5), 2: (A.DEC_TIMED_OUT, 9), 3: (A.DEC_PENDING, 0)}}
    rc, _, _, _, _, n, nxt = CT.commit_timed(L, t, tim, st, result(L, 1, ready=[0, 1, 2, 3, 4]), None, 1, (), area, 10, True)
    assert rc == 0 and (n, nxt) == (2, 10)   # step 2 is stored (kept, not counted); step 4 has no timing
    assert T.armed(area[0]) == [(1, 15, A.DEC_SUCCEED), (2, 50, A.DEC_TIMED_OUT), (3, 10, A.DEC_PENDING), (4, 60, A.DEC_FAIL)]


def test_hold_error_skip_and_fail_arm_nothing():
    t, L, st, area = setup([SLEEP, GATE, SLEEP, WAIT], [[0] * 4, [0] * 4], K=4)
    tim = {0: {s: (A.DEC_FAIL, 1) for s in range(4)}}
    res = result(L, 2, ready={0: [0, 1, 2, 3], 1: [0, 1]}, skip={0: [2]}, fail={0: [3]})
    ents = [(0, 1, M.HOLD, 0), (1, 0, M.ERROR, 0)]
    rc, _, _, _, touched, n, _ = CT.commit_timed(L, t, tim, st, res, None, 2, ents, area, 0, True)
    assert rc == 0 and n == 1 and touched == {0}
    assert T.armed(area[0]) == [(0, 1, A.DEC_FAIL)] and T.armed(area[1]) == []


def test_not_sync_steps_and_unlaunched_steps_arm_nothing():
    t, L, st, area = setup([COND, E, SLEEP], [[0] * 3])
    assert CT.commit_timed(L, t, {0: {2: (A.DEC_SUCCEED, 3)}}, st, result(L, 1, ready=[0, 1]), None, 1, (), area, 0, True)[5] == 0
    assert T.armed(area[0]) == []


@pytest.mark.parametrize("decision", [True, False])
def test_overflow_and_missing_decision_planes_refuse_at_the_lowest_run_and_step(decision):
    t, L, st, area = setup([SLEEP, GATE, WAIT, STOP], [[0] * 4] * 3, K=1)
    area[1] = T.canonical({3: (9, A.DEC_PENDING)}, 1)
    tim = {0: {0: (A.DEC_SUCCEED, 1), 1: (A.DEC_TIMED_OUT, 1), 2: (A.DEC_PENDING, 1)}}
    res = result(L, 3, ready={0: [2], 1: [0, 2], 2: [1, 2]})
    st0, a0 = st.copy(), area.copy()
    rc, br, bs, *_ = CT.commit_timed(L, t, tim, st, res, None, 3, (), area, 0, decision)
    if decision:   # run 0 arms one wake-only slot; run 1 holds one and would arm two more: overflow at its lowest new step
        assert (rc, br, bs) == (CT.ENOMEM, 1, 0)
    else:          # run 1's step 0 writes a code on a batch without decision planes (it wins the tie with the overflow)
        assert (rc, br, bs) == (M.EINVAL, 1, 0)
    assert np.array_equal(st, st0) and np.array_equal(area, a0)
    # an entry offence at the same (run, step) wins over the arming offence
    rc, br, bs, *_ = CT.commit_timed(L, t, tim, st, res, None, 3, [(1, 0, M.PHASE, A.PHASE_SUCCEEDED)], area, 0, decision)
    assert (rc, br, bs) == (M.EINVAL, 1, 0)
    # a lower entry offence wins outright
    rc, br, bs, *_ = CT.commit_timed(L, t, tim, st, res, None, 3, [(0, 3, M.HOLD, 0)], area, 0, decision)
    assert (rc, br, bs) == (M.EINVAL, 0, 3)
    assert np.array_equal(st, st0) and np.array_equal(area, a0)


def test_wake_only_timing_needs_no_decision_planes():
    t, L, st, area = setup([WAIT], [[0]], fields=A.F_ALL_OUT)
    rc, _, _, _, _, n, nxt = CT.commit_timed(L, t, {0: {0: (A.DEC_PENDING, 4)}}, st, result(L, 1, ready=[0]), None, 1, (), area, 6, False)
    assert rc == 0 and (n, nxt) == (1, 10)


def test_deadline_saturates_below_none():
    t, L, st, area = setup([SLEEP, GATE], [[0, 0]])
    tim = {0: {0: (A.DEC_SUCCEED, 0xFFFFFFFF), 1: (A.DEC_TIMED_OUT, 5)}}
    rc, _, _, _, _, n, nxt = CT.commit_timed(L, t, tim, st, result(L, 1, ready=[0, 1]), None, 1, (), area, T.NONE - 3, True)
    assert rc == 0 and (n, nxt) == (2, T.NONE - 1)
    assert T.armed(area[0]) == [(0, T.NONE - 1, A.DEC_SUCCEED), (1, T.NONE - 1, A.DEC_TIMED_OUT)]


def test_arm_requests_are_what_the_timed_commit_arms():
    """the two-call form of the loop (commit, then bf_resident_timers_arm with these requests) arms the same slots"""
    from bobrapet_b200.frontier import Frontier
    t, L, st, area = setup([SLEEP, GATE, WAIT, E], [[0] * 4] * 2, K=3)
    area[1] = T.canonical({1: (3, A.DEC_TIMED_OUT)}, 3)
    tim = {0: {0: (A.DEC_SUCCEED, 2), 1: (A.DEC_TIMED_OUT, 4), 2: (A.DEC_PENDING, 1)}}
    res = result(L, 2, ready={0: [0, 1, 2, 3], 1: [0, 1]})
    b_st, b_area = st.copy(), area.copy()
    req = CT.arm_requests(L, t, tim, st, res, None, 2, (), area, 20, Frontier.TIMER_DTYPE)
    assert CT.commit_timed(L, t, tim, st, res, None, 2, (), area, 20, True)[0] == 0
    assert M.commit(L, t, b_st, res, None, 2)[0] == 0 and T.arm(b_area, L, req) == 0
    assert np.array_equal(st, b_st) and np.array_equal(area, b_area)
