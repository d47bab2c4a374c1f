"""tests/timers.py, the host model of a resident batch's step timers, pinned by known answers taken from the reference's timer
handling (dag.go checkSyncSleepSteps, the gate and wait timeouts, pruneTerminal; storyrun_controller.go's redrive patches).  No
GPU: these define what tests/test_gpu_timers.py compares the device with."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import timers as T

REQ = Frontier.TIMER_DTYPE


def _req(*rows):
    """(run, step, code, deadline) rows -> bf_timer requests"""
    out = np.zeros(len(rows), dtype=REQ)
    for i, (run, step, code, deadline) in enumerate(rows):
        out[i]["run"], out[i]["step"], out[i]["code"], out[i]["deadline"] = run, step, code, deadline
    return out


def _batch(n=4, S=64, fields=A.F_DECISION, K=4):
    L = make_layout(S, 0, fields)
    state = np.zeros((n, L.state_stride), dtype=np.uint8)
    for r in range(n):
        for s in range(S):
            T._set(state[r], L.off_phase, L.words, 4, s, A.PHASE_RUNNING)
    return L, state, T.empty_area(n, K)


def test_due_exactly_at_the_deadline():
    """remaining <= 0 fires a sleep (dag.go:1266): deadline == now is due, now = deadline - 1 is not"""
    L, st, area = _batch()
    assert T.arm(area, L, _req((1, 3, A.DEC_SUCCEED, 100))) == 0
    out = T.fire(area, L, st, 4, 99)
    assert out["n_fired"] == 0 and out["next_deadline"] == 100 and T.armed(area[1]) == [(3, 100, A.DEC_SUCCEED)]
    out = T.fire(area, L, st, 4, 100)
    assert out["fired"] == [(1, 3, A.DEC_SUCCEED, 1)] and out["touched"] == {1} and out["next_deadline"] == T.NONE
    assert T.decision(L, st[1], 3) == A.DEC_SUCCEED and T.armed(area[1]) == []


def test_an_approved_gate_stays_approved_when_its_timeout_is_due():
    """an approve already delivered takes precedence over the timeout (dag.go:1501-1533)"""
    L, st, area = _batch()
    T._set(st[2], L.off_decision, L.words, 2, 7, A.DEC_SUCCEED)
    T.arm(area, L, _req((2, 7, A.DEC_TIMED_OUT, 50)))
    before = st.copy()
    out = T.fire(area, L, st, 4, 60)
    assert out["fired"] == [(2, 7, A.DEC_TIMED_OUT, 0)] and out["n_written"] == 0 and not out["touched"]
    assert np.array_equal(st, before) and T.decision(L, st[2], 7) == A.DEC_SUCCEED


def test_a_timer_on_a_terminal_step_is_pruned_before_it_is_due():
    """pruneTerminal (dag.go:173-190): a terminal step's timer goes whatever its deadline"""
    L, st, area = _batch()
    T._set(st[0], L.off_phase, L.words, 4, 5, A.PHASE_SUCCEEDED)
    T.arm(area, L, _req((0, 5, A.DEC_TIMED_OUT, 1000), (0, 9, A.DEC_TIMED_OUT, 2000)))
    out = T.fire(area, L, st, 4, 10)
    assert out["n_pruned"] == 1 and out["n_fired"] == 0 and out["next_deadline"] == 2000
    assert T.armed(area[0]) == [(9, 2000, A.DEC_TIMED_OUT)]


def test_a_wake_only_timer_is_listed_and_writes_nothing():
    """a wait step's pollInterval (dag.go:1440): reported when due, the host re-evaluates `until` itself"""
    L, st, area = _batch(fields=0)
    assert T.arm(area, L, _req((3, 1, A.DEC_PENDING, 5))) == 0
    assert T.arm(area, L, _req((3, 2, A.DEC_TIMED_OUT, 5))) == T.EINVAL   # a code that writes needs decision planes
    before = st.copy()
    out = T.fire(area, L, st, 4, 5)
    assert out["fired"] == [(3, 1, A.DEC_PENDING, 0)] and not out["touched"] and np.array_equal(st, before)


def test_a_redrive_from_a_step_clears_every_timer_of_the_run():
    """both redrive patches delete the whole step-timers annotation (storyrun_controller.go:477-478, :524-525)"""
    L, st, area = _batch()
    T.arm(area, L, _req((1, 2, A.DEC_SUCCEED, 10), (1, 40, A.DEC_TIMED_OUT, 20), (2, 3, A.DEC_SUCCEED, 30)))
    rq = np.zeros(2, dtype=Frontier.REDRIVE_DTYPE)
    rq[0]["run"], rq[0]["step"] = 1, 39       # from step 39: the reset set does not hold step 2
    rq[1]["run"], rq[1]["step"] = 2, 0        # stale: status 0
    area = T.redrive(area, rq, [1, 0])
    assert T.armed(area[1]) == [] and T.armed(area[2]) == [(3, 30, A.DEC_SUCCEED)]


def test_arm_replaces_cancels_and_keeps_the_slots_sorted():
    L, st, area = _batch(K=3)
    T.arm(area, L, _req((0, 9, 1, 90), (0, 2, 3, 20)))
    assert T.armed(area[0]) == [(2, 20, 3), (9, 90, 1)]
    T.arm(area, L, _req((0, 9, 3, 95), (0, 5, 1, 50), (0, 2, 0, T.NONE)))
    assert T.armed(area[0]) == [(5, 50, 1), (9, 95, 3)]
    assert area[0][2] == T.EMPTY


def test_arm_refusals_change_nothing():
    L, st, area = _batch(K=2)
    T.arm(area, L, _req((1, 1, 1, 10), (1, 2, 1, 10)))
    before = area.copy()
    assert T.check_arm(area, L, _req((1, 3, 1, 10))) == (T.ENOMEM, 1)
    assert T.arm(area, L, _req((1, 3, 1, 10), (1, 1, 0, T.NONE))) == 0   # a cancel in the same call makes room
    area[:] = before
    for bad in (_req((4, 0, 1, 1)), _req((0, 64, 1, 1)), _req((0, 0, 4, 1)), _req((0, 0, 1, 1), (0, 0, 2, 2))):
        assert T.arm(area, L, bad) == T.EINVAL
    r = _req((0, 0, 1, 1))
    r[0]["reserved2"] = 1
    assert T.arm(area, L, r) == T.EINVAL and np.array_equal(area, before)


def test_retire_migrate_transfer_and_extent_re_key_the_slots():
    L, st, area = _batch(n=6, K=2)
    T.arm(area, L, _req((1, 4, 1, 10), (4, 6, 3, 40), (5, 1, 0, 50), (5, 9, 2, 55)))
    m, moves = T.retire_moves(6, [1, 2])
    assert m == 4 and moves == {4: 1, 5: 2}
    ra = T.retire(area, 6, [1, 2])
    assert T.armed(ra[1]) == [(6, 40, 3)] and T.armed(ra[2]) == [(1, 50, 0), (9, 55, 2)] and T.armed(ra[4]) == T.armed(ra[5]) == []
    mg = T.migrate(area, [5], np.array([T.MIGRATE_GONE, 12, 3, 4, 5, 6, 7, 8, 9, 0], np.uint16))
    assert T.armed(mg[5]) == [(0, 55, 2), (12, 50, 0)]
    assert not T.fits(area, 5, 1) and T.fits(area, 4, 1) and T.fits(None, 5, 0)
    src, dst = T.transfer(area, T.empty_area(3, 1), 6, 1, [4])
    assert T.armed(dst[1]) == [(6, 40, 3)] and T.armed(src[4]) == [(1, 50, 0), (9, 55, 2)] and T.armed(src[5]) == []
    assert T.extent(area) == (10, T.F_DECISION, 5)
    assert T.reshape(area, 9).shape == (9, 2) and T.grow(area, 5)[5, 1] == area[5, 1]
