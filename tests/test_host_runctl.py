"""The host model of StoryRun stops and deadlines (tests/runctl.py) against known answers from the reference: the story timeout
of enforceStoryTimeout (dag.go:544-578, checked before the step syncs :393-420), the redrive resets of storyrun_controller.go
(resetStoryRunForRedrive :414-438 clears StartedAt, resetStoryRunForStepRedrive keeps it) and the graceful-cancel drain
deadline of handleGracefulCancel (:1517-1578)."""
from types import SimpleNamespace

import numpy as np

from tests import runctl as R
from tests import timers as T

# one word of steps: phase planes at 16, decision planes at 32, 48-byte records
L = SimpleNamespace(words=1, off_phase=16, off_decision=32, steps_max=32, state_stride=48)
RUNNING = 2
FLAGS = 0x01 | 0x04   # FAIL_FAST | TOPOLOGY_TERMINATED


def batch(n=2, flags=FLAGS):
    state = np.zeros((n, L.state_stride), dtype=np.uint8)
    for r in range(n):
        state[r][4] = flags
        for s in range(4):
            T._set(state[r], L.off_phase, L.words, 4, s, RUNNING)
    return state, R.defaults(n)


def put(area, state, run, story=R.NONE, drain=R.NONE, stop=0, timers=None, sched=None):
    q = np.zeros(1, dtype=R.PUT_DTYPE)
    q[0] = (run, story, drain, stop, (0, 0, 0))
    return R.put(area, state, q, timers, sched)


def test_story_timeout_is_due_exactly_at_the_deadline():
    state, area = batch()
    put(area, state, 0, story=100)
    out = R.fire(area, L, state, None, 2, 99)
    assert out["n_fired"] == 0 and out["next_deadline"] == 100 and not area["stop"][0]
    out = R.fire(area, L, state, None, 2, 100)
    assert out["fired"] == [(0, R.FIRED_STORY, R.DEC_TIMED_OUT, 1)]
    assert out["n_written"] == 1 and out["touched"] == {0}
    assert area["stop"][0] == R.STOP_TIMEOUT and area["saved_flags"][0] == FLAGS and state[0][4] == R.STOPPED_FLAGS
    assert out["next_deadline"] == R.NONE   # the stopped run's story deadline is dormant
    assert area["story_deadline"][0] == 100


def test_story_timeout_precedes_a_due_sleep():
    state, area = batch()
    timers = T.empty_area(2, 4)
    rq = np.zeros(2, dtype=[("run", "<u4"), ("step", "<u2"), ("code", "u1"), ("reserved", "u1"), ("deadline", "<u4"),
                            ("reserved2", "<u4")])
    rq[0] = (0, 1, 1, 0, 50, 0)    # a sleep of step 1, due
    rq[1] = (0, 2, 3, 0, 900, 0)   # a gate timeout of step 2, not due
    assert T.arm(timers, L, rq) == 0
    put(area, state, 0, story=50)
    sched = np.zeros(2, dtype=[("run", "<u4"), ("run_phase", "<u4")])
    out = R.fire(area, L, state, timers, 2, 50, sched)
    assert out["fired"] == [(0, R.FIRED_STORY, R.DEC_TIMED_OUT, 1)]
    assert out["n_pruned"] == 2 and out["n_written"] == 1
    assert T.decision(L, state[0], 1) == R.DEC_PENDING   # the sleep wrote nothing
    assert all(v == T.EMPTY for v in timers[0])
    assert sched["run_phase"][0] == R.PHASE_TIMEOUT and sched["run_phase"][1] == 0


def test_a_step_redrive_of_a_timed_out_run_times_out_again():
    state, area = batch()
    put(area, state, 0, story=10)
    R.fire(area, L, state, None, 1, 20)
    state[0][4] &= ~R.RF_TOPOLOGY_TERMINATED & 0xFF   # the record reset of the redrive
    rq = np.array([(0, 0, 2, 0)], dtype=[("run", "<u4"), ("slot", "<u4"), ("step", "<u4"), ("reserved", "<u4")])
    R.redrive(area, state, rq, [1])
    assert not area["stop"][0] and state[0][4] == FLAGS & ~R.RF_TOPOLOGY_TERMINATED
    assert area["story_deadline"][0] == 10   # StartedAt kept
    out = R.fire(area, L, state, None, 1, 21)
    assert out["fired"] == [(0, R.FIRED_STORY, R.DEC_TIMED_OUT, 1)] and area["stop"][0] == R.STOP_TIMEOUT


def test_a_full_redrive_does_not_time_out_again():
    state, area = batch()
    put(area, state, 0, story=10, drain=500)
    R.fire(area, L, state, None, 1, 20)
    rq = np.array([(0, 0, R.REDRIVE_ALL, 0)], dtype=[("run", "<u4"), ("slot", "<u4"), ("step", "<u4"), ("reserved", "<u4")])
    R.redrive(area, state, rq, [1])
    assert state[0][4] == FLAGS & ~R.RF_TOPOLOGY_TERMINATED   # the original byte, without TOPOLOGY_TERMINATED
    assert area[0].tobytes() == R.defaults(1)[0].tobytes()   # StartedAt = nil; the drain deadline goes too
    out = R.fire(area, L, state, None, 1, 10_000)
    assert out["n_fired"] == 0 and out["next_deadline"] == R.NONE


def test_a_drain_deadline_is_wake_only():
    state, area = batch()
    before = state.copy()
    put(area, state, 1, drain=30, stop=R.STOP_CANCEL)
    assert state[1][4] == R.STOPPED_FLAGS and area["saved_flags"][1] == FLAGS
    out = R.fire(area, L, state, None, 2, 29)
    assert out["n_fired"] == 0 and out["next_deadline"] == 30
    out = R.fire(area, L, state, None, 2, 30)
    assert out["fired"] == [(1, R.FIRED_DRAIN, R.DEC_PENDING, 0)]
    assert out["n_written"] == 0 and not out["touched"] and out["next_deadline"] == R.NONE
    assert area["drain_deadline"][1] == R.NONE
    assert np.array_equal(state[0], before[0])


def test_a_run_flags_delta_to_a_stopped_run_changes_only_saved_flags():
    state, area = batch()
    put(area, state, 0, stop=R.STOP_HOST)
    ds = np.zeros(2, dtype=[("run", "<u4"), ("index", "<u2"), ("field", "u1"), ("code", "u1")])
    ds[0] = (0, 0, 4, 0x02)
    ds[1] = (1, 0, 4, 0x02)
    rest = R.deltas(area, state, ds)
    assert len(rest) == 1 and rest[0]["run"] == 1
    assert state[0][4] == R.STOPPED_FLAGS and area["saved_flags"][0] == 0x02


def test_a_second_stop_keeps_the_first_reason():
    state, area = batch()
    put(area, state, 0, stop=R.STOP_CANCEL)
    rc, touched = put(area, state, 0, story=5, stop=R.STOP_TIMEOUT)
    assert rc == 0 and not touched
    assert area["stop"][0] == R.STOP_CANCEL and area["saved_flags"][0] == FLAGS
    out = R.fire(area, L, state, None, 1, 100)   # a stopped run's story deadline never fires
    assert out["n_fired"] == 0
    rc, _ = put(area, state, 0, stop=R.STOP_NONE)   # a put cannot un-stop
    assert rc == 0 and area["stop"][0] == R.STOP_CANCEL


def test_put_refusals():
    state, area = batch()
    q = np.zeros(2, dtype=R.PUT_DTYPE)
    q[0] = (0, 1, 1, 0, (0, 0, 0))
    q[1] = (0, 2, 2, 0, (0, 0, 0))
    assert R.put(area, state, q)[0] == R.EINVAL               # one request per run
    q[1] = (1, 2, 2, 4, (0, 0, 0))
    assert R.put(area, state, q)[0] == R.EINVAL               # stop > BF_STOP_HOST
    q[1] = (1, 2, 2, 0, (0, 1, 0))
    assert R.put(area, state, q)[0] == R.EINVAL               # reserved
    q[1] = (2, 2, 2, 0, (0, 0, 0))
    assert R.put(area, state, q)[0] == R.EINVAL               # run outside the capacity
    assert R.put(None, state, q[:1])[0] == R.EINVAL           # no area
    assert area.tobytes() == R.defaults(2).tobytes()


def test_upload_keeps_the_stop_and_retire_moves_records():
    state, area = batch(4)
    put(area, state, 3, story=7, stop=R.STOP_CANCEL)
    fresh = np.zeros((4, L.state_stride), dtype=np.uint8)
    fresh[:, 4] = 0x02
    R.upload(area, state, 0, fresh)
    assert state[3][4] == R.STOPPED_FLAGS and area["saved_flags"][3] == 0x02 and state[0][4] == 0x02
    out = R.retire(area, 4, [1])
    assert out[1].tobytes() == area[3].tobytes() and out[3].tobytes() == R.defaults(1)[0].tobytes()
    assert not R.fits(area, None, 3) and R.fits(area, None, 0)
