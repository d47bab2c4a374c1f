"""The host model of bf_resident_status (tests/runstatus.py) against the object-shaped restatement of the reference: finalizeStoryRun
and summarizeStepProgress (tests/finalize.py) over pyoracle's loop body, pinned by the reference's own vectors, then on random
Stories and StoryRuns packed with tests/packing.py."""
import collections
import random

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import make_layout, pack_state
from oracle import pyoracle as O
from tests import finalize as F
from tests import packing as P
from tests import runctl as R
from tests import runstatus as M
from tests.test_oracle_differential import _clone_run, _evaluator, _rand_run, _rand_story

OUTCOME = {("Failed", "CleanupFailed"): A.OUTCOME_CLEANUP_FAILED, ("Failed", "CompensationFailed"): A.OUTCOME_COMPENSATION_FAILED,
           ("Compensated", "Compensated"): A.OUTCOME_COMPENSATED, ("Failed", "DependencyFailed"): A.OUTCOME_DEPENDENCY_FAILED,
           ("Succeeded", ""): A.OUTCOME_SUCCEEDED}


def _chain(phases, fail_fast=True):
    """SURVEY.md 8.2: `A; B needs [A]; C needs [B]`, all engram steps"""
    story = O.Story([O.Step("A", ref=True), O.Step("B", ref=True, needs=["A"]), O.Step("C", ref=True, needs=["B"])], [], [],
                    continue_on_step_failure=None if fail_fast else True)
    srun = O.StoryRun()
    for n, ph in zip("ABC", phases):
        if ph:
            srun.step_states[n] = O.StepState(ph)
    return story, srun


def test_finalize_compensated():
    """dag_test.go:154 TestFinalizeStoryRunCompensated: a failed main step with compensations -> Compensated"""
    story = O.Story([O.Step("main", ref=True)], [O.Step("rollback", ref=True)], [])
    phase, reason, _msg, listed = F.finalize_story_run(story, {"main": O.StepState("Failed")}, {"main": True}, {}, {})
    assert (phase, reason) == ("Compensated", "Compensated") and listed == {"main": "Failed"}


def test_finalize_all_succeeded():
    """8.2: `Succeeded Succeeded Succeeded` -> group done, finalize Succeeded (dag.go:725-752)"""
    story, srun = _chain(["Succeeded"] * 3)
    it = O.run_dag_iteration(srun, story)
    assert it.group == "finalize"
    assert F.finalize_story_run(story, srun.step_states, *F.failed_sets(story, srun.step_states))[:2] == ("Succeeded", "")
    assert F.summarize_step_progress(srun.step_states) == (0, 3, 0, 0)


def test_finalize_fail_fast():
    """8.2: `Failed "" ""` with failFast: B, C Skipped by fail-fast, group done, StoryRun Failed / DependencyFailed naming A"""
    story, srun = _chain(["Failed", "", ""])
    it = O.run_dag_iteration(srun, story)
    assert it.group == "finalize"
    phase, reason, msg, listed = F.finalize_story_run(story, srun.step_states, *F.failed_sets(story, srun.step_states))
    assert (phase, reason) == ("Failed", "DependencyFailed") and msg == "Story completed with failed step: A." and listed == {"A": "Failed"}
    assert F.summarize_step_progress(srun.step_states) == (0, 0, 1, 2)
    # the same run packed: the model reports the pass's rewrites (B, C Skipped) and the finalize of that state
    ps = P.pack_story(story)
    L, st = P.pack_runs([story], [ps], [_chain(["Failed", "", ""])[1]], [0], [0])
    recs, ev, n = M.status(L, P.topology_set([ps]), [0], st, 1)
    r = recs[0]
    assert (r["group"], r["outcome"], r["story_phase"], r["first_failed"]) == (A.GROUP_DONE, A.OUTCOME_DEPENDENCY_FAILED, A.PHASE_FAILED, 0)
    assert (r["active"], r["completed"], r["failed"], r["skipped"]) == (0, 0, 1, 2)
    assert n == 1 and ev.tolist() == [0 | A.PHASE_FAILED << 10 | A.STATUS_EVT_FAILED << 14]


def test_cond_fail_is_not_reported():
    """A step the pass fails by its cond code (stage D) is written only by a commit: the report keeps its input code"""
    ts = TopologySet([2], [0], np.zeros(3, np.uint32), np.zeros(0, np.uint16), np.array([0, 0], np.uint8), [0], None)
    L = make_layout(2, 0, A.F_COND)
    st = pack_state(L, np.zeros(1, np.uint32), np.zeros(1, np.uint8), np.array([[0, A.PHASE_SUCCEEDED]], np.uint8),
                    cond=np.array([[A.COND_FAIL, A.COND_PASS]], np.uint8))
    recs, ev, n = M.status(L, ts, [0], st, 1)
    r = recs[0]
    assert (r["group"], r["outcome"], r["failed"], r["completed"], r["n_events"]) == (A.GROUP_MAIN, A.OUTCOME_NONE, 0, 1, 0)
    assert n == 0


def test_stops_and_subsets():
    """a stopped run takes its outcome from the stop reason and lists only its allowed failures; runs lists a subset"""
    story = O.Story([O.Step("A", ref=True, allow_failure=True), O.Step("B", ref=True)], [], [])
    srun = O.StoryRun({"A": O.StepState("Failed"), "B": O.StepState("Failed")})
    ps = P.pack_story(story)
    L, st = P.pack_runs([story], [ps], [srun] * 4, [0] * 4, [0], host_groups=["finalize"] * 3 + [None])
    area = R.defaults(4)
    area["stop"][:3] = [A.STOP_TIMEOUT, A.STOP_CANCEL, A.STOP_HOST]
    recs, ev, n = M.status(L, P.topology_set([ps]), [0], st, 4, runctl=area)
    assert recs["outcome"].tolist() == [A.OUTCOME_TIMED_OUT, A.OUTCOME_CANCELED, A.OUTCOME_STOPPED, A.OUTCOME_DEPENDENCY_FAILED]
    assert recs["story_phase"].tolist() == [A.PHASE_TIMEOUT, A.PHASE_FINISHED, 0, A.PHASE_FAILED]
    assert recs["first_failed"].tolist() == [A.STATUS_NO_STEP] * 3 + [1]
    allowed = A.PHASE_FAILED << 10 | A.STATUS_EVT_ALLOWED << 14
    assert n == 5 and ev.tolist() == [allowed] * 4 + [1 | A.PHASE_FAILED << 10 | A.STATUS_EVT_FAILED << 14]
    sub, sev, sn = M.status(L, P.topology_set([ps]), [0], st, 4, runs=[1, 3], runctl=area, events_cap=2)
    assert sub["run"].tolist() == [1, 3] and sub["first_event"].tolist() == [0, 1] and sn == 3 and sev.tolist() == [allowed] * 2


@pytest.mark.parametrize("seed", range(300))
def test_model_vs_object_oracle(seed):
    """random object-shaped Stories and StoryRuns: the model's report is what the reference holds after one iteration's stages
    G / H / I (cond-FAIL writes of findReadySteps set back), and finalizeStoryRun's verdict when the group is done"""
    if _compare(seed) is None:
        pytest.skip("generated an invalid graph or a dangling cross-group alias reference")


def _compare(seed):
    """-> the outcome of the seed's run, None when the seed gives no valid Story"""
    rng = random.Random(seed)
    story, codes = _rand_story(rng)
    if O.validate_runtime_dependency_graph(O.all_story_steps(story)) is not None:
        return None
    try:
        ps = P.pack_story(story)
    except ValueError:
        return None
    srun, step_runs = _rand_run(rng, story)
    ev, now = _evaluator(codes), 100.0
    L, state = P.pack_runs([story], [ps], [_clone_run(srun)], [0], [0], [step_runs], ev, {"inputs": {}, "steps": {}}, now)
    recs, events, n = M.status(L, P.topology_set([ps]), [0], state, 1)

    before = _clone_run(srun)
    it = O.run_dag_iteration(srun, story, step_runs, ev, {"inputs": {}, "steps": {}}, now)
    states = srun.step_states
    for name in it.ready.failed_now:   # stage D's writes reach a record only through a commit
        if name in before.step_states:
            states[name] = before.step_states[name]
        else:
            states.pop(name, None)
    names = ps.names
    idx = {nm: i for i, nm in enumerate(names)}
    r = recs[0]
    assert (int(r["active"]), int(r["completed"]), int(r["failed"]), int(r["skipped"])) == F.summarize_step_progress(states)
    want_events = []
    if it.group == "finalize":
        phase, reason, _msg, listed = F.finalize_story_run(story, states, *F.failed_sets(story, states))
        outcome = OUTCOME[(phase, reason)]
        assert r["story_phase"] == A.PHASE_NAMES.index(phase)
        first = min((idx[nm] for nm in listed), default=A.STATUS_NO_STEP)
        assert r["first_failed"] == first and (not listed or names[first] in _msg or outcome == A.OUTCOME_COMPENSATED)
        want_events += [(idx[nm], O.PHASE_CODE[ph], A.STATUS_EVT_FAILED) for nm, ph in listed.items()]
    else:
        outcome = A.OUTCOME_NONE
        assert r["first_failed"] == A.STATUS_NO_STEP and r["story_phase"] == 0
    assert r["outcome"] == outcome and r["group"] == {"main": 0, "compensation": 1, "finally": 2, "finalize": 3}[it.group]
    want_events += [(idx[nm], O.PHASE_CODE[states[nm].phase], A.STATUS_EVT_ALLOWED)
                    for nm in O.collect_allowed_failures(O.all_story_steps(story), states)]
    got = [(int(e) & 0x3FF, (int(e) >> 10) & 0xF, int(e) >> 14) for e in events]
    assert got == sorted(want_events) and n == r["n_events"] == len(want_events)
    return outcome


def test_every_outcome_branch():
    """more random Stories, compared the same way, until every outcome the object oracle gives a run without stops was met"""
    want = {A.OUTCOME_NONE, A.OUTCOME_SUCCEEDED, A.OUTCOME_DEPENDENCY_FAILED, A.OUTCOME_COMPENSATED,
            A.OUTCOME_COMPENSATION_FAILED, A.OUTCOME_CLEANUP_FAILED}
    seen = collections.Counter(_compare(seed) for seed in range(10_000, 13_000))
    assert want <= set(seen), dict(seen)
