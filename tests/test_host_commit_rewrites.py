"""The host model of bf_resident_commit_rewrites (tests/commit_rewrites.py): the precondition the device relies on (only a run whose
result record carries BF_SUM_PHASE_CHANGED can have a rewrite), and the rewriting commit loop (single-pass tick + rewriting commit
until a commit writes nothing) against one BF_EVAL_FIXPOINT pass of the packed oracle, run by run, on the seeded batches of
tests/test_host_commit.py."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import unpack_result
from oracle import packed as PK
from tests import commit as M
from tests import commit_rewrites as CR
from tests import resync as RS
from tests.runstatus import _codes
from tests.test_host_commit import PINNED, differences, phases, seeded_batch

E, COND, PAR, SLEEP, STOP, WAIT, EXEC, GATE = range(8)

# The runs where the rewriting commit loop differs from one fixpoint pass, with the finding that explains each: "cond-fail" as in
# tests/test_host_commit.py; "later-reconcile": the run left its main group under fail-fast or a terminated topology, and the loop's
# later ticks read the stage I Failed / Skipped codes its commits stored (as the reference's next reconcile reads the persisted
# StepStates), so they fail-fast skip, and ready compensation or finally steps, past what the one-reconcile fixpoint's phase_out
# holds.  Every "left-main" run of the plain commit loop (tests/test_host_commit.py:PINNED) agrees here.
PINNED_REWRITES = {
    (64, False, 1, 300): {},
    (64, True, 2, 300): {49: "later-reconcile", 116: "cond-fail"},
    (256, True, 3, 300): {},
    (64, True, 2, 2000): {166: "cond-fail+later-reconcile", 270: "later-reconcile", 452: "later-reconcile", 576: "cond-fail",
                          622: "later-reconcile", 698: "later-reconcile", 709: "later-reconcile", 902: "cond-fail",
                          909: "cond-fail+later-reconcile", 999: "later-reconcile", 1084: "cond-fail", 1150: "cond-fail+later-reconcile",
                          1153: "later-reconcile", 1196: "cond-fail", 1211: "cond-fail+later-reconcile", 1441: "cond-fail",
                          1456: "later-reconcile"},
    (256, True, 3, 2000): {563: "cond-fail", 584: "later-reconcile", 1012: "later-reconcile", 1460: "later-reconcile",
                           1921: "cond-fail"},
    (1024, False, 4, 2000): {1265: "cond-fail"},
}


def rewrite_loop(ts, L, st0, n, rounds_cap=2000, check_precondition=False):
    """single-pass ticks, each followed by a rewriting commit, until a commit writes nothing -> (union ready, union skip, last
    result, final records)"""
    slots = np.arange(ts.count, dtype=np.uint32)
    pt = PK.PackedTopologies(ts, slots)
    topo, topos = M.Topologies(ts, slots), RS.Topos(ts, slots)
    st = st0.copy()
    ready = np.zeros((n, 32 * L.words), bool)
    skip = np.zeros_like(ready)
    for _ in range(rounds_cap):
        res, _ = PK.evaluate(pt, L, st)
        u = unpack_result(L, res, 32 * L.words)
        ready |= u["ready"]
        skip |= u["skip"]
        if check_precondition:
            changed = (u["summary"].astype(np.int64) & A.SUM_PHASE_CHANGED) != 0
            assert all(changed[r] for r in CR.post_differs(L, topos, st, n))
        rc, _, _, counts, _, _, _ = CR.commit(L, topo, topos, st, res, None, n)
        assert rc == 0
        if counts["n_runs_written"] == 0:
            return ready, skip, u, st
    raise AssertionError("the rewriting commit loop did not settle")


def rewrite_loop_differences(ts, L, st):
    n = st.shape[0]
    ready, skip, last, final = rewrite_loop(ts, L, st, n)
    fx, _ = PK.evaluate(PK.PackedTopologies(ts, np.arange(ts.count, dtype=np.uint32)), L, st, flags=A.EVAL_FIXPOINT)
    f = unpack_result(L, fx, 32 * L.words)
    got = differences(st, ready, skip, last, f)
    # the stored phases themselves end at the fixpoint's phase_out
    stored = np.stack([_codes(final[r], L.off_phase, L.words, 32 * L.words) for r in range(n)]) if n else None
    for r in np.nonzero(np.any(stored != f["phase_out"], axis=1))[0]:
        got.setdefault(int(r), "")
    # a run that leaves its main group under fail-fast or a terminated topology: the loop's later ticks read the stage I codes its
    # commits stored (as the reference's next reconcile reads the persisted StepStates), the fixpoint's later iterations did not
    return {r: why.replace("left-main", "later-reconcile") for r, why in got.items()}


def check_later_reconcile(ts, L, st, runs):
    """the direction the "later-reconcile" finding claims: the loop goes further than the fixpoint, never elsewhere.  Its ready
    and skipped steps are supersets of the fixpoint's, and every stored code that differs from the fixpoint's phase_out is at a
    step the fixpoint left without a phase, and is a stage I Skipped or Failed code or the launch write of a step only the loop
    readied"""
    n = st.shape[0]
    ready, skip, _last, final = rewrite_loop(ts, L, st, n)
    fx, _ = PK.evaluate(PK.PackedTopologies(ts, np.arange(ts.count, dtype=np.uint32)), L, st, flags=A.EVAL_FIXPOINT)
    f = unpack_result(L, fx, 32 * L.words)
    for r in runs:
        assert np.all(ready[r] | ~f["ready"][r]) and np.all(skip[r] | ~f["skip"][r]), r
        stored = _codes(final[r], L.off_phase, L.words, 32 * L.words)
        off = np.flatnonzero(stored != f["phase_out"][r])
        assert off.size and np.all(f["phase_out"][r][off] == 0), r
        extra = ready[r] & ~f["ready"][r]
        assert all(int(stored[s]) in (M.SKIPPED, M.FAILED) or extra[s] for s in off), (r, stored[off], off)


@pytest.mark.parametrize("key", sorted(PINNED))
def test_only_phase_changed_runs_have_rewrites(key):
    """every run whose post-stage phases differ from its stored codes carries BF_SUM_PHASE_CHANGED, at every round of the loop"""
    ts, L, st, _ = seeded_batch(*key)
    slots = np.arange(ts.count, dtype=np.uint32)
    res, _ = PK.evaluate(PK.PackedTopologies(ts, slots), L, st)
    u = unpack_result(L, res, 32 * L.words)
    differ = CR.post_differs(L, RS.Topos(ts, slots), st, st.shape[0])
    assert differ, "the batch exercises no rewrite"
    assert all(int(u["summary"][r]) & A.SUM_PHASE_CHANGED for r in differ)
    if key[3] == 300:
        rewrite_loop(ts, L, st, st.shape[0], check_precondition=True)


@pytest.mark.parametrize("key", sorted(PINNED))
def test_rewrite_loop_matches_one_fixpoint_pass(key):
    """ready and skipped steps over the rounds, the final phase_out and the final stored phases agree with BF_EVAL_FIXPOINT run
    by run, but for the pinned runs"""
    ts, L, st, _ = seeded_batch(*key)
    got = rewrite_loop_differences(ts, L, st)
    assert got == PINNED_REWRITES[key]
    if any("later-reconcile" in why for why in got.values()):
        check_later_reconcile(ts, L, st, [r for r, why in got.items() if "later-reconcile" in why])
    assert all(r not in got for r, why in PINNED[key].items() if why == "left-main")


def test_fired_sleep_is_stored_and_marked():
    """a sleep with a fired timer decision becomes Succeeded in the record, and the item is marked as a rewrite"""
    from tests.test_host_commit import topo
    from bobrapet_b200.records import make_layout, pack_state
    ts = topo([E, SLEEP])
    L = make_layout(2, 0, A.F_ALL_OUT | A.F_DECISION)
    ph = np.array([[A.PHASE_RUNNING, A.PHASE_PAUSED]], np.uint8)
    dec = np.array([[0, A.DEC_SUCCEED]], np.uint8)
    st = pack_state(L, np.zeros(1, np.uint32), np.zeros(1, np.uint8), ph, decision=dec)
    slots = np.zeros(1, np.uint32)
    res, _ = PK.evaluate(PK.PackedTopologies(ts, slots), L, st)
    before = st.copy()
    rc, _, _, counts, touched, n_rw, masked = CR.commit(L, M.Topologies(ts, slots), RS.Topos(ts, slots), st, res, None, 1)
    assert rc == 0 and touched == {0} and n_rw == 1 and counts["n_runs_written"] == 1
    assert phases(L, st, 2)[0].tolist() == [A.PHASE_RUNNING, A.PHASE_SUCCEEDED]
    items, runs = CR.journal(L, before, st, 1, masked)
    assert items == [(0, 1, A.DELTA_PHASE, CR.REWRITE, A.PHASE_PAUSED, A.PHASE_SUCCEEDED)] and runs == [0]
    # the plain commit stores nothing of it
    st2 = before.copy()
    assert M.commit(L, M.Topologies(ts, slots), st2, res, None, 1)[3]["n_runs_written"] == 0


def test_error_and_stopped_runs_get_no_rewrite():
    from tests.test_host_commit import topo
    from bobrapet_b200.records import make_layout, pack_state
    ts = topo([E, SLEEP])
    L = make_layout(2, 0, A.F_ALL_OUT | A.F_DECISION)
    ph = np.array([[0, A.PHASE_PAUSED]] * 3, np.uint8)
    dec = np.array([[0, A.DEC_SUCCEED]] * 3, np.uint8)
    stopped_flags = A.RF_HOST_GROUP | A.GROUP_DONE << A.RF_HOST_GROUP_SHIFT   # what a stop leaves in the record
    st = pack_state(L, np.zeros(3, np.uint32), np.array([0, 0, stopped_flags], np.uint8), ph, decision=dec)
    slots = np.zeros(1, np.uint32)
    res, _ = PK.evaluate(PK.PackedTopologies(ts, slots), L, st)
    runctl = np.zeros(3, dtype=[("stop", "u1")])
    runctl["stop"][2] = 2
    rc, _, _, counts, touched, n_rw, _ = CR.commit(L, M.Topologies(ts, slots), RS.Topos(ts, slots), st, res, None, 3,
                                                   [(0, 0, M.ERROR, 0)], runctl=runctl)
    assert rc == 0 and touched == {1} and n_rw == 1
    assert phases(L, st, 2)[:, 1].tolist() == [A.PHASE_PAUSED, A.PHASE_SUCCEEDED, A.PHASE_PAUSED]
