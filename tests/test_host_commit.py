"""The host model of bf_resident_commit (tests/commit.py) pinned with known answers from the reference, and the commit loop
(single-pass tick + commit until a commit writes nothing) against one BF_EVAL_FIXPOINT pass of the packed oracle."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import PAR_DTYPE, make_layout, pack_state, unpack_result
from oracle import packed as PK
from tests import commit as M
from tests import randgen

E, COND, PAR, SLEEP, STOP, WAIT, EXEC, GATE = range(8)


def topo(types, par_branches=()):
    """one topology of independent steps of the given types; the parallel steps get par_branches branches each"""
    S = len(types)
    par = np.zeros(len(par_branches), PAR_DTYPE)
    steps = [i for i, t in enumerate(types) if t == PAR]
    for q, (s, b) in enumerate(zip(steps, par_branches)):
        par[q] = (s, b, 0)
    return TopologySet([S], [0], np.zeros(S + 1, np.uint32), np.zeros(0, np.uint16), np.asarray(types, np.uint8), [len(par)], par)


def batch(types, phases, fields=A.F_ALL_OUT, reg=None):
    """one topology at slot 0, one run per row of `phases`"""
    ts = topo(types, [2] * sum(1 for t in types if t == PAR))
    S = len(types)
    L = make_layout(S, 0, fields)
    ph = np.asarray(phases, np.uint8).reshape(-1, S)
    n = ph.shape[0]
    reg = np.zeros(n, np.uint64) if reg is None else np.asarray(reg, np.uint64)
    st = pack_state(L, np.zeros(n, np.uint32), np.zeros(n, np.uint8), ph, registered=reg)
    return M.Topologies(ts, [0]), L, st


def result(L, n, **masks):
    """result records of n runs with the given step lists per mask (ready / skip / fail), run 0 unless given as (run, steps)"""
    res = np.zeros((n, L.result_stride), np.uint8)
    for name, spec in masks.items():
        off = {"ready": L.off_ready, "skip": L.off_skip, "fail": L.off_fail}[name]
        for r, steps in (spec if isinstance(spec, dict) else {0: spec}).items():
            v = sum(1 << s for s in steps)
            res[r, off:off + 4 * L.words] = np.frombuffer(v.to_bytes(4 * L.words, "little"), np.uint8)
    return res


def phases(L, st, S):
    from bobrapet_b200.records import _unpack_planes
    return _unpack_planes(st[:, L.off_phase:L.off_phase + 16 * L.words], L.words, 4, S)


def test_if_false_is_skipped():
    """dag_test.go:690: a step whose `if` evaluates false is marked Skipped in the same reconcile"""
    t, L, st = batch([E, E], [[A.PHASE_SUCCEEDED, 0]])
    rc, _, _, counts, touched = M.commit(L, t, st, result(L, 1, skip=[1]), None, 1)
    assert rc == 0 and touched == {0}
    assert phases(L, st, 2)[0].tolist() == [A.PHASE_SUCCEEDED, A.PHASE_SKIPPED]
    assert counts["n_skipped"] == 1 and counts["n_runs_written"] == 1


def test_two_queued_steps_get_code_14():
    """dag_test.go:744: the steps the limits cut are Pending with a "Queued due to ..." message"""
    t, L, st = batch([E, E, E], [[0, 0, 0]])
    rc, _, _, counts, _ = M.commit(L, t, st, result(L, 1, ready=[0, 1, 2]), {0: (0b001, 0b110)}, 1)
    assert rc == 0
    assert phases(L, st, 3)[0].tolist() == [A.PHASE_RUNNING, A.PHASE_PENDING_QUEUED, A.PHASE_PENDING_QUEUED]
    assert counts["n_queued"] == 2 and counts["n_launched"] == 1


def test_blocked_engram_stays_blocked_and_queued_one_runs():
    """dag.go:1770-1774: a launched engram step becomes Running only from no phase or the queued Pending"""
    t, L, st = batch([E, E, EXEC], [[A.PHASE_BLOCKED, A.PHASE_PENDING_QUEUED, A.PHASE_SCHEDULING]])
    rc, _, _, counts, touched = M.commit(L, t, st, result(L, 1, ready=[0, 1, 2]), None, 1)
    assert rc == 0
    assert phases(L, st, 3)[0].tolist() == [A.PHASE_BLOCKED, A.PHASE_RUNNING, A.PHASE_SCHEDULING]
    assert counts["n_launched"] == 1 and touched == {0}


def test_condition_succeeds_and_primitives_pause():
    """step_executor.go:168-179"""
    t, L, st = batch([COND, GATE, SLEEP, WAIT], [[0, 0, 0, 0]])
    assert M.commit(L, t, st, result(L, 1, ready=[0, 1, 2, 3]), None, 1)[0] == 0
    assert phases(L, st, 4)[0].tolist() == [A.PHASE_SUCCEEDED, A.PHASE_PAUSED, A.PHASE_PAUSED, A.PHASE_PAUSED]


def test_parallel_runs_and_registers():
    """step_executor.go:808-809: the parallel step is Running with its children registered"""
    t, L, st = batch([E, PAR, PAR], [[0, 0, 0]])
    rc, _, _, counts, _ = M.commit(L, t, st, result(L, 1, ready=[2]), None, 1)
    assert rc == 0
    assert phases(L, st, 3)[0].tolist() == [0, 0, A.PHASE_RUNNING]
    assert int(st[0, 8:16].view("<u8")[0]) == 0b10   # desc 1 is step 2
    assert counts["n_launched"] == 1
    # a parallel step already Running that registers only now counts once too
    t, L, st = batch([PAR], [[A.PHASE_RUNNING]])
    assert M.commit(L, t, st, result(L, 1, ready=[0]), None, 1)[3]["n_launched"] == 1
    assert int(st[0, 8:16].view("<u8")[0]) == 1


def test_stop_takes_the_phase_of_its_entry():
    """step_executor.go:1096-1106; a launched stop step without an entry is refused"""
    t, L, st = batch([E, STOP], [[0, 0]])
    res = result(L, 1, ready=[0, 1])
    before = st.copy()
    assert M.commit(L, t, st, res, None, 1)[:3] == (M.EINVAL, 0, 1)
    assert np.array_equal(st, before)
    assert M.commit(L, t, st, res, None, 1, [(0, 1, M.PHASE, A.PHASE_FAILED)])[0] == 0
    assert phases(L, st, 2)[0].tolist() == [A.PHASE_RUNNING, A.PHASE_FAILED]


def test_error_leaves_the_run_and_hold_its_step():
    """dag.go:1750-1768: an Execute error persists nothing of the run; a blocked template holds only its step"""
    t, L, st = batch([E, E, E], [[0, 0, 0], [0, 0, 0]])
    res = result(L, 2, ready={0: [0, 1], 1: [0, 1]}, skip={0: [2], 1: [2]})
    rc, _, _, counts, touched = M.commit(L, t, st, res, None, 2, [(0, 1, M.ERROR, 0), (1, 1, M.HOLD, 0)])
    assert rc == 0 and touched == {1}
    ph = phases(L, st, 3)
    assert ph[0].tolist() == [0, 0, 0]
    assert ph[1].tolist() == [A.PHASE_RUNNING, 0, A.PHASE_SKIPPED]


def test_cond_fail_is_failed():
    t, L, st = batch([E, E], [[0, 0]])
    rc, _, _, counts, _ = M.commit(L, t, st, result(L, 1, fail=[1]), None, 1)
    assert rc == 0 and counts["n_failed"] == 1
    assert phases(L, st, 2)[0].tolist() == [0, A.PHASE_FAILED]


def test_second_commit_writes_nothing():
    t, L, st = batch([E, COND, PAR, GATE, E], [[0, 0, 0, 0, 0]] * 3)
    res = result(L, 3, ready={0: [0, 1, 2, 3], 1: [0], 2: [2]}, skip={0: [4], 2: [4]})
    first = M.commit(L, t, st, res, {0: (0b1111, 0), 1: (0, 0b1), 2: (0b100, 0)}, 3)
    assert first[0] == 0 and first[3]["n_runs_written"] == 3
    again = st.copy()
    second = M.commit(L, t, st, res, {0: (0b1111, 0), 1: (0, 0b1), 2: (0b100, 0)}, 3)
    assert second[0] == 0 and second[4] == set() and all(v == 0 for v in second[3].values())
    assert np.array_equal(st, again)


@pytest.mark.parametrize("bad", ["run", "step", "kind", "code", "hold-code", "dup", "not-launched", "not-stop"])
def test_refusals_name_the_offender_and_change_nothing(bad):
    t, L, st = batch([E, STOP, E], [[0, 0, 0], [0, 0, 0]])
    res = result(L, 2, ready={0: [0, 1], 1: [0]})
    ents = [(0, 1, M.PHASE, A.PHASE_SUCCEEDED), (1, 0, M.HOLD, 0)]
    want = {"run": (2, 0), "step": (1, 3), "kind": (1, 0), "code": (0, 1), "hold-code": (1, 0), "dup": (1, 0),
            "not-launched": (1, 2), "not-stop": (1, 0)}[bad]
    if bad == "run":
        ents.append((2, 0, M.HOLD, 0))
    elif bad == "step":
        ents.append((1, 3, M.HOLD, 0))
    elif bad == "kind":
        ents[1] = (1, 0, 4, 0)
    elif bad == "code":
        ents[0] = (0, 1, M.PHASE, A.PHASE_PENDING_QUEUED)
    elif bad == "hold-code":
        ents[1] = (1, 0, M.HOLD, 3)
    elif bad == "dup":
        ents.append((1, 0, M.ERROR, 0))
    elif bad == "not-launched":
        ents.append((1, 2, M.HOLD, 0))
    else:
        ents[1] = (1, 0, M.PHASE, A.PHASE_SUCCEEDED)
    before = st.copy()
    assert M.commit(L, t, st, res, None, 2, ents)[:3] == (M.EINVAL,) + want
    assert np.array_equal(st, before)


def commit_loop(pt, t, L, st0, n, rounds_cap=2000):
    """single-pass ticks, each followed by a commit, until a commit writes nothing -> (union ready, union skip, last result)"""
    st = st0.copy()
    ready = np.zeros((n, 32 * L.words), bool)
    skip = np.zeros_like(ready)
    for _ in range(rounds_cap):
        res, _ = PK.evaluate(pt, L, st)
        u = unpack_result(L, res, 32 * L.words)
        ready |= u["ready"]
        skip |= u["skip"]
        rc, _, _, counts, _ = M.commit(L, t, st, res, None, n)
        assert rc == 0
        if counts["n_runs_written"] == 0:
            return ready, skip, u, st
    raise AssertionError("the commit loop did not settle")


def no_stops(ts):
    """the same topologies with every stop step an engram step (a stop step hands the fixpoint's run to the host)"""
    f = ts.step_flags.copy()
    f[(f & A.SF_TYPE_MASK) == A.STEP_STOP] &= ~np.uint8(A.SF_TYPE_MASK)
    return TopologySet(ts.S, ts.E, ts.row_ptr, ts.col_idx, f, ts.P, ts.parallel, ts.allow_bits)


# The runs where the commit loop differs from one fixpoint pass, with the finding that explains each (DESIGN.md, "Tick commits"),
# for the seeded batches of this file and of tests/test_gpu_commit.py: (S, parallel topologies, seed, runs) -> {run: finding}.
# Every other run must agree exactly.  "cond-fail": the fixpoint ended on an iteration whose only change was a cond FAIL, and the
# loop readied and skipped a superset of its steps; "left-main": the run left its main group under fail-fast or a terminated
# topology, so the fixpoint's main-group stage I rewrites are not re-derived by the loop's last pass.
PINNED = {
    (64, False, 1, 300): {},
    (64, True, 2, 300): {116: "cond-fail"},
    (256, True, 3, 300): {},
    (64, True, 2, 2000): {25: "left-main", 166: "cond-fail+left-main", 576: "cond-fail", 902: "cond-fail", 909: "cond-fail+left-main",
                          1084: "cond-fail", 1196: "cond-fail", 1211: "cond-fail+left-main", 1441: "cond-fail", 1629: "left-main"},
    (256, True, 3, 2000): {55: "left-main", 563: "cond-fail", 1921: "cond-fail"},
    (1024, False, 4, 2000): {1265: "cond-fail"},
}


def seeded_batch(S, parallel, seed, n, clean=True):
    """the random batch of a PINNED key: topologies without stop steps, records whose unregistered descs hold no child phases"""
    rng = np.random.default_rng(seed)
    ts = no_stops(randgen.random_topologies(rng, 6, S // 2, S, max_deg=3, parallel=parallel, fill=0.5))
    L, st, topo_of = randgen.random_state(rng, ts, np.arange(ts.count, dtype=np.uint32), n, A.F_COND | A.F_DECISION | A.F_ALL_OUT,
                                          phase_mix="progress")
    if clean:
        unregistered_children_zero(L, st, ts, topo_of)
    return ts, L, st, topo_of


def differences(st, ready, skip, last, f):
    """{run: finding} of the runs whose loop unions (ready, skip) or last phase_out differ from the fixpoint pass f; the finding is
    "cond-fail", "left-main", both joined by "+", or "" when neither explains the run"""
    same = np.all(ready == f["ready"], axis=1) & np.all(skip == f["skip"], axis=1) & np.all(last["phase_out"] == f["phase_out"], axis=1)
    out = {}
    for r in np.nonzero(~same)[0]:
        flags = int(st[r, 4])
        cf = bool(f["fail"][r].any()) and bool(np.all(ready[r] | ~f["ready"][r])) and bool(np.all(skip[r] | ~f["skip"][r]))
        lm = bool(flags & (A.RF_FAIL_FAST | A.RF_TOPOLOGY_TERMINATED)) and int(f["summary"][r]) & A.SUM_GROUP_MASK != A.GROUP_MAIN \
            and not flags & A.RF_HOST_GROUP
        out[int(r)] = "+".join(name for name, hit in (("cond-fail", cf), ("left-main", lm)) if hit)
    return out


def loop_differences(ts, L, st):
    n = st.shape[0]
    slots = np.arange(ts.count, dtype=np.uint32)
    pt = PK.PackedTopologies(ts, slots)
    ready, skip, last, _ = commit_loop(pt, M.Topologies(ts, slots), L, st, n)
    fx, _ = PK.evaluate(pt, L, st, flags=A.EVAL_FIXPOINT)
    return differences(st, ready, skip, last, unpack_result(L, fx, 32 * L.words))


@pytest.mark.parametrize("key", [k for k in PINNED if k[3] == 300])
def test_commit_loop_matches_one_fixpoint_pass(key):
    """ready and skipped steps over the rounds and the final phase_out agree with BF_EVAL_FIXPOINT run by run, but for the pinned
    runs, each with its finding"""
    ts, L, st, _ = seeded_batch(*key)
    assert loop_differences(ts, L, st) == PINNED[key]


def unregistered_children_zero(L, st, ts, topo_of):
    """zero the child nibbles of every parallel desc whose children_registered bit is 0: a StoryRun has no child StepRuns of a
    parallel step before it registers them (step_executor.go:808-809), so their phases are absent"""
    cfs, _ = randgen.child_layout(ts)
    pos = np.concatenate([[0], np.cumsum(ts.P)]).astype(np.int64)
    for r in range(st.shape[0]):
        i = int(topo_of[r])
        reg = int(st[r, 8:16].view("<u8")[0])
        for q in range(int(ts.P[i])):
            if (reg >> q) & 1:
                continue
            first, B = int(cfs[i][q]), int(ts.parallel["branches"][pos[i] + q])
            for c in range(first, first + B):
                byte = L.off_child + c // 2
                st[r, byte] &= np.uint8(0xF0 if c % 2 == 0 else 0x0F)


def test_launched_parallel_with_terminal_children_differs_from_the_fixpoint():
    """The third finding (DESIGN.md, "Tick commits"): the fixpoint launches a parallel step without registering its children, so
    it never joins it in a later iteration; a commit registers them, and the next tick joins the step when the record already
    holds terminal child phases for it.  A live record never does (children are created by the launch): with those phases zeroed
    the same batch differs only in its pinned run; with them kept, exactly these runs differ, and every added one holds child
    phases under an unregistered desc."""
    ts, L, clean, _ = seeded_batch(64, True, 2, 300)
    _, _, raw, _ = seeded_batch(64, True, 2, 300, clean=False)
    assert loop_differences(ts, L, clean) == PINNED[(64, True, 2, 300)]
    got = loop_differences(ts, L, raw)
    assert sorted(got) == [3, 5, 14, 35, 86, 108, 109, 116, 117, 150, 284]
    added = [r for r in got if r not in PINNED[(64, True, 2, 300)]]
    assert np.all(np.any(raw[added] != clean[added], axis=1))
