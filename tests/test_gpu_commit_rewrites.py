"""Rewriting tick commits (bf_resident_commit_rewrites) on the device against the host model tests/commit_rewrites.py, byte for
byte: the state records, the counts, n_rewritten, the journal and the touched runs, round after round.  Over both kernels' widths
(S = 32, 64, 256, 1024), with and without cond / decision planes and a child area, with stopped runs, dead and too-wide slots,
HOLD and ERROR entries, a limiter area and arming; pinned and pageable buffers and a small items_cap; every refusal of the
journaled commit; a twin batch committed with bf_resident_commit_journal; the rewriting commit loop against one BF_EVAL_FIXPOINT
pass; and the resync of the cluster view after rewriting commits."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import unpack_result
from tests import commit as M
from tests import commit_journal as J
from tests import commit_rewrites as CR
from tests import randgen
from tests import resync as RS
from tests import runctl as R
from tests.runstatus import _codes
from tests.test_gpu_commit import ALL, BIG, NONE_D, TABLES, entries_for
from tests.test_gpu_commit_timers import put_all, random_timings
from tests.test_gpu_resync import cluster_view, _subset
from tests.test_host_commit import differences, no_stops, seeded_batch
from tests.test_host_commit_rewrites import PINNED_REWRITES

pytestmark = pytest.mark.gpu


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def cap_for(L, n):
    """a journal cap no commit of n runs can exceed: a phase item per step, a registered bit per desc, 64 timer slots"""
    return n * (32 * L.words + 128)


def rewrites_pinned(fr, h, n, ents, now, items_cap):
    """bf_resident_commit_rewrites into pinned items and runs -> the dict of Frontier.resident_commit(rewrites=True)"""
    ib = fr.alloc_pinned(max(items_cap, 1) * 16)
    rb = fr.alloc_pinned(max(n, 1) * 4)
    ents = np.ascontiguousarray(ents, dtype=Frontier.COMMIT_DTYPE)
    out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
    arm = None if now is None else A.CommitArm(struct_size=ctypes.sizeof(A.CommitArm), now=now)
    j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal), items=ib.ctypes.data, items_cap=items_cap,
                        runs=rb.ctypes.data, runs_cap=n)
    nrw = ctypes.c_uint32(77)
    rc = fr._lib.bf_resident_commit_rewrites(fr._ctx, h, n, ents.ctypes.data if ents.shape[0] else None, ents.shape[0],
                                             ctypes.byref(out), None if arm is None else ctypes.byref(arm), ctypes.byref(j),
                                             ctypes.byref(nrw))
    assert rc == A.BF_OK, fr._lib.bf_last_error(fr._ctx).decode()
    got = {k: int(getattr(out, k)) for k in M.COUNT_KEYS}
    if arm is not None:
        got.update(n_armed=int(arm.n_armed), next_deadline=int(arm.next_deadline))
    got.update(items=ib.view(Frontier.COMMIT_WRITE_DTYPE)[:min(int(j.n_items), items_cap)].copy(), n_items=int(j.n_items),
               runs=rb.view(np.uint32)[:int(j.n_runs_listed)].copy(), n_runs_listed=int(j.n_runs_listed), n_rewritten=int(nrw.value))
    return got


class Batch:
    """one resident batch with its host copy: records, schedule rows and run control"""

    def __init__(self, fr, ts, slots, L, st, sched, runctl):
        self.fr, self.L, self.n = fr, L, st.shape[0]
        self.topo, self.topos = M.Topologies(ts, slots), RS.Topos(ts, slots)
        self.h = fr.resident_create(L, self.n)
        fr.resident_upload(self.h, 0, st)
        self.sched = None
        if sched:
            fr.resident_sched(self.h)
            q = np.zeros(self.n, dtype=Frontier.SCHED_PUT_DTYPE)
            q["run"], q["story_key"], q["queue_key"] = np.arange(self.n), np.arange(self.n) % 4, np.arange(self.n) % 3
            q["priority"], q["queued_since"], q["run_phase"] = np.arange(self.n) % 5, A.SCHED_NONE, A.PHASE_RUNNING
            fr.resident_sched_put(self.h, q)
            self.sched = {}
        self.area = None
        if runctl:
            fr.resident_runctl(self.h)
            self.area = R.defaults(self.n)

    def tick(self):
        res = self.fr.resident_tick(self.h, self.L, self.n, NONE_D)[0]
        if self.sched is not None:
            out = self.fr.resident_schedule([dict(handle=self.h, n_runs=self.n, runs_cap=self.n, events_cap=BIG)], TABLES, 100)
            M.sched_rows(self.L, out["parts"][0], self.sched)
        return res

    def state(self):
        return self.fr.resident_download(self.h, 0, self.n, self.L.state_stride)


def _wide_slot(fr, L):
    """a slot of one word more than the layout"""
    S = 32 * L.words + 32
    wide = TopologySet([S], [0], np.zeros(S + 1, np.uint32), np.zeros(0, np.uint16), np.full(S, A.STEP_ENGRAM, np.uint8), [0],
                       np.zeros(0, dtype=[("step", "<u2"), ("branches", "<u2"), ("allow_first", "<u4")]))
    return int(fr.put_topologies(wide)[0])


# (S, fields, parallel, runs, limiter area, run control, timer slots per run)
CASES = [(32, ALL, True, 2000, False, True, 0), (64, A.F_DECISION | A.F_OUT_FAIL, True, 3000, True, False, 8),
         (256, ALL | A.F_CHILD, True, 8000, False, True, 16), (256, A.F_DECISION | A.F_ALL_OUT, False, 4000, True, True, 0),
         (1024, ALL, True, 300, True, False, 64), (1024, A.F_DECISION | A.F_ALL_OUT, False, 200, False, True, 0)]


@pytest.mark.parametrize("S,fields,parallel,n,sched,runctl,K", CASES)
def test_rewrites_match_the_model(fr, S, fields, parallel, n, sched, runctl, K):
    rng = np.random.default_rng(S * 31 + n + K)
    ts = no_stops(randgen.random_topologies(rng, 12, max(2, S // 2), S, max_deg=4, parallel=parallel, fill=0.5)) \
        if S == 32 else randgen.random_topologies(rng, 12, max(2, S // 2), S, max_deg=4, parallel=parallel, fill=0.5)
    slots = fr.put_topologies(ts)
    L, st, _ = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
    st = st.copy()
    if L.words < 32:   # a slot too wide for the layout: no masks, no rewrite (32 words is the widest topology)
        st[7, :4] = np.frombuffer(np.uint32(_wide_slot(fr, L)).tobytes(), np.uint8)
    a = Batch(fr, ts, slots, L, st, sched, runctl)
    b = Batch(fr, ts, slots, L, st, sched, runctl)   # the twin, committed with bf_resident_commit_journal
    if K:
        for x in (a, b):
            fr.resident_timers(x.h, K)
        timings = random_timings(rng, ts, slots)
        for slot in timings:
            t = {s: cd for s, cd in timings[slot].items() if L.off_decision != A.OFF_NONE or cd[0] == A.DEC_PENDING}
            timings[slot] = dict(sorted(t.items())[:8])
        put_all(fr, timings)
    dead = int(slots[0])
    fr.drop_topology(dead)
    for x in (a, b):
        x.topo.drop(dead)
    if runctl:
        q = np.zeros(min(n, 40), dtype=R.PUT_DTYPE)
        q["run"] = rng.choice(n, size=q.shape[0], replace=False)
        q["story_deadline"] = R.NONE
        q["drain_deadline"] = R.NONE
        q["stop"] = 2
        for x in (a, b):
            fr.resident_runctl_put(x.h, q)
        R.put(a.area, a.state(), q)
    rewritten, kinds = 0, set()
    for rnd in range(4):
        now = 100 + rnd if K else None
        res = a.tick()
        before = a.state()
        ents = entries_for(rng, L, a.topo, before, res, a.sched, n)
        t0 = fr.resident_timers_download(a.h, 0, n, K).view("<u8").copy() if K else None
        want_st = before.copy()
        rc, _, _, counts, touched, n_rw, masked = CR.commit(L, a.topo, a.topos, want_st, res, a.sched, n, ents, a.area)
        assert rc == 0
        cap = cap_for(L, n)
        if rnd == 1:
            got = rewrites_pinned(fr, a.h, n, ents, now, cap)
        elif rnd == 2:
            got = fr.resident_commit(a.h, n, ents, now=now, journal_cap=5, rewrites=True)
        else:
            got = fr.resident_commit(a.h, n, ents, now=now, journal_cap=cap, rewrites=True)
        after = a.state()
        assert np.array_equal(after, want_st), np.nonzero(np.any(after != want_st, axis=1))[0][:10]
        t1 = fr.resident_timers_download(a.h, 0, n, K).view("<u8").copy() if K else None
        want_items, want_runs = CR.journal(L, before, after, n, masked, t0, t1)
        items = J.as_tuples(got["items"])
        assert got["n_items"] == len(want_items) and items == want_items[:len(items)]
        assert len(items) == min(len(want_items), 5 if rnd == 2 else cap)
        assert got["runs"].tolist() == want_runs == sorted(touched)
        assert {k: got[k] for k in M.COUNT_KEYS} == counts and got["n_rewritten"] == n_rw
        assert n_rw == sum(1 for x in want_items if x[2] == J.PHASE and x[3] == CR.REWRITE)
        assert L.words == 32 or 7 not in want_runs
        assert not {r for r in range(n) if int(before[r][:4].view("<u4")[0]) == dead} & set(want_runs)
        if runctl:
            assert not set(np.nonzero(a.area["stop"][:n])[0].tolist()) & set(want_runs)
        rewritten += n_rw
        if rnd == 0:   # the twin's journaled commit differs only by the rewrite items
            assert np.array_equal(res, b.tick())
            jb = fr.resident_commit(b.h, n, ents, now=now, journal_cap=cap)
            assert J.as_tuples(jb["items"]) == [x for x in want_items if x[3] != CR.REWRITE or x[2] != J.PHASE]
        for r, s, f, code, _b, after_code in want_items:   # which stage each rewrite comes from
            if f == J.PHASE and code == CR.REWRITE:
                t = a.topo.by_slot[int(before[r][:4].view("<u4")[0])]
                kinds.add("G" if (t["sync"] >> s) & 1 else "H" if (t["par"] >> s) & 1 else "I%d" % after_code)
        # the next touched tick evaluates exactly the written runs and lists those whose result record changed
        ev = fr.eval(L, after)[0]
        want_listed = [r for r in sorted(touched) if not np.array_equal(ev[r], res[r])]
        t = fr.resident_tick_touched(a.h, n, NONE_D, max(n, 1), BIG)
        assert t["full"] == 0 and t["n_evaluated"] == len(touched) and t["runs"].tolist() == want_listed
    assert rewritten > 0
    # the inputs reach every kind of rewrite the layout allows: stage G (sleep / gate / wait), stage H (joins), stage I
    # (fail-fast and compensation skips, terminated-topology fails)
    assert {"I%d" % M.SKIPPED} <= kinds, kinds
    if L.off_decision != A.OFF_NONE:
        assert "G" in kinds, kinds
    if L.off_child != A.OFF_NONE:
        assert "H" in kinds, kinds


def test_refusals_change_nothing(fr):
    rng = np.random.default_rng(91)
    n = 1500
    ts = randgen.random_topologies(rng, 12, 32, 64, max_deg=4, parallel=True, fill=0.5)
    slots = fr.put_topologies(ts)
    L, st, _ = randgen.random_state(rng, ts, slots, n, ALL, phase_mix="progress")
    a = Batch(fr, ts, slots, L, st, False, False)
    res = a.tick()
    state = a.state()
    ents = entries_for(rng, L, a.topo, state, res, None, n, p_error=0)
    launched = {(int(e["run"]), int(e["step"])) for e in ents}
    r0 = next(r for r in range(n) if M.masks(L, a.topo, state, res, None, r)[1])
    free = next(s for s in range(L.steps_max) if (r0, s) not in launched and not (M.masks(L, a.topo, state, res, None, r0)[1] >> s) & 1)
    for bad in (np.concatenate([ents, ents[:1]]), np.concatenate([ents, np.array([(r0, free, M.HOLD, 0)], dtype=Frontier.COMMIT_DTYPE)])):
        for pinned in (False, True):
            items = fr.alloc_pinned(64 * 16) if pinned else np.zeros(64 * 16, np.uint8)
            runs = fr.alloc_pinned(n * 4) if pinned else np.zeros(n * 4, np.uint8)
            out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
            j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal), items=items.ctypes.data, items_cap=64,
                                runs=runs.ctypes.data, runs_cap=n, n_items=5, n_runs_listed=5)
            nrw = ctypes.c_uint32(9)
            rc = fr._lib.bf_resident_commit_rewrites(fr._ctx, a.h, n, bad.ctypes.data, bad.shape[0], ctypes.byref(out), None,
                                                     ctypes.byref(j), ctypes.byref(nrw))
            assert rc == A.BF_EINVAL and (j.n_items, j.n_runs_listed, nrw.value) == (0, 0, 0)
            assert not items.any() and not runs.any()
    out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
    j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal))
    nrw = ctypes.c_uint32(0)
    assert fr._lib.bf_resident_commit_rewrites(fr._ctx, a.h, n, None, 0, ctypes.byref(out), None, None, ctypes.byref(nrw)) == A.BF_EINVAL
    assert fr._lib.bf_resident_commit_rewrites(fr._ctx, a.h, n, None, 0, ctypes.byref(out), None, ctypes.byref(j), None) == A.BF_EINVAL
    with pytest.raises(ValueError):
        fr.resident_commit(a.h, n, rewrites=True)
    assert np.array_equal(a.state(), state)
    # the device's entry offences with rewrites staged: a PHASE entry on a launched step that is not a stop step, and a launched
    # stop step without an entry
    stops = [(r, s) for r in range(n) for s in range(L.steps_max)
             if (M.masks(L, a.topo, state, res, None, r)[1] >> s) & 1 and (a.topo.by_slot[int(state[r][:4].view("<u4")[0])]["stop"] >> s) & 1]
    plain = next((int(e["run"]), int(e["step"])) for e in ents if int(e["kind"]) != M.PHASE)
    cases = [np.concatenate([ents[(ents["run"] != plain[0]) | (ents["step"] != plain[1])],
                             np.array([(plain[0], plain[1], M.PHASE, A.PHASE_SUCCEEDED)], dtype=Frontier.COMMIT_DTYPE)])]
    if stops:
        cases.append(ents[(ents["run"] != stops[0][0]) | (ents["step"] != stops[0][1])])
    for bad in cases:
        want = M.check(L, a.topo, state, res, None, n, bad)
        assert want[0]
        with pytest.raises(A.FrontierError) as e:
            fr.resident_commit(a.h, n, bad, journal_cap=cap_for(L, n), rewrites=True)
        assert (e.value.bad_run, e.value.bad_step) == want[1:]
        assert np.array_equal(a.state(), state)
    # the call-level refusals: a fixpoint tick since the last single-pass tick, a dropped slot since the last tick
    fr.resident_tick(a.h, L, n, NONE_D, flags=A.EVAL_FIXPOINT)
    with pytest.raises(A.FrontierError):
        fr.resident_commit(a.h, n, ents, journal_cap=cap_for(L, n), rewrites=True)
    res = a.tick()
    fr.drop_topology(int(slots[-1]))
    with pytest.raises(A.FrontierError):
        fr.resident_commit(a.h, n, ents, journal_cap=cap_for(L, n), rewrites=True)
    assert np.array_equal(a.state(), state)
    a.topo.drop(int(slots[-1]))
    res = a.tick()
    state = a.state()
    ents = entries_for(rng, L, a.topo, state, res, None, n, p_error=0)
    # the commit goes through afterwards, and a second one without a tick between is refused (the first wrote)
    want = state.copy()
    rc, _, _, counts, touched, n_rw, _ = CR.commit(L, a.topo, a.topos, want, res, None, n, ents)
    got = fr.resident_commit(a.h, n, ents, journal_cap=cap_for(L, n), rewrites=True)
    assert np.array_equal(a.state(), want) and got["n_rewritten"] == n_rw and got["n_runs_written"] == len(touched) > 0
    with pytest.raises(A.FrontierError):
        fr.resident_commit(a.h, n, ents, journal_cap=cap_for(L, n), rewrites=True)


@pytest.mark.parametrize("key", [k for k in PINNED_REWRITES if k[3] == 2000])
def test_rewrite_loop_matches_one_fixpoint_pass_on_the_device(fr, key):
    """the device form of test_host_commit_rewrites.test_rewrite_loop_matches_one_fixpoint_pass"""
    ts, L, st, topo_of = seeded_batch(*key)
    slots = fr.put_topologies(ts)
    st[:, :4] = np.ascontiguousarray(slots[topo_of], dtype="<u4").view(np.uint8).reshape(-1, 4)
    n = st.shape[0]
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    W = 32 * L.words
    ready = np.zeros((n, W), bool)
    skip = np.zeros_like(ready)
    for _ in range(key[0] + 4):
        u = unpack_result(L, fr.resident_tick(h, L, n, NONE_D)[0], W)
        ready |= u["ready"]
        skip |= u["skip"]
        if fr.resident_commit(h, n, journal_cap=cap_for(L, n), rewrites=True)["n_runs_written"] == 0:
            break
    else:
        raise AssertionError("the rewriting commit loop did not settle")
    f = unpack_result(L, fr.eval(L, st, flags=A.EVAL_FIXPOINT)[0], W)
    got = differences(st, ready, skip, u, f)
    final = fr.resident_download(h, 0, n, L.state_stride)
    stored = np.stack([_codes(final[r], L.off_phase, L.words, W) for r in range(n)])
    for r in np.nonzero(np.any(stored != f["phase_out"], axis=1))[0]:
        got.setdefault(int(r), "")
    assert {r: why.replace("left-main", "later-reconcile") for r, why in got.items()} == PINNED_REWRITES[key]


def _looped_rewrites(fr, rng, S, fields, n, ticks=4, parallel=True):
    """tests/test_gpu_resync.py:_looped with rewriting commits"""
    ts = no_stops(randgen.random_topologies(rng, 10, max(2, S // 2), S, max_deg=4, parallel=parallel, fill=0.5))
    slots = fr.put_topologies(ts)
    L, st, topo = randgen.random_state(rng, ts, slots, n, fields | A.F_ALL_OUT, phase_mix="progress")
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    keep = np.ones(ts.count, bool)
    keep[ts.count - 1] = False
    fr.drop_topology(int(slots[-1]))
    fr.resident_timers(h, 2)
    fr.resident_sched(h)
    fr.resident_runctl(h)
    runs = np.sort(rng.choice(n, size=n // 3, replace=False))
    tq = np.zeros(runs.size, dtype=Frontier.TIMER_DTYPE)
    tq["run"], tq["step"] = runs, rng.integers(0, 2, runs.size)
    tq["code"] = rng.choice([A.DEC_SUCCEED, A.DEC_FAIL, A.DEC_TIMED_OUT], runs.size) if L.off_decision != A.OFF_NONE else A.DEC_PENDING
    tq["deadline"] = rng.integers(0, 12, runs.size)
    fr.resident_timers_arm(h, tq)
    q = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
    q["run"], q["story_key"], q["queue_key"] = np.arange(n), np.arange(n) % 4, np.arange(n) % 3
    q["priority"], q["queued_since"], q["run_phase"] = np.arange(n) % 5, A.SCHED_NONE, A.PHASE_RUNNING
    fr.resident_sched_put(h, q)
    c = np.zeros(runs.size, dtype=Frontier.RUNCTL_PUT_DTYPE)
    c["run"], c["story_deadline"], c["drain_deadline"] = runs, rng.integers(5, 40, runs.size), A.TIMER_NONE
    c["stop"] = np.where(np.arange(runs.size) % 7 == 0, A.STOP_HOST, A.STOP_NONE)
    fr.resident_runctl_put(h, c)
    for k in range(ticks):
        fr.resident_fire(h, n, 4 * k)
        d = np.zeros(30, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"] = rng.choice(n, size=30, replace=False), rng.integers(0, 2, 30)
        d["field"], d["code"] = A.DELTA_PHASE, rng.choice([A.PHASE_RUNNING, A.PHASE_SUCCEEDED, A.PHASE_FAILED], 30)
        fr.resident_tick_touched(h, n, d, n, n * 1024)
        fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], TABLES, 4 * k)
        fr.resident_commit(h, n, journal_cap=cap_for(L, n), rewrites=True)
    return RS.Topos(_subset(ts, keep), slots[keep]), L, h


# the keys of tests/test_gpu_resync.py whose plain commits leave "tt-then-ff" runs: (S, planes, parallel)
TT_KEYS = [(32, 0, True), (32, 0, False), (32, A.F_COND | A.F_DECISION, False), (256, 0, False)]


@pytest.mark.parametrize("S,planes,parallel", TT_KEYS)
def test_cluster_view_after_rewriting_commits_lists_nothing(fr, S, planes, parallel):
    """the same seeds as test_gpu_resync.test_cluster_view_lists_nothing_and_perturbations_match: with the rewrites stored, the
    cluster view (the phases after a pass's rewrites) equals the device's records for every run"""
    rng = np.random.default_rng(S * 7 + planes + (0 if parallel else 1000))
    n = 500
    topos, L, h = _looped_rewrites(fr, rng, S, planes, n, parallel=parallel)
    state = fr.resident_download(h, 0, n, L.state_stride)
    area = fr.resident_runctl_download(h, 0, n)
    got = fr.resident_resync(h, n, cluster_view(L, topos, state, area), check=True)
    assert got["n_items"] == 0 and got["drifted"].size == 0, (got["drifted"], got["items"][:10])
