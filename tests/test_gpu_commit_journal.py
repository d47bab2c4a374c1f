"""Journaled tick commits (bf_resident_commit_journal) on the device: the journal equals the byte difference of the state records
(bf_resident_download) and timer slots (bf_resident_timers_download) around the call, and a twin batch committed with
bf_resident_commit or bf_resident_commit_timed ends byte-identical with the same counts.  Over both kernels' widths, with and
without cond / decision / child planes, a limiter area, run control and timers; pinned and pageable buffers; a small items_cap
(true count, a prefix, records still fully written); refusals (both batches and the journal untouched); a commit with an ERROR
entry in every launching run (those runs are neither written nor listed)."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import commit as M
from tests import commit_journal as J
from tests import runctl as R
from tests.test_gpu_commit import ALL, Twin, _batch, entries_for
from tests.test_gpu_commit_timers import put_all, random_timings

pytestmark = pytest.mark.gpu


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def journal_pinned(fr, h, n, ents, now, items_cap):
    """bf_resident_commit_journal with the items and runs in pinned memory -> (counts dict, items, runs).  The buffers stay
    allocated until the ctx closes, so that nothing a failing assertion shows points at freed memory."""
    ib = fr.alloc_pinned(max(items_cap, 1) * 16)
    rb = fr.alloc_pinned(max(n, 1) * 4)
    ents = np.ascontiguousarray(ents, dtype=Frontier.COMMIT_DTYPE)
    out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
    arm = None if now is None else A.CommitArm(struct_size=ctypes.sizeof(A.CommitArm), now=now)
    j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal), items=ib.ctypes.data, items_cap=items_cap,
                        runs=rb.ctypes.data, runs_cap=n)
    rc = fr._lib.bf_resident_commit_journal(fr._ctx, h, n, ents.ctypes.data if ents.shape[0] else None, ents.shape[0],
                                            ctypes.byref(out), None if arm is None else ctypes.byref(arm), ctypes.byref(j))
    assert rc == A.BF_OK, fr._lib.bf_last_error(fr._ctx).decode()
    got = {k: int(getattr(out, k)) for k in M.COUNT_KEYS}
    if arm is not None:
        got.update(n_armed=int(arm.n_armed), next_deadline=int(arm.next_deadline))
    items = ib.view(Frontier.COMMIT_WRITE_DTYPE)[:min(int(j.n_items), items_cap)].copy()
    runs = rb.view(np.uint32)[:int(j.n_runs_listed)].copy()
    got.update(n_items=int(j.n_items), n_runs_listed=int(j.n_runs_listed))
    return got, items, runs


def bound(L, res):
    """the items a commit of these results can list: a launched step has a phase item and at most a registered bit or an arm"""
    pc = lambda off: int(np.unpackbits(res[:, off:off + 4 * L.words]).sum()) if off != A.OFF_NONE else 0   # noqa: E731
    return max(3 * pc(L.off_ready) + pc(L.off_skip) + pc(L.off_fail), 1)


# (S, fields, parallel, runs, limiter area, run control, timer slots per run)
CASES = [(64, ALL, True, 3000, False, False, 0), (64, A.F_OUT_FAIL, True, 2000, True, False, 8),
         (256, ALL | A.F_CHILD, True, 20_000, False, True, 16), (256, A.F_DECISION | A.F_ALL_OUT, False, 4000, True, True, 0),
         (1024, ALL, True, 300, True, False, 64), (1024, A.F_ALL_OUT, False, 40, False, True, 0)]


@pytest.mark.parametrize("S,fields,parallel,n,sched,runctl,K", CASES)
def test_journal_is_the_byte_difference(fr, S, fields, parallel, n, sched, runctl, K):
    rng = np.random.default_rng(S * 13 + n + K)
    ts, slots, L, st = _batch(fr, rng, S, fields, parallel, n)
    a, b = Twin(fr, ts, slots, L, st, n + 3, sched, runctl), Twin(fr, ts, slots, L, st, n + 3, sched, runctl)
    if K:
        for tw in (a, b):
            fr.resident_timers(tw.h, K)
        timings = random_timings(rng, ts, slots)
        for slot in timings:   # at most 8 per slot, so that no run overflows; a code other than PENDING needs decision planes
            t = {s: cd for s, cd in timings[slot].items() if L.off_decision != A.OFF_NONE or cd[0] == A.DEC_PENDING}
            timings[slot] = dict(sorted(t.items())[:8])
        put_all(fr, timings)
    dead = int(slots[0])   # a dead slot: its runs have no masks and list nothing
    fr.drop_topology(dead)
    a.topo.drop(dead)
    b.topo.drop(dead)
    if runctl:
        q = np.zeros(min(n, 30), dtype=R.PUT_DTYPE)
        q["run"] = rng.choice(n, size=q.shape[0], replace=False)
        q["story_deadline"] = R.NONE
        q["drain_deadline"] = R.NONE
        q["stop"] = 2
        for tw in (a, b):
            fr.resident_runctl_put(tw.h, q)
    listed = 0
    for rnd in range(4):
        now = 100 + rnd if K else None
        res = a.tick()
        assert np.array_equal(res, b.tick())
        ents = entries_for(rng, L, a.topo, fr.resident_download(a.h, 0, n, L.state_stride), res, a.sched, n)
        before = fr.resident_download(a.h, 0, n, L.state_stride)
        t0 = fr.resident_timers_download(a.h, 0, n, K).view("<u8").copy() if K else None
        full = bound(L, res)
        if rnd == 1:   # pinned buffers
            got, items, runs = journal_pinned(fr, a.h, n, ents, now, full)
        elif rnd == 2:   # a small cap: the true count and a prefix
            got = fr.resident_commit(a.h, n, ents, now=now, journal_cap=7)
            items, runs = got.pop("items"), got.pop("runs")
        else:
            got = fr.resident_commit(a.h, n, ents, now=now, journal_cap=full)
            items, runs = got.pop("items"), got.pop("runs")
        want_b = fr.resident_commit(b.h, n, ents, now=now)
        after = fr.resident_download(a.h, 0, n, L.state_stride)
        t1 = fr.resident_timers_download(a.h, 0, n, K).view("<u8").copy() if K else None
        want_items, want_runs = J.journal(L, before, after, n, t0, t1)
        assert got.pop("n_items") == len(want_items) and got.pop("n_runs_listed") == len(want_runs) == got["n_runs_written"]
        assert got == want_b
        assert J.as_tuples(items) == want_items[:len(items)] and len(items) == min(len(want_items), 7 if rnd == 2 else full)
        assert runs.tolist() == want_runs
        if K:
            assert sum(1 for x in want_items if x[2] == J.TIMER) == got["n_armed"]
        assert np.array_equal(after, fr.resident_download(b.h, 0, n, L.state_stride))
        if K:
            assert np.array_equal(t1, fr.resident_timers_download(b.h, 0, n, K).view("<u8"))
        listed += len(want_items)
        if runctl:   # a stopped run lists nothing
            stopped = set(np.nonzero(fr.resident_runctl_download(a.h, 0, n)["stop"])[0].tolist())
            assert not stopped & {x[0] for x in want_items}
        dead_runs = set(np.nonzero(before[:, :4].view("<u4")[:, 0] == dead)[0].tolist())
        assert not dead_runs & {x[0] for x in want_items}
    if n >= 300:
        assert listed > 0


def test_refusals_and_error_runs_list_nothing(fr):
    rng = np.random.default_rng(77)
    n = 2000
    ts, slots, L, st = _batch(fr, rng, 128, ALL, True, n)
    a, b = Twin(fr, ts, slots, L, st, n), Twin(fr, ts, slots, L, st, n)
    res = a.tick()
    assert np.array_equal(res, b.tick())
    state = fr.resident_download(a.h, 0, n, L.state_stride)
    ents = entries_for(rng, L, a.topo, state, res, None, n, p_error=0)
    # a duplicated (run, step) is refused by the host, an entry on a step not launched by the device: nothing changes or is listed
    bad_dup = np.concatenate([ents, ents[:1]])
    launched = {(int(e["run"]), int(e["step"])) for e in ents}
    r0 = next(r for r in range(n) if M.masks(L, a.topo, state, res, None, r)[1])
    free = next(s for s in range(L.steps_max) if (r0, s) not in launched and not (M.masks(L, a.topo, state, res, None, r0)[1] >> s) & 1)
    bad_dev = np.concatenate([ents, np.array([(r0, free, M.HOLD, 0)], dtype=Frontier.COMMIT_DTYPE)])
    for bad in (bad_dup, bad_dev):
        out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
        items = np.zeros(64, Frontier.COMMIT_WRITE_DTYPE)
        runs = np.zeros(n, np.uint32)
        j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal), items=items.ctypes.data, items_cap=64, runs=runs.ctypes.data,
                            runs_cap=n, n_items=5, n_runs_listed=5)
        rc = fr._lib.bf_resident_commit_journal(fr._ctx, a.h, n, bad.ctypes.data, bad.shape[0], ctypes.byref(out), None, ctypes.byref(j))
        assert rc == A.BF_EINVAL and (j.n_items, j.n_runs_listed) == (0, 0) and not items.view(np.uint8).any() and not runs.any()
    for size in (0, ctypes.sizeof(A.CommitJournal) + 8):   # a wrong struct_size, and a NULL journal
        out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
        j = A.CommitJournal(struct_size=size)
        assert fr._lib.bf_resident_commit_journal(fr._ctx, a.h, n, None, 0, ctypes.byref(out), None, ctypes.byref(j)) == A.BF_EINVAL
    assert fr._lib.bf_resident_commit_journal(fr._ctx, a.h, n, None, 0, ctypes.byref(out), None, None) == A.BF_EINVAL
    j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal), items_cap=4)   # items NULL with a cap
    assert fr._lib.bf_resident_commit_journal(fr._ctx, a.h, n, None, 0, ctypes.byref(out), None, ctypes.byref(j)) == A.BF_EINVAL
    assert np.array_equal(fr.resident_download(a.h, 0, n, L.state_stride), state)
    # an ERROR entry in every launching run: those runs are neither written nor listed (runs that only skip or fail still are)
    errs = [(r, s, M.ERROR, 0) for r in range(n) for s in [next((x for x in range(L.steps_max)
                                                                 if (M.masks(L, a.topo, state, res, None, r)[1] >> x) & 1), None)]
            if s is not None]
    assert errs
    errs = np.array(errs, dtype=Frontier.COMMIT_DTYPE)
    got = fr.resident_commit(a.h, n, errs, journal_cap=bound(L, res))
    want = fr.resident_commit(b.h, n, errs)
    after = fr.resident_download(a.h, 0, n, L.state_stride)
    assert np.array_equal(after, fr.resident_download(b.h, 0, n, L.state_stride))
    want_items, want_runs = J.journal(L, state, after, n)
    assert J.as_tuples(got["items"]) == want_items and got["runs"].tolist() == want_runs
    assert {k: got[k] for k in want} == want
    assert not set(want_runs) & set(errs["run"].tolist())


@pytest.mark.parametrize("pinned", [False, True])
def test_entries_on_dead_and_too_wide_slots_are_refused(fr, pinned):
    """a run on a dead slot or on a slot wider than the layout has no masks: an entry on it is refused by the journaled commit with
    the offender bf_resident_commit names, nothing changes and nothing is listed; the ctx serves the next commit as before"""
    from bobrapet_b200.frontier import TopologySet
    rng = np.random.default_rng(23)
    n = 1500
    ts, slots, L, st = _batch(fr, rng, 64, ALL, True, n)
    wide = TopologySet([96], [0], np.zeros(97, np.uint32), np.zeros(0, np.uint16), np.full(96, A.STEP_ENGRAM, np.uint8), [0],
                       np.zeros(0, dtype=[("step", "<u2"), ("branches", "<u2"), ("allow_first", "<u4")]))
    wide_slot = int(fr.put_topologies(wide)[0])
    st = st.copy()
    st[7, :4] = np.frombuffer(np.uint32(wide_slot).tobytes(), np.uint8)   # run 7 names a slot of 3 words in a 2-word layout
    a, b = Twin(fr, ts, slots, L, st, n), Twin(fr, ts, slots, L, st, n)
    dead = int(slots[0])
    fr.drop_topology(dead)
    for tw in (a, b):
        tw.topo.drop(dead)
    res = a.tick()
    assert np.array_equal(res, b.tick())
    state = fr.resident_download(a.h, 0, n, L.state_stride)
    on_dead = int(np.nonzero(state[:, :4].copy().view("<u4")[:, 0] == dead)[0][0])
    ents = entries_for(rng, L, a.topo, state, res, None, n, p_error=0)
    for run, kind in ((on_dead, M.HOLD), (7, M.PHASE)):
        bad = np.concatenate([ents, np.array([(run, 3, kind, A.PHASE_SUCCEEDED if kind == M.PHASE else 0)],
                                             dtype=Frontier.COMMIT_DTYPE)])
        with pytest.raises(A.FrontierError) as want:
            fr.resident_commit(b.h, n, bad)
        out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
        cap = 256
        ib = fr.alloc_pinned(cap * 16) if pinned else np.zeros(cap * 16, np.uint8)
        rb = fr.alloc_pinned(n * 4) if pinned else np.zeros(n * 4, np.uint8)
        j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal), items=ib.ctypes.data, items_cap=cap, runs=rb.ctypes.data,
                            runs_cap=n)
        rc = fr._lib.bf_resident_commit_journal(fr._ctx, a.h, n, bad.ctypes.data, bad.shape[0], ctypes.byref(out), None,
                                                ctypes.byref(j))
        assert (rc, out.bad_run, out.bad_step) == (want.value.status, want.value.bad_run, want.value.bad_step)
        assert (out.bad_run, out.bad_step) == (run, 3)
        assert (j.n_items, j.n_runs_listed) == (0, 0) and not ib.any() and not rb.any()
        assert np.array_equal(fr.resident_download(a.h, 0, n, L.state_stride), state)
    got = fr.resident_commit(a.h, n, ents, journal_cap=bound(L, res))
    want_b = fr.resident_commit(b.h, n, ents)
    after = fr.resident_download(a.h, 0, n, L.state_stride)
    assert np.array_equal(after, fr.resident_download(b.h, 0, n, L.state_stride))
    want_items, want_runs = J.journal(L, state, after, n)
    assert J.as_tuples(got["items"]) == want_items and got["runs"].tolist() == want_runs and want_items
    assert {k: got[k] for k in want_b} == want_b
    assert not {on_dead, 7} & set(want_runs)
