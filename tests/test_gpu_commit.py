"""Tick commits of a resident batch on the device (bf_resident_commit) against the host model tests/commit.py, byte for byte: the
state records, the counts and the touched runs (the next touched tick evaluates exactly them).  Also: batches with a limiter area
(the launches and queue marks of the last schedule), runs stopped by run control, dead slots, every refusal (records, timers and
the touched bookkeeping unchanged), launch counts, the commit loop against one BF_EVAL_FIXPOINT pass on the device, and a commit
after every other resident call (refused until a tick comes between)."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import commit as M
from tests import randgen
from tests import runctl as R
from tests.test_host_commit import PINNED, differences, no_stops, seeded_batch
from bobrapet_b200.records import unpack_result

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
TABLES = dict(story_limit=[3, 0, 0, 0], queue_limit=[0, 4, 0], queue_aging_s=[0, 60, 10], global_limit=0)   # <= 0: no limit


def _batch(fr, rng, S, fields, parallel, n, stops=True):
    """random topologies of at most S steps on the device and n runs of them -> (topologies, slots, layout, records)"""
    ts = randgen.random_topologies(rng, 12, max(2, S // 2), S, max_deg=4, parallel=parallel, fill=0.5)
    ts = ts if stops else no_stops(ts)
    slots = fr.put_topologies(ts)
    L, st, _ = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
    return ts, slots, L, st


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def entries_for(rng, L, topo, state, result, sched, n, p_hold=0.05, p_error=0.03):
    """random HOLD / ERROR entries on launched steps, and a PHASE entry for every other launched stop step"""
    out = []
    for r in range(n):
        t, launched, _q, _s, _f = M.masks(L, topo, state, result, sched, r)
        if not launched:
            continue
        steps = [s for s in range(launched.bit_length()) if (launched >> s) & 1]
        named = {}
        if rng.random() < p_error:
            named[int(rng.choice(steps))] = (M.ERROR, 0)
        elif rng.random() < p_hold:
            named[int(rng.choice(steps))] = (M.HOLD, 0)
        for s in steps:
            if (t["stop"] >> s) & 1 and s not in named:
                named[s] = (M.PHASE, int(rng.integers(A.PHASE_PENDING, A.PHASE_SKIPPED + 1)))
        out += [(r, s, k, c) for s, (k, c) in named.items()]
    rng.shuffle(out)
    return np.array(out, dtype=Frontier.COMMIT_DTYPE) if out else np.zeros(0, Frontier.COMMIT_DTYPE)


class Twin:
    def __init__(self, fr, ts, slots, L, st, cap, sched=False, runctl=False):
        self.fr, self.L, self.n = fr, L, st.shape[0]
        self.topo = M.Topologies(ts, slots)
        self.h = fr.resident_create(L, cap)
        if self.n:
            fr.resident_upload(self.h, 0, st)
        self.sched = None
        if sched:
            fr.resident_sched(self.h)
            rng = np.random.default_rng(self.n)
            q = np.zeros(self.n, dtype=Frontier.SCHED_PUT_DTYPE)
            q["run"] = np.arange(self.n)
            q["story_key"] = rng.integers(0, 4, self.n)
            q["queue_key"] = rng.integers(0, 3, self.n)
            q["priority"] = rng.integers(0, 5, self.n)
            q["queued_since"] = A.SCHED_NONE
            q["run_phase"] = A.PHASE_RUNNING
            if self.n:
                fr.resident_sched_put(self.h, q)
            self.sched = {}
        if runctl:
            fr.resident_runctl(self.h)
            self.area = R.defaults(cap)
        self.state = fr.resident_download(self.h, 0, cap, L.state_stride)

    def tick(self, now=100):
        """a dense single-pass tick (and a schedule) -> the current result records"""
        res = self.fr.resident_tick(self.h, self.L, self.n, NONE_D)[0]
        if self.sched is not None:
            out = self.fr.resident_schedule([dict(handle=self.h, n_runs=self.n, runs_cap=self.n, events_cap=BIG)], TABLES, now)
            M.sched_rows(self.L, out["parts"][0], self.sched)
        return res

    def commit(self, res, ents, n=None):
        n = self.n if n is None else n
        want = M.commit(self.L, self.topo, self.state, res, self.sched, n, ents)
        if want[0]:
            with pytest.raises(A.FrontierError) as e:
                self.fr.resident_commit(self.h, n, ents)
            assert (e.value.bad_run, e.value.bad_step) == (want[1], want[2]), (str(e.value), want[1:3])
        else:
            got = self.fr.resident_commit(self.h, n, ents)
            assert got == want[3], (got, want[3])
        self.check()
        return want

    def check(self):
        got = self.fr.resident_download(self.h, 0, self.state.shape[0], self.L.state_stride)
        assert np.array_equal(got, self.state), np.nonzero(np.any(got != self.state, axis=1))[0][:10]

    def touched_tick(self):
        return self.fr.resident_tick_touched(self.h, self.n, NONE_D, max(self.n, 1), BIG)


# (S, fields, parallel, runs, limiter area, run control)
CASES = [(64, ALL, False, 700, False, False), (64, A.F_OUT_FAIL, True, 3000, True, False), (256, ALL, True, 30_000, False, True),
         (256, A.F_DECISION | A.F_ALL_OUT, False, 5000, True, True), (1024, ALL, True, 300, True, False), (1024, A.F_ALL_OUT, False, 1, False, False),
         (64, ALL, True, 0, True, False)]


@pytest.mark.parametrize("S,fields,parallel,n,sched,runctl", CASES)
def test_commits_match_the_model(fr, S, fields, parallel, n, sched, runctl):
    rng = np.random.default_rng(S + n + fields)
    ts, slots, L, st = _batch(fr, rng, S, fields, parallel, n)
    tw = Twin(fr, ts, slots, L, st, n + 5, sched, runctl)
    if runctl and n:
        q = np.zeros(min(n, 50), dtype=R.PUT_DTYPE)
        q["run"] = rng.choice(n, size=q.shape[0], replace=False)
        q["story_deadline"] = R.NONE
        q["drain_deadline"] = R.NONE
        q["stop"] = 2
        fr.resident_runctl_put(tw.h, q)
        R.put(tw.area, tw.state, q)
    for rnd in range(3):
        res = tw.tick()
        ents = entries_for(rng, L, tw.topo, tw.state, res, tw.sched, n)
        rc, _, _, counts, touched = tw.commit(res, ents)
        assert rc == 0
        if runctl and n:
            stopped = set(np.nonzero(tw.area["stop"][:n])[0].tolist())
            assert not (touched & stopped)
        t = tw.touched_tick()
        assert t["full"] == 0 and t["n_evaluated"] == len(touched), (t["n_evaluated"], len(touched))
    # a commit that wrote ends the tick: the next commit is refused until a tick comes between
    res = tw.tick()
    ents = entries_for(rng, L, tw.topo, tw.state, res, tw.sched, n, p_hold=0, p_error=0)
    if tw.commit(res, ents)[3]["n_runs_written"]:
        with pytest.raises(A.FrontierError) as e:
            fr.resident_commit(tw.h, n, ents)
        assert (e.value.bad_run, e.value.bad_step) == (M.NONE, M.NONE)
        tw.check()


def test_dead_slots_get_nothing(fr):
    """a slot dropped between a tick and its commit refuses the commit; after a tick the runs on it get nothing"""
    rng = np.random.default_rng(11)
    ts, slots, L, st = _batch(fr, rng, 64, ALL, True, 2000)
    tw = Twin(fr, ts, slots, L, st, 2000)
    res = tw.tick()
    dead = int(slots[0])
    fr.drop_topology(dead)
    tw.topo.drop(dead)
    ents = entries_for(rng, L, tw.topo, tw.state, res, None, 2000, p_error=0)
    with pytest.raises(A.FrontierError) as e:
        fr.resident_commit(tw.h, 2000, ents)
    assert (e.value.bad_run, e.value.bad_step) == (M.NONE, M.NONE) and "slot" in str(e.value)
    tw.check()
    res = tw.tick()
    ents = entries_for(rng, L, tw.topo, tw.state, res, None, 2000, p_error=0)
    rc, _, _, counts, touched = tw.commit(res, ents)
    assert rc == 0 and counts["n_runs_written"] > 0
    on_dead = set(np.nonzero(tw.state[:, :4].copy().view("<u4")[:, 0] == dead)[0].tolist())
    assert on_dead and not (touched & on_dead)


def test_refusals_change_nothing(fr):
    rng = np.random.default_rng(13)
    n = 1500
    ts, slots, L, st = _batch(fr, rng, 128, ALL, True, n)
    tw = Twin(fr, ts, slots, L, st, n, sched=True)
    fr.resident_timers(tw.h, 2)
    tq = np.zeros(3, dtype=Frontier.TIMER_DTYPE)
    tq[:] = [(0, 1, 1, 0, 500, 0), (1, 2, 3, 0, 600, 0), (2, 0, 0, 0, 700, 0)]
    fr.resident_timers_arm(tw.h, tq)
    timers = fr.resident_timers_download(tw.h, 0, n, 2)

    def refused(call, bad=(M.NONE, M.NONE)):
        with pytest.raises(A.FrontierError) as e:
            call()
        assert (e.value.bad_run, e.value.bad_step) == bad, str(e.value)
        tw.check()
        assert np.array_equal(fr.resident_timers_download(tw.h, 0, n, 2), timers)

    refused(lambda: fr.resident_commit(tw.h, n))   # no tick yet
    fr.resident_tick(tw.h, L, n, NONE_D)
    refused(lambda: fr.resident_commit(tw.h, n))   # a limiter area and no schedule
    res = tw.tick()
    refused(lambda: fr.resident_commit(tw.h, n + 1))   # n_runs past the capacity
    ents = entries_for(rng, L, tw.topo, tw.state, res, tw.sched, n, p_hold=0.2, p_error=0)
    assert len(ents) > 3
    for bad in ("run", "step", "kind", "code", "dup", "not-launched"):
        e = ents.copy()
        if bad == "run":
            e[1]["run"] = n
        elif bad == "step":
            e[1]["step"] = L.steps_max
        elif bad == "kind":
            e[1]["kind"] = 0
        elif bad == "code":
            e[1]["kind"], e[1]["code"] = M.PHASE, 15
        elif bad == "dup":
            e = np.concatenate([e, e[1:2]])
            e[-1]["kind"], e[-1]["code"] = M.ERROR, 0
        else:
            res_ready = [r for r in range(n) if M.masks(L, tw.topo, tw.state, res, tw.sched, r)[1] == 0 and
                         M.masks(L, tw.topo, tw.state, res, tw.sched, r)[0] is not None]
            e[1] = (res_ready[0], 0, M.HOLD, 0)
        want = M.check(L, tw.topo, tw.state, res, tw.sched, n, [tuple(x) for x in e])
        assert want[0] == M.EINVAL
        refused(lambda: fr.resident_commit(tw.h, n, e), want[1:])
    # the device's offences: a PHASE entry on a step that is not a stop step, a launched stop step without an entry, and that
    # offence against an entry on a step not launched in the same run (the lower step wins either way)
    stops = [i for i, x in enumerate(ents) if x["kind"] == M.PHASE]
    holds = [i for i, x in enumerate(ents) if x["kind"] == M.HOLD and not (tw.topo.by_slot[int(tw.state[x["run"], :4].view("<u4")[0])]["stop"] >> int(x["step"])) & 1]
    assert stops and holds
    cases = []
    e = ents.copy()
    e[holds[0]]["kind"], e[holds[0]]["code"] = M.PHASE, A.PHASE_SUCCEEDED
    cases.append(e)
    cases.append(np.delete(ents, stops[0]))
    for i in stops:
        r, s0 = int(ents[i]["run"]), int(ents[i]["step"])
        t, launched = M.masks(L, tw.topo, tw.state, res, tw.sched, r)[:2]
        named = {int(x["step"]) for x in ents if int(x["run"]) == r}
        idle = [q for q in range(t["S"]) if not (launched >> q) & 1 and q not in named]
        for q in (min(idle, default=None), max(idle, default=None)):
            if q is not None:
                cases.append(np.concatenate([np.delete(ents, i), np.array([(r, q, M.HOLD, 0)], dtype=Frontier.COMMIT_DTYPE)]))
    assert len(cases) >= 4
    for e in cases:
        want = M.check(L, tw.topo, tw.state, res, tw.sched, n, [tuple(x) for x in e])
        assert want[0] == M.EINVAL
        refused(lambda: fr.resident_commit(tw.h, n, e), want[1:])
    # NULL entries with n > 0
    out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
    assert fr._lib.bf_resident_commit(fr._ctx, tw.h, n, None, 3, ctypes.byref(out)) == A.BF_EINVAL
    assert (out.bad_run, out.bad_step) == (M.NONE, M.NONE)
    tw.check()
    assert tw.touched_tick()["n_evaluated"] == 0   # no refusal touched a run
    # a fixpoint tick, a delta and a layout with cond planes and no fail mask
    fr.resident_tick(tw.h, L, n, NONE_D, flags=A.EVAL_FIXPOINT)
    fr.resident_schedule([dict(handle=tw.h, n_runs=n)], TABLES, 100)
    refused(lambda: fr.resident_commit(tw.h, n))
    tw.tick()
    d = np.zeros(1, dtype=Frontier.DELTA_DTYPE)
    d[0] = (0, 0, A.DELTA_COND, 0)
    fr.resident_apply(tw.h, d)
    tw.state = fr.resident_download(tw.h, 0, n, L.state_stride)
    refused(lambda: fr.resident_commit(tw.h, n))
    assert tw.touched_tick()["n_evaluated"] == 1   # the delta's run alone: no refusal touched a run
    from bobrapet_b200.records import make_layout
    L2 = make_layout(64, 0, A.F_COND)
    h2 = fr.resident_create(L2, 4)
    fr.resident_tick(h2, L2, 4, NONE_D)
    with pytest.raises(A.FrontierError):
        fr.resident_commit(h2, 4)


def _launches(fr, call):
    before = fr.stats()["kernel_launches"]
    call()
    return fr.stats()["kernel_launches"] - before


def test_launch_counts(fr):
    """a commit is two launches (check, apply) and none over no runs; the tick before it launches what it did before"""
    rng = np.random.default_rng(17)
    n = 400
    _ts, _slots, L, st = _batch(fr, rng, 64, A.F_ALL_OUT, False, n, stops=False)
    a = fr.resident_create(L, n)
    b = fr.resident_create(L, n)
    fr.resident_upload(a, 0, st)
    fr.resident_upload(b, 0, st)
    assert _launches(fr, lambda: fr.resident_tick(a, L, n, NONE_D)) == _launches(fr, lambda: fr.resident_tick(b, L, n, NONE_D))
    assert _launches(fr, lambda: fr.resident_commit(a, n)) == 2
    fr.resident_tick(a, L, 0, NONE_D)
    assert _launches(fr, lambda: fr.resident_commit(a, 0)) == 0


@pytest.mark.parametrize("key", [k for k in PINNED if k[3] == 2000])
def test_commit_loop_matches_one_fixpoint_pass_on_the_device(fr, key):
    """the device form of test_host_commit.test_commit_loop_matches_one_fixpoint_pass: exact agreement but for the pinned runs"""
    ts, L, st, topo_of = seeded_batch(*key)
    slots = fr.put_topologies(ts)
    st[:, :4] = np.ascontiguousarray(slots[topo_of], dtype="<u4").view(np.uint8).reshape(-1, 4)
    n = st.shape[0]
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    W = 32 * L.words
    ready = np.zeros((n, W), bool)
    skip = np.zeros_like(ready)
    for _ in range(key[0] + 2):
        u = unpack_result(L, fr.resident_tick(h, L, n, NONE_D)[0], W)
        ready |= u["ready"]
        skip |= u["skip"]
        if fr.resident_commit(h, n)["n_runs_written"] == 0:
            break
    else:
        raise AssertionError("the commit loop did not settle")
    assert fr.resident_commit(h, n)["n_runs_written"] == 0   # a commit that wrote nothing keeps the tick: idempotent
    f = unpack_result(L, fr.eval(L, st, flags=A.EVAL_FIXPOINT)[0], W)
    assert differences(st, ready, skip, u, f) == PINNED[key]
