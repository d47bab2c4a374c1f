"""bf_resident_schedule against bf_schedule and the host model (tests/sched_resident.py): parity after every tick kind, several
batches of different layouts under one set of totals, the reference's limiter known answers, edges, every refusal, the inputs
through every lifecycle call, and the launch counts of batches without the area."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import make_layout, pack_state
from tests import randgen
from tests import sched_resident as SRM
from tests import schedref as SR

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)


@pytest.fixture(scope="module")
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _batch(rng, fr, n, smax, smin=1, parallel=True, count=30, fields=A.F_COND | A.F_DECISION):
    ts = randgen.random_topologies(rng, count, smin, smax, parallel=parallel)
    slots = fr.put_topologies(ts)
    L, state, topo = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
    return ts, slots, L, state, topo


def _inputs(rng, n, ns, nq, now, edges=True):
    p = SRM.defaults(n)
    p["run"] = np.arange(n)
    s = SR.random_sched(rng, n, ns, nq, edges=edges, out_of_range=0.05)
    for f in ("story_key", "queue_key", "priority", "run_phase"):
        p[f] = s[f]
    since = rng.integers(0, now + 200, size=n).astype(np.uint32)
    if edges:
        e = rng.random(n) < 0.2
        since[e] = rng.choice(np.array([0, 1, now - 1, now, now + 1, SRM.NONE], np.uint32), size=int(e.sum()))
    since[rng.random(n) < 0.25] = SRM.NONE
    p["queued_since"] = since
    return p


def _deltas(rng, ts, topo, n, k):
    runs = rng.choice(n, size=k, replace=False)
    d = np.zeros(k, Frontier.DELTA_DTYPE)
    d["run"] = runs
    d["index"] = [int(rng.integers(0, int(ts.S[int(topo[r])]))) for r in runs]
    d["field"] = A.DELTA_PHASE
    d["code"] = rng.choice([0, 1, 2, 2, 3, 14], size=k)
    return d


class Resident:
    """a resident batch with its limiter inputs and its model twin"""

    def __init__(self, fr, L, state, cap, descs):
        self.fr, self.L, self.descs = fr, L, descs
        self.h = fr.resident_create(L, cap)
        fr.resident_upload(self.h, 0, state)
        fr.resident_sched(self.h)
        self.model = SRM.Batch(L, cap)
        self.n = state.shape[0]

    def put(self, req):
        self.fr.resident_sched_put(self.h, req)
        self.model.put(req)

    def current(self, flags=0, max_iterations=0):
        """the device's state records and what a pass over them gives (the current result records the ticks left)"""
        st = self.fr.resident_download(self.h, 0, self.n, self.L.state_stride)
        res, _ = self.fr.eval(self.L, st, flags=flags, max_iterations=max_iterations)
        return st, res

    def close(self):
        self.fr.resident_destroy(self.h)


def _schedule(fr, batches, tables, now, caps=None, cur=None):
    """the device schedule and the model's, compared: totals, listed runs, heads and events.  cur: each batch's (state, result)
    when a pass over the current state would not give the result records its last tick left"""
    parts = [dict(handle=b.h, n_runs=b.n, **(caps[i] if caps else {})) for i, b in enumerate(batches)]
    got = fr.resident_schedule(parts, tables, now)
    cur = cur or [b.current() for b in batches]
    want = SRM.schedule([(b.model, b.n, st, res, b.descs) for b, (st, res) in zip(batches, cur)], tables, now)
    for k in ("story_running", "queue_running", "queue_max_priority"):
        assert np.array_equal(got[k], want[k]), k
    assert got["global_running"] == want["global_running"]
    for i, (g, w) in enumerate(zip(got["parts"], want["parts"])):
        assert g["n_listed"] == w["listed"].size and g["n_events"] == w["n_events"] and g["full"] == w["full"], (i, g["n_listed"], w["listed"].size)
        nl = g["runs"].size
        assert np.array_equal(g["runs"], w["listed"][:nl]), i
        hv = np.stack([g["heads"][f] for f in g["heads"].dtype.names], axis=1) if nl else np.zeros((0, 4), np.uint32)
        assert np.array_equal(hv, w["heads"][:nl]), i
        assert np.array_equal(g["events"], w["events"][:g["events"].size]), i
    return got, want, cur


# ------------------------------------------------------------------------------------------ parity with bf_schedule
@pytest.mark.parametrize("kind", ["dense", "compact", "changed", "touched", "fixpoint"])
def test_parity_with_bf_schedule(fr, kind):
    rng = np.random.default_rng(100 + len(kind))
    n = 3000
    ts, slots, L, state, topo = _batch(rng, fr, n, 180)
    descs = SR.from_topology_set(ts, slots)
    now = 50_000
    tables = SR.random_tables(rng, 40, 5, n, maxprio_base=True)
    b = Resident(fr, L, state, n + 100, descs)
    try:
        inp = _inputs(rng, n, 40, 5, now)
        b.put(inp)
        cache = None
        for step in range(3):
            dd = NONE_D if step == 0 else _deltas(rng, ts, topo, n, 60)
            flags = A.EVAL_FIXPOINT if kind == "fixpoint" else 0
            if kind in ("dense", "fixpoint"):
                fr.resident_tick(b.h, L, n, dd, flags=flags, max_iterations=4 if flags else 0)
            elif kind == "compact":
                fr.resident_tick_compact(b.h, n, dd, 1 << 22)
            elif kind == "changed":
                fr.resident_tick_compact(b.h, n, dd, 1 << 22, flags=A.EVAL_CHANGED_ONLY)
            else:
                out = fr.resident_tick_touched(b.h, n, dd, n, 1 << 22)
                assert bool(out["full"]) == (step == 0)
            got = fr.resident_schedule([dict(handle=b.h, n_runs=n)], tables, now + 7 * step)
            p = got["parts"][0]
            if step == 0:
                assert p["full"] == 1 and p["n_listed"] == n
                cache = SRM.decode(L.words, n, p["runs"], p["heads"], p["events"])
            else:   # the cache updated from the listed runs alone
                upd = SRM.decode(L.words, n, p["runs"], p["heads"], p["events"])
                cache[p["runs"].astype(np.int64)] = upd[p["runs"].astype(np.int64)]
            want = fr.schedule(L, n, SRM.sched_runs(inp, now + 7 * step), **tables)
            assert np.array_equal(cache, want["records"]), "%s step %d" % (kind, step)
            for k in ("story_running", "queue_running", "queue_max_priority"):
                assert np.array_equal(got[k], want[k]), k
            assert got["global_running"] == want["global_running"]
            # and the listed set is the model's
            st, res = b.current(flags, 4 if flags else 0)
            w = SRM.schedule([(b.model, n, st, res, descs)], tables, now + 7 * step)["parts"][0]
            assert np.array_equal(p["runs"], w["listed"])
    finally:
        b.close()


# ------------------------------------------------------------------------------------------ several batches
@pytest.mark.parametrize("shapes", [((64, True), (1024, False)), ((64, False), (256, True), (1024, True))])
def test_several_batches(fr, shapes):
    rng = np.random.default_rng(sum(s for s, _ in shapes))
    now = 10_000
    tables = SR.random_tables(rng, 30, 4, 5000, maxprio_base=True)
    bs = []
    try:
        for smax, par in shapes:
            n = int(rng.integers(500, 1500))
            ts, slots, L, state, topo = _batch(rng, fr, n, smax, smin=max(1, smax - 40), parallel=par)
            b = Resident(fr, L, state, n, SR.from_topology_set(ts, slots))
            b.put(_inputs(rng, n, 30, 4, now))
            fr.resident_tick_compact(b.h, n, NONE_D, 1 << 22)
            bs.append(b)
        got, want, cur = _schedule(fr, bs, tables, now)
        # each batch equals bf_schedule with the other batches' contributions as bases
        for i, (b, (st, res)) in enumerate(zip(bs, cur)):
            t = dict(tables)
            sr_, qr_, gl_, mp_ = (np.asarray(tables["story_running_base"], np.int64), np.asarray(tables["queue_running_base"], np.int64),
                                  int(tables["global_running_base"]), np.asarray(tables["queue_max_priority_base"], np.int32))
            for j, (o, (sto, reso)) in enumerate(zip(bs, cur)):
                if j == i:
                    continue
                e = SR.expected(o.L, sto, reso, o.descs, SRM.sched_runs(o.model.inputs[:o.n], now),
                                {**tables, "story_running_base": None, "queue_running_base": None, "global_running_base": 0,
                                 "queue_max_priority_base": None})
                sr_ += e["story_running"]; qr_ += e["queue_running"]; gl_ += e["global_running"]
                mp_ = np.maximum(mp_, e["queue_max_priority"])
            t.update(story_running_base=(sr_ % (1 << 32)).astype(np.uint32), queue_running_base=(qr_ % (1 << 32)).astype(np.uint32),
                     global_running_base=gl_ % (1 << 32), queue_max_priority_base=mp_)
            fr.resident_eval(b.h, b.L, b.n)
            one = fr.schedule(b.L, b.n, SRM.sched_runs(b.model.inputs[:b.n], now), **t)
            assert np.array_equal(one["records"], want["parts"][i]["records"]), i
            assert np.array_equal(one["story_running"], got["story_running"]) and one["global_running"] == got["global_running"]
        # a second schedule with nothing changed lists nothing
        got2, _, _ = _schedule(fr, bs, tables, now)
        assert all(p["n_listed"] == 0 for p in got2["parts"])
    finally:
        for b in bs:
            b.close()


# ------------------------------------------------------------------------------------------ the reference's known answers
def _kat_batch(fr, phases):
    """runs of a 2-step engram topology without needs; phases[r] = the two step phase codes"""
    ts = TopologySet(S=[2], E=[0], row_ptr=[0, 0, 0], col_idx=np.zeros(0, np.uint16), step_flags=[0, 0])
    slot = fr.put_topologies(ts)
    L = make_layout(2, 0, 0)
    n = len(phases)
    state = pack_state(L, np.full(n, slot[0], np.uint32), np.zeros(n, np.uint8), np.asarray(phases, np.uint8))
    b = Resident(fr, L, state, n, SR.from_topology_set(ts, slot))
    fr.resident_tick(b.h, L, n, NONE_D)
    return b


def _put(b, rows):
    req = SRM.defaults(len(rows))
    for i, (run, sk, qk, prio, since, ph) in enumerate(rows):
        req[i] = (run, sk, qk, prio, since, ph, (0, 0))
    b.put(req)


def test_kat_priority_blocks_lower_priority(fr):
    """dag_test.go:528: high (prio 10, Running) blocks low (prio 1, Pending) in the same queue"""
    b = _kat_batch(fr, [[3, 3], [0, 0]])
    try:
        _put(b, [(0, SRM.NONE, 0, 10, SRM.NONE, A.PHASE_RUNNING), (1, SRM.NONE, 0, 1, SRM.NONE, A.PHASE_PENDING)])
        t = dict(story_limit=np.zeros(0, np.int32), queue_limit=[0], queue_aging_s=[60])
        got, _, _ = _schedule(fr, [b], t, 1000)
        h = got["parts"][0]["heads"]
        assert h["n_launch"][1] == 0 and h["n_queued_sched"][1] == 2 and h["reason"][1] == A.QUEUED_PRIORITY
    finally:
        b.close()


@pytest.mark.parametrize("queued_for, launched", [(120, True), (59, False)])
def test_kat_aged_run(fr, queued_for, launched):
    """dag_test.go:579: low (prio 1) queued 2 minutes under 60 s aging reaches 3 > 2; at 59 s it stays blocked"""
    b = _kat_batch(fr, [[3, 3], [0, 0]])
    try:
        now = 10_000
        _put(b, [(0, SRM.NONE, 0, 2, SRM.NONE, A.PHASE_RUNNING), (1, SRM.NONE, 0, 1, now - queued_for, A.PHASE_PENDING)])
        t = dict(story_limit=np.zeros(0, np.int32), queue_limit=[0], queue_aging_s=[60])
        got, _, _ = _schedule(fr, [b], t, now)
        h = got["parts"][0]["heads"]
        assert (h["n_launch"][1] == 2) == launched
    finally:
        b.close()


def test_kat_story_concurrency(fr):
    """dag_test.go:744: story limit 1 with one Running StepRun: the other run's two ready steps are both queued"""
    b = _kat_batch(fr, [[2, 3], [0, 0]])
    try:
        _put(b, [(0, 0, SRM.NONE, 0, SRM.NONE, A.PHASE_RUNNING), (1, 0, SRM.NONE, 0, SRM.NONE, A.PHASE_RUNNING)])
        t = dict(story_limit=[1], queue_limit=np.zeros(0, np.int32), queue_aging_s=np.zeros(0, np.int32))
        got, _, _ = _schedule(fr, [b], t, 5)
        h = got["parts"][0]["heads"]
        assert h["n_launch"][1] == 0 and h["n_queued_story"][1] == 2 and got["story_running"][0] == 1
    finally:
        b.close()


# ------------------------------------------------------------------------------------------ edges
def test_edges(fr):
    """n_runs = 0, runs never put (defaults), dead slots, a topology drop between tick and schedule, caps below the lists"""
    rng = np.random.default_rng(9)
    n = 1200
    ts, slots, L, state, topo = _batch(rng, fr, n, 300)
    descs = SR.from_topology_set(ts, slots)
    tables = SR.random_tables(rng, 10, 3, n, maxprio_base=True)
    b = Resident(fr, L, state, n, descs)
    try:
        b.put(_inputs(rng, n // 2, 10, 3, 100))   # the rest keep the defaults
        fr.resident_tick_compact(b.h, n, NONE_D, 1 << 22)
        got = fr.resident_schedule([dict(handle=b.h, n_runs=0)], tables, 100)
        assert got["parts"][0]["full"] == 1 and got["parts"][0]["n_listed"] == 0
        assert np.array_equal(got["queue_max_priority"], tables["queue_max_priority_base"])
        _schedule(fr, [b], tables, 100, caps=[dict(runs_cap=37, events_cap=101)])     # caps smaller than the lists
        cur = [b.current()]
        fr.drop_topology(int(slots[3]))          # a drop between tick and schedule: its runs count nothing, their results stay
        b.descs = {s: d for s, d in descs.items() if s != int(slots[3])}
        _schedule(fr, [b], tables, 100, cur=cur)
        _schedule(fr, [b], tables, 0xFFFFFFFE, cur=cur)                               # elapsed past INT32_MAX
    finally:
        b.close()


# ------------------------------------------------------------------------------------------ refusals
def _snapshot(fr, b):
    return fr.resident_download(b.h, 0, b.model.cap, b.L.state_stride), fr.resident_sched_download(b.h, 0, b.model.cap)


def test_refusals(fr):
    rng = np.random.default_rng(12)
    n = 400
    ts, slots, L, state, topo = _batch(rng, fr, n, 100)
    descs = SR.from_topology_set(ts, slots)
    tables = SR.random_tables(rng, 10, 3, n)
    b = Resident(fr, L, state, n + 50, descs)
    plain = fr.resident_create(L, n)
    try:
        b.put(_inputs(rng, n, 10, 3, 100))
        fr.resident_tick_compact(b.h, n, NONE_D, 1 << 22)
        _schedule(fr, [b], tables, 100)
        before = _snapshot(fr, b)

        def refused(parts, now=100, t=tables):
            with pytest.raises(A.FrontierError) as e:
                fr.resident_schedule(parts, t, now)
            assert e.value.status == A.BF_EINVAL
            after = _snapshot(fr, b)
            assert all(np.array_equal(x, y) for x, y in zip(before, after))

        refused([dict(handle=b.h, n_runs=n), dict(handle=b.h, n_runs=n)])           # a duplicate handle
        refused([dict(handle=plain, n_runs=n)])                                       # no inputs area
        refused([dict(handle=999, n_runs=1)])                                         # unknown batch
        refused([dict(handle=b.h, n_runs=n + 51)])                                    # n_runs past the capacity
        refused([dict(handle=b.h, n_runs=n + 1)])                                     # no tick over n + 1 runs
        refused([dict(handle=b.h, n_runs=n)], now=SRM.NONE)
        for bad in ([(n + 50, 0, 0, 0, 0, 0, (0, 0))], [(0, 0, 0, 0, 0, 0, (1, 0))], [(1, 0, 0, 0, 0, 0, (0, 0))] * 2):
            with pytest.raises(A.FrontierError):
                fr.resident_sched_put(b.h, np.array(bad, SRM.PUT_DTYPE))
            assert all(np.array_equal(x, y) for x, y in zip(before, _snapshot(fr, b)))
        with pytest.raises(A.FrontierError):
            fr.resident_sched_put(plain, np.array([(0, 0, 0, 0, 0, 0, (0, 0))], SRM.PUT_DTYPE))
        # the baselines survived every refusal: nothing listed
        assert _schedule(fr, [b], tables, 100)[0]["parts"][0]["n_listed"] == 0
        def fire_writing():
            """a due sleep timer on a Running step whose decision is still PENDING: the fire writes its code"""
            dd = np.array([(4, 0, A.DELTA_PHASE, A.PHASE_RUNNING), (4, 0, A.DELTA_DECISION, A.DEC_PENDING)], Frontier.DELTA_DTYPE)
            fr.resident_tick_compact(b.h, n, dd, 1 << 22)
            fr.resident_timers(b.h, 1)
            fr.resident_timers_arm(b.h, np.array([(4, 0, A.DEC_SUCCEED, 0, 1, 0)], Frontier.TIMER_DTYPE))
            assert fr.resident_fire(b.h, n, 5)["n_written"] == 1

        # after each state-changing call, no schedule until a tick
        d = _deltas(rng, ts, topo, n, 5)
        calls = [("apply", lambda: fr.resident_apply(b.h, d)),
                 ("upload", lambda: (fr.resident_upload(b.h, 3, state[3:5]), b.model.upload(3, 2))),
                 ("redrive", lambda: fr.resident_redrive(b.h, np.array([(1, int(slots[topo[1]]), A.REDRIVE_ALL, 0)], Frontier.REDRIVE_DTYPE))),
                 ("fire", fire_writing)]
        for name, call in calls:
            call()
            before = _snapshot(fr, b)
            refused([dict(handle=b.h, n_runs=n)])
            fr.resident_tick_compact(b.h, n, NONE_D, 1 << 22)
            _schedule(fr, [b], tables, 100)
            before = _snapshot(fr, b)
        # a put alone needs no tick
        b.put(np.array([(7, 1, 1, 3, 50, 2, (0, 0))], SRM.PUT_DTYPE))
        got, _, _ = _schedule(fr, [b], tables, 100)
    finally:
        b.close()
        fr.resident_destroy(plain)


# ------------------------------------------------------------------------------------------ the inputs through the lifecycle
def test_lifecycle(fr):
    rng = np.random.default_rng(21)
    now = 500
    tables = SR.random_tables(rng, 12, 3, 3000, maxprio_base=True)
    ts1, sl1, L1, st1, topo1 = _batch(rng, fr, 800, 60)
    ts2, sl2, L2, st2, topo2 = _batch(rng, fr, 600, 250, smin=100)
    d1, d2 = SR.from_topology_set(ts1, sl1), SR.from_topology_set(ts2, sl2)
    a = Resident(fr, L1, st1, 1000, {**d1, **d2})
    c = Resident(fr, L2, st2, 1000, {**d1, **d2})
    try:
        a.put(_inputs(rng, 800, 12, 3, now))
        c.put(_inputs(rng, 600, 12, 3, now))

        def needs_tick(b):
            """no schedule of b until a tick, and the refusal changes nothing"""
            before = _snapshot(fr, b)
            with pytest.raises(A.FrontierError):
                fr.resident_schedule([dict(handle=a.h, n_runs=a.n), dict(handle=c.h, n_runs=c.n)], tables, now)
            assert all(np.array_equal(x, y) for x, y in zip(before, _snapshot(fr, b)))

        def tick_and_schedule():
            for b in (a, c):
                fr.resident_tick_compact(b.h, b.n, NONE_D, 1 << 22)
            return _schedule(fr, [a, c], tables, now)

        tick_and_schedule()
        # retire: moved runs carry their inputs, vacated indices get the defaults
        gone = rng.choice(800, size=60, replace=False)
        m, mf, mt = fr.resident_retire(a.h, 800, gone)
        moves = a.model.retire(800, gone)
        assert sorted(moves) == sorted(zip(mf.tolist(), mt.tolist()))
        a.n = m
        got_in, want_in = fr.resident_sched_download(a.h, 0, 1000), a.model.download(0, 1000)
        for f in ("run", "story_key", "queue_key", "priority", "queued_since", "run_phase"):
            assert np.array_equal(got_in[f], want_in[f]), f
        needs_tick(a)
        tick_and_schedule()
        # transfer a -> c: inputs arrive with their runs
        runs = rng.choice(a.n, size=40, replace=False)
        arriving = a.model.inputs[runs].copy()
        t = fr.resident_transfer(a.h, c.h, a.n, c.n, runs)
        a.model.retire(a.n, runs)
        c.model.receive(c.n, arriving)
        a.n, c.n = t["src_n_runs"], t["dst_n_runs"]
        needs_tick(a)
        needs_tick(c)
        tick_and_schedule()
        # a destination without an area refuses a source that has one, both batches byte-identical
        plain = fr.resident_create(L2, 1000)
        before = _snapshot(fr, a)
        with pytest.raises(A.FrontierError):
            fr.resident_transfer(a.h, plain, a.n, 0, [0])
        assert all(np.array_equal(x, y) for x, y in zip(before, _snapshot(fr, a)))
        fr.resident_destroy(plain)
        tick_and_schedule()
        # reshape to more steps and a larger capacity: defaults for the new runs, no baselines (words changed)
        L1b = make_layout(L2.steps_max, L1.child_nibbles, L1.fields)
        fr.resident_reshape(a.h, L1b, 1200)
        a.model.resize(1200)
        a.model.relayout(L1b)
        a.L = L1b
        needs_tick(a)
        got, _, _ = tick_and_schedule()
        assert got["parts"][0]["full"] == 1
        # narrow back: the area stays
        fr.resident_narrow(a.h, L1, a.n)
        a.model.relayout(L1)
        a.L = L1
        needs_tick(a)
        got, _, _ = tick_and_schedule()
        assert got["parts"][0]["full"] == 1
        assert tick_and_schedule()[0]["parts"][0]["n_listed"] == 0
        # redrive: the inputs stay and nothing but changed records is listed
        fr.resident_redrive(c.h, np.array([(2, int(fr.resident_download(c.h, 2, 1, L2.state_stride)[0, :4].view("<u4")[0]), A.REDRIVE_ALL, 0)],
                                          Frontier.REDRIVE_DTYPE))
        needs_tick(c)
        tick_and_schedule()
        # migrate: the migrated runs lose their baselines
        slot = int(fr.resident_download(c.h, 0, 1, L2.state_stride)[0, :4].view("<u4")[0])
        S = int(ts2.S[list(sl2).index(slot)]) if slot in list(sl2) else int(ts1.S[list(sl1).index(slot)])
        new_ts = TopologySet(S=[S], E=[0], row_ptr=np.zeros(S + 1, np.uint32), col_idx=np.zeros(0, np.uint16), step_flags=np.zeros(S, np.uint8))
        new_slot = int(fr.put_topologies(new_ts)[0])
        c.descs = {**c.descs, **SR.from_topology_set(new_ts, [new_slot])}
        st_c = fr.resident_download(c.h, 0, c.n, L2.state_stride)
        on = np.nonzero(st_c[:, :4].copy().view("<u4")[:, 0] == slot)[0]
        # the new generation has no parallel step, so no branch count can change: the migration goes through
        assert on.size > 0 and fr.resident_migrate(c.h, slot, new_slot, np.arange(S, dtype=np.uint16), c.n) == on.size
        c.model.lose_baseline(on)
        needs_tick(c)
        got, _, _ = tick_and_schedule()
        assert set(on.tolist()) <= set(got["parts"][1]["runs"].tolist())
    finally:
        a.close()
        c.close()


# ------------------------------------------------------------------------------------------ launch counts
def test_launch_counts_without_the_area(fr):
    """every lifecycle call launches the same on a batch with the area as on one without; put and schedule launch 1 and 1 + 4"""
    rng = np.random.default_rng(33)
    ts, slots, L, state, topo = _batch(rng, fr, 300, 80)
    counts = []
    for with_area in (False, True):
        h = fr.resident_create(L, 400)
        h2 = fr.resident_create(L, 400)
        fr.resident_upload(h, 0, state)
        if with_area:
            fr.resident_sched(h)
            fr.resident_sched(h2)
        seq = []

        def launches(call):
            before = fr.stats()["kernel_launches"]
            call()
            seq.append(fr.stats()["kernel_launches"] - before)

        launches(lambda: fr.resident_tick_compact(h, 300, NONE_D, 1 << 22))
        launches(lambda: fr.resident_upload(h, 10, state[10:20]))
        launches(lambda: fr.resident_apply(h, _deltas(np.random.default_rng(1), ts, topo, 300, 10)))
        launches(lambda: fr.resident_retire(h, 300, [4, 8, 299]))
        launches(lambda: fr.resident_transfer(h, h2, 297, 0, [0, 1]))
        launches(lambda: fr.resident_reshape(h, make_layout(L.steps_max + 40, L.child_nibbles, L.fields), 500))
        launches(lambda: fr.resident_narrow(h, L, 295))
        launches(lambda: fr.resident_tick_touched(h, 295, NONE_D, 295, 1 << 20))
        slot = int(fr.resident_download(h, 0, 1, L.state_stride)[0, :4].view("<u4")[0])
        S = int(ts.S[list(slots).index(slot)])
        flat = TopologySet(S=[S], E=[0], row_ptr=np.zeros(S + 1, np.uint32), col_idx=np.zeros(0, np.uint16), step_flags=np.zeros(S, np.uint8))
        new_slot = int(fr.put_topologies(flat)[0])
        launches(lambda: fr.resident_migrate(h, slot, new_slot, np.arange(S, dtype=np.uint16), 295))
        launches(lambda: fr.resident_redrive(h, np.array([(0, new_slot, A.REDRIVE_ALL, 0), (7, new_slot, 1, 0)], Frontier.REDRIVE_DTYPE)))
        launches(lambda: fr.resident_timers(h, 2))
        launches(lambda: fr.resident_timers_arm(h, np.array([(3, 0, A.DEC_SUCCEED, 0, 4, 0)], Frontier.TIMER_DTYPE)))
        launches(lambda: fr.resident_fire(h, 295, 9))
        launches(lambda: fr.resident_tick_touched(h, 295, NONE_D, 295, 1 << 20))
        counts.append(seq)
        if with_area:
            before = fr.stats()["kernel_launches"]
            fr.resident_sched_put(h, np.array([(1, 0, 0, 0, 0, 0, (0, 0))], SRM.PUT_DTYPE))
            fr.resident_schedule([dict(handle=h, n_runs=295)], dict(story_limit=[1], queue_limit=[1], queue_aging_s=[1]), 5)
            assert fr.stats()["kernel_launches"] - before == 1 + 1 + 4
        fr.resident_destroy(h)
        fr.resident_destroy(h2)
    assert counts[0] == counts[1], counts
