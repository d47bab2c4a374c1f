"""bf_resident_schedule_ctxs and bf_resident_transfer_ctx on twin deployments: deployment A holds every batch in one ctx, deployment
B the same batches spread over two or three ctxs (on device 0, or on two devices when two are visible), each ctx with the Stories
put in its own order, so that slot maps are not the identity.  The same calls go to both (in-ctx ones on A, span and cross-ctx ones
on B where the batches live apart) and every output and every download is compared, with slots read as the Story they hold."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import resident_schedule_ctxs
from bobrapet_b200.records import make_layout
from tests.packing import topology_set
from tests.seqrig import random_records, story_pool

pytestmark = pytest.mark.gpu

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT
NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
K = 4          # timer slots per run
N_Q = 3        # queues


def _device_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 1


DEVS = [(0, 0), (0, 1)]


class Deployment:
    """Frontiers and the batches held in them: batch b lives in ctx home[b].  Every Story of the pool is put into every ctx, in the
    order order[c]; slot[c][k] is Story k's slot in ctx c and story[c][slot] the reverse."""

    def __init__(self, devices, home, pool, rng):
        self.frs = [Frontier(d) for d in devices]
        self.home = list(home)
        self.pool = pool
        self.slot, self.story = [], []
        for c, fr in enumerate(self.frs):
            order = list(range(len(pool))) if c == 0 and len(self.frs) == 1 else list(rng.permutation(len(pool)))
            sl = {}
            for k in order:
                sl[k] = int(fr.put_topologies(topology_set([pool[k]]))[0])
            self.slot.append(sl)
            self.story.append({s: k for k, s in sl.items()})
        self.h, self.L, self.n = [], [], []

    def fr(self, b):
        return self.frs[self.home[b]]

    def create(self, L, cap):
        b = len(self.h)
        self.h.append(self.fr(b).resident_create(L, cap))
        self.L.append(L)
        self.n.append(0)
        return b

    def close(self):
        for fr in self.frs:
            fr.close()

    def slot_map(self, c_src, c_dst):
        m = np.full(max(self.story[c_src]) + 1, A.SLOT_NONE, np.uint32)
        for s, k in self.story[c_src].items():
            m[s] = self.slot[c_dst][k]
        return m

    def records(self, b, recs_story):
        """state records whose slot word holds a Story index -> the same with this ctx's slots"""
        r = recs_story.copy()
        w = r[:, :4].view(np.uint32)
        w[:, 0] = [self.slot[self.home[b]][int(k)] for k in w[:, 0]]
        return r

    def snapshot(self, b):
        fr, h, n = self.fr(b), self.h[b], self.n[b]
        st = fr.resident_download(h, 0, n, self.L[b].state_stride).copy()
        w = st[:, :4].view(np.uint32)
        w[:, 0] = [self.story[self.home[b]].get(int(s), 0xFFFF) for s in w[:, 0]]
        return {"state": st, "timers": fr.resident_timers_download(h, 0, n, K), "sched": fr.resident_sched_download(h, 0, n),
                "runctl": fr.resident_runctl_download(h, 0, n)}


def _eq(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _eq(a[k], b[k], "%s.%s" % (what, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _eq(x, y, "%s[%d]" % (what, i))
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), what
    else:
        assert a == b, (what, a, b)


class Twins:
    """A and B, built by the same calls: three width classes (64 steps, no input planes; 256 with cond, decision, child and
    output fields; 1024 with cond, decision, child and the fail mask a commit needs with cond planes), each with timers, limiter inputs, run control and commit marks"""

    SPECS = [(64, 0), (256, COND | DEC | CHILD | OUT), (1024, COND | DEC | CHILD | A.F_OUT_FAIL)]

    def __init__(self, seed, homes, devices, sizes=(300, 200, 100), cap_extra=400):
        self.rng = np.random.default_rng(seed)
        self.pool = story_pool(self.rng, 20, 50, 2, 3)
        for p in self.pool:   # the commits here name no steps: a launched stop step would need a BF_COMMIT_PHASE entry
            stop = (p.flags & A.SF_TYPE_MASK) == A.STEP_STOP
            p.flags[stop] = (p.flags[stop] & np.uint8(0xFF ^ A.SF_TYPE_MASK)) | A.STEP_ENGRAM
        n_ctx = max(homes) + 1
        self.A = Deployment([devices[0]], [0] * len(self.SPECS), self.pool, self.rng)
        self.B = Deployment([devices[min(c, len(devices) - 1)] if c < 2 else devices[0] for c in range(n_ctx)], homes, self.pool,
                            self.rng)
        self.deps = (self.A, self.B)
        child = max(p.child_nibbles() for p in self.pool)
        self.tables = {"story_limit": np.zeros(len(self.pool), np.int32), "queue_limit": np.array([0, 40, 9], np.int32),
                       "queue_aging_s": np.array([0, 30, 5], np.int32), "global_limit": 0}
        for b, ((S, f), n) in enumerate(zip(self.SPECS, sizes)):
            L = make_layout(S, child if f & CHILD else 0, f)
            Lg = make_layout(S, child if f & CHILD else 0, f & (COND | DEC | CHILD) & ~DEC)   # no decision codes: transfers fit
            story = self.rng.integers(0, len(self.pool), n)
            recs = random_records(self.rng, Lg, [self.pool[k] for k in story], story)
            recs = _relay(Lg, L, recs)
            timers = self._timers(n, S, f)
            sched = self._sched(n, story)
            ctl = self._runctl(n)
            for d in self.deps:
                d.create(L, n + cap_extra)
                fr, h = d.fr(b), d.h[b]
                fr.resident_upload(h, 0, d.records(b, recs))
                fr.resident_timers(h, K)
                fr.resident_timers_arm(h, timers)
                fr.resident_sched(h)
                fr.resident_sched_put(h, sched)
                fr.resident_runctl(h)
                fr.resident_runctl_put(h, ctl)
                fr.resident_commit_marks(h)
                d.n[b] = n

    def _timers(self, n, S, f):
        runs = self.rng.choice(n, size=n // 3, replace=False)
        t = np.zeros(len(runs), Frontier.TIMER_DTYPE)
        t["run"] = runs
        t["step"] = self.rng.integers(0, min(S, 20), len(runs))
        t["code"] = self.rng.integers(0, 4, len(runs)) if f & DEC else A.DEC_PENDING
        t["deadline"] = self.rng.integers(10, 200, len(runs))
        return t

    def _sched(self, n, story):
        q = np.zeros(n, Frontier.SCHED_PUT_DTYPE)
        q["run"] = np.arange(n)
        q["story_key"] = story
        q["queue_key"] = self.rng.integers(0, N_Q, n)
        q["priority"] = self.rng.integers(0, 4, n)
        q["queued_since"] = np.where(self.rng.random(n) < 0.5, A.TIMER_NONE, self.rng.integers(0, 100, n))
        q["run_phase"] = 2
        return q

    def _runctl(self, n):
        runs = self.rng.choice(n, size=n // 5, replace=False)
        q = np.zeros(len(runs), Frontier.RUNCTL_PUT_DTYPE)
        q["run"] = runs
        q["story_deadline"] = np.where(self.rng.random(len(runs)) < 0.5, A.TIMER_NONE, self.rng.integers(50, 400, len(runs)))
        q["drain_deadline"] = A.TIMER_NONE
        q["stop"] = np.where(self.rng.random(len(runs)) < 0.2, A.STOP_HOST, A.STOP_NONE)
        return q

    def close(self):
        for d in self.deps:
            d.close()

    # ---- the same operation on both, outputs compared
    def compare(self, what):
        for b in range(len(self.SPECS)):
            assert self.A.n[b] == self.B.n[b]
            _eq(self.A.snapshot(b), self.B.snapshot(b), "%s: batch %d" % (what, b))

    def tick(self):
        outs = []
        for d in self.deps:
            outs.append([d.fr(b).resident_tick_touched(d.h[b], d.n[b], NONE_D, d.n[b], d.n[b] * 1024)
                         for b in range(len(self.SPECS))])
        for o in outs:
            for x in o:
                x.pop("counts")
                for k in ("runs", "head", "events"):
                    x[k] = x[k].copy()
        _eq(outs[0], outs[1], "touched tick")
        return outs[0]

    def parts(self, d):
        return [{"handle": d.h[b], "n_runs": d.n[b]} for b in range(len(self.SPECS))]

    def schedule(self, now=100):
        a = self.A.frs[0].resident_schedule(self.parts(self.A), self.tables, now)
        b = resident_schedule_ctxs(list(zip([self.B.fr(x) for x in range(len(self.SPECS))], self.parts(self.B))), self.tables, now)
        _eq(a, b, "schedule")
        return a

    def commit(self):
        outs = []
        for d in self.deps:
            outs.append([d.fr(b).resident_commit(d.h[b], d.n[b], journal_cap=1 << 16, touched=True)
                         for b in range(len(self.SPECS))])
        _eq(outs[0], outs[1], "touched commit")
        return outs[0]

    def fire(self, now):
        outs = [[d.fr(b).resident_fire(d.h[b], d.n[b], now) for b in range(len(self.SPECS))] for d in self.deps]
        _eq(outs[0], outs[1], "fire")

    def retire(self, b, runs):
        outs = []
        for d in self.deps:
            o = d.fr(b).resident_retire(d.h[b], d.n[b], runs)
            d.n[b] -= len(runs)
            outs.append(o)
        _eq(outs[0], outs[1], "retire")

    def transfer(self, s, t, runs):
        a = self.A.fr(s).resident_transfer(self.A.h[s], self.A.h[t], self.A.n[s], self.A.n[t], runs)
        B = self.B
        if B.home[s] == B.home[t]:
            b = B.fr(s).resident_transfer(B.h[s], B.h[t], B.n[s], B.n[t], runs)
        else:
            b = B.fr(s).resident_transfer_ctx(B.fr(t), B.h[s], B.h[t], B.n[s], B.n[t], runs, B.slot_map(B.home[s], B.home[t]))
        _eq(a, b, "transfer %d -> %d" % (s, t))
        for d in self.deps:
            d.n[s] -= len(runs)
            d.n[t] += len(runs)
        return b


def _relay(Lg, L, recs):
    from tests.transfer import relay_state
    return relay_state(Lg, L, recs)


def _devices(pair):
    if pair[1] >= _device_count():
        pytest.skip("a cross-device pair needs two visible GPUs")
    return pair


@pytest.mark.parametrize("pair", DEVS, ids=["dev%d%d" % p for p in DEVS])
@pytest.mark.parametrize("homes", [(0, 1, 0), (0, 1, 2)], ids=["two-ctxs", "three-ctxs"])
def test_schedule_commit_transfer_equal_one_ctx(pair, homes):
    tw = Twins(11 + sum(homes), homes, _devices(pair))
    try:
        tw.compare("setup")
        tw.tick()
        tw.schedule()
        tw.commit()
        tw.compare("after commit")
        for s, t in ((0, 1), (0, 2), (1, 2)):
            runs = tw.rng.choice(tw.A.n[s], size=min(37, tw.A.n[s]), replace=False).astype(np.uint32)
            out = tw.transfer(s, t, runs)
            assert out["dst_n_runs"] == tw.A.n[t]
            tw.compare("after transfer %d -> %d" % (s, t))
            # the arrivals carry the destination's slot of their Story
            B = tw.B
            st = B.fr(t).resident_download(B.h[t], B.n[t] - len(runs), len(runs), B.L[t].state_stride)
            assert all(int(x) in B.story[B.home[t]] for x in st[:, :4].view(np.uint32)[:, 0])
            tw.tick()
            tw.schedule()
            tw.commit()
            tw.compare("after the next commit")
    finally:
        tw.close()


@pytest.mark.parametrize("pair", DEVS, ids=["dev%d%d" % p for p in DEVS])
def test_shared_story_limit_binds_across_ctxs(pair):
    """a Story limit that is full only with every ctx's Running steps counted: the span schedule queues what one schedule of A
    queues, where per-ctx schedules would launch it"""
    devs = _devices(pair)
    scout = Twins(71, (0, 1, 0), devs)   # the Running totals, from a schedule without limits
    try:
        scout.tick()
        running = scout.A.frs[0].resident_schedule(scout.parts(scout.A), scout.tables, 100)["story_running"]
    finally:
        scout.close()
    # each Story's limit is its Running count over every batch plus one: each run of it may launch one step, no more
    limits = running.astype(np.int32) + 1
    tw, third = Twins(71, (0, 1, 0), devs), Twins(71, (0, 1, 0), devs)   # the span schedule, the per-ctx schedules
    try:
        for t in (tw, third):
            t.tables["story_limit"] = limits
            t.tick()
        a = tw.schedule()   # the first schedule of each batch lists every run
        launched = sum(int(p["heads"]["n_launch"].sum()) for p in a["parts"])
        assert all(p["full"] for p in a["parts"])
        B = third.B
        per_ctx = 0
        for c in range(len(B.frs)):
            bs = [b for b in range(len(Twins.SPECS)) if B.home[b] == c]
            o = B.frs[c].resident_schedule([{"handle": B.h[b], "n_runs": B.n[b]} for b in bs], third.tables, 100)
            per_ctx += sum(int(p["heads"]["n_launch"].sum()) for p in o["parts"])
        assert per_ctx > launched, "the limits do not bind across ctxs: the case would pass vacuously"
        tw.commit()
        tw.compare("after the limited commit")
    finally:
        tw.close()
        third.close()


def _allow_failure_variant(p):
    """the Story p with SF_ALLOW_FAILURE flipped on its step 0: a topology record of the same size and other bytes"""
    import dataclasses
    flags = p.flags.copy()
    flags[0] ^= A.SF_ALLOW_FAILURE
    return dataclasses.replace(p, flags=flags)


def _record(p):
    """the packed topology record of Story p, built on the host (bf_topology_record_build)"""
    import ctypes as C
    lib = A.load()
    ts = topology_set([p])
    desc = ts.descriptors()
    n = C.c_uint32()
    assert lib.bf_topology_record_build(desc.ctypes.data_as(C.POINTER(A.Topology)), None, 0, C.byref(n)) == A.BF_ENOMEM   # the size only
    buf = np.zeros(n.value, np.uint8)
    assert lib.bf_topology_record_build(desc.ctypes.data_as(C.POINTER(A.Topology)), buf.ctypes.data, n.value, C.byref(n)) == A.BF_OK
    return buf


def _downloads(tw):
    return [tw.B.snapshot(b) for b in range(len(Twins.SPECS))]


def _refused(fn, reason=None):
    with pytest.raises(A.FrontierError) as ei:
        fn()
    assert ei.value.status == A.BF_EINVAL
    if reason is not None:
        assert ei.value.unfit_reason == reason, ei.value
    return ei.value


@pytest.mark.parametrize("pair", DEVS, ids=["dev%d%d" % p for p in DEVS])
def test_refusals_leave_both_ctxs_byte_identical(pair):
    tw = Twins(91, (0, 1, 0), _devices(pair))
    B = tw.B
    try:
        tw.tick()
        tw.schedule()
        f0, f1 = B.frs
        m = B.slot_map(0, 1)
        before = _downloads(tw)
        # an unfit run: a non-PASS cond code cannot move into the 64-step batch without cond planes (batch 1 -> batch 0)
        f1.resident_apply(B.h[1], np.array([(5, 0, A.DELTA_COND, A.COND_SKIP)], dtype=Frontier.DELTA_DTYPE))
        tw.A.fr(1).resident_apply(tw.A.h[1], np.array([(5, 0, A.DELTA_COND, A.COND_SKIP)], dtype=Frontier.DELTA_DTYPE))
        tw.tick()
        before = _downloads(tw)
        m10 = B.slot_map(1, 0)
        e = _refused(lambda: f1.resident_transfer_ctx(f0, B.h[1], B.h[0], B.n[1], B.n[0], [5], m10), A.UNFIT_LAYOUT)
        assert e.unfit == 0
        _eq(before, _downloads(tw), "unfit run")
        # unmapped and past-the-map slots
        st = f0.resident_download(B.h[0], 0, 1, B.L[0].state_stride)
        s0 = int(st[0, :4].view(np.uint32)[0])
        um = m.copy()
        um[s0] = A.SLOT_NONE
        _refused(lambda: f0.resident_transfer_ctx(f1, B.h[0], B.h[1], B.n[0], B.n[1], [0], um), A.UNFIT_SLOT_UNMAPPED)
        _refused(lambda: f0.resident_transfer_ctx(f1, B.h[0], B.h[1], B.n[0], B.n[1], [0], m[:s0]), A.UNFIT_SLOT_PAST_MAP)
        _eq(before, _downloads(tw), "unmapped slot")
        # a mapped slot whose destination record differs: map it onto another Story's slot
        k0 = B.story[0][s0]
        other = next(B.slot[1][k] for k in range(len(tw.pool)) if tw.pool[k].S != tw.pool[k0].S)
        bad = m.copy()
        bad[s0] = other
        _refused(lambda: f0.resident_transfer_ctx(f1, B.h[0], B.h[1], B.n[0], B.n[1], [0], bad))
        # a record of the same size with other bytes: the Story with one more step allowed to fail, put into ctx 1 alone
        twin = _allow_failure_variant(tw.pool[k0])
        assert _record(twin).size == _record(tw.pool[k0]).size and _record(twin).tobytes() != _record(tw.pool[k0]).tobytes()
        same_size = m.copy()
        same_size[s0] = int(f1.put_topologies(topology_set([twin]))[0])
        _refused(lambda: f0.resident_transfer_ctx(f1, B.h[0], B.h[1], B.n[0], B.n[1], [0], same_size))
        dead_dst = m.copy()
        dead_dst[s0] = 0xFFFF
        _refused(lambda: f0.resident_transfer_ctx(f1, B.h[0], B.h[1], B.n[0], B.n[1], [0], dead_dst))
        _eq(before, _downloads(tw), "bad map entries")
        # the same ctx twice
        _refused(lambda: f0.resident_transfer_ctx(f0, B.h[0], B.h[2], B.n[0], B.n[2], [0], B.slot_map(0, 0)))
        # a bad struct_size
        import ctypes as C
        t = A.CtxTransfer(struct_size=C.sizeof(A.CtxTransfer) - 8, src_n_runs=B.n[0], dst_n_runs=B.n[1], n=0)
        assert f0._lib.bf_resident_transfer_ctx(f0._ctx, B.h[0], f1._ctx, B.h[1], C.byref(t)) == A.BF_EINVAL
        _eq(before, _downloads(tw), "same ctx, struct_size")
        # a dead slot in the source: its Story dropped from ctx 0 while run 0 still holds it
        f0.drop_topology(s0)
        _refused(lambda: f0.resident_transfer_ctx(f1, B.h[0], B.h[1], B.n[0], B.n[1], [0], m), A.UNFIT_SLOT_DEAD)
        _eq(before, _downloads(tw), "dead slot")
    finally:
        tw.close()


@pytest.mark.parametrize("pair", DEVS, ids=["dev%d%d" % p for p in DEVS])
def test_schedule_refusals_change_nothing(pair):
    tw = Twins(93, (0, 1, 0), _devices(pair))
    B = tw.B
    try:
        tw.tick()
        ps = list(zip([B.fr(b) for b in range(3)], tw.parts(B)))
        with pytest.raises(A.FrontierError):   # a batch twice
            resident_schedule_ctxs(ps + [ps[0]], tw.tables, 100)
        import ctypes as C
        call_ps = (A.CtxSchedPart * 1)()
        call_ps[0] = A.CtxSchedPart(struct_size=C.sizeof(A.CtxSchedPart) + 8, ctx=B.frs[0]._ctx)
        out = A.SchedOut(struct_size=C.sizeof(A.SchedOut))
        t = A.SchedTables(struct_size=C.sizeof(A.SchedTables))
        assert B.frs[0]._lib.bf_resident_schedule_ctxs(C.byref(t), 100, call_ps, 1, C.byref(out)) == A.BF_EINVAL
        # a part whose state changed since its tick: refused on its ctx, and nothing scheduled on the other
        B.fr(1).resident_apply(B.h[1], np.array([(2, 1, A.DELTA_PHASE, 3)], dtype=Frontier.DELTA_DTYPE))
        with pytest.raises(A.FrontierError):
            resident_schedule_ctxs(ps, tw.tables, 100)
        tw.A.fr(1).resident_apply(tw.A.h[1], np.array([(2, 1, A.DELTA_PHASE, 3)], dtype=Frontier.DELTA_DTYPE))
        tw.tick()
        tw.schedule()   # the refused calls left no schedule baseline behind: the first schedule of both sides is alike
        tw.commit()
        tw.compare("after refusals")
    finally:
        tw.close()


@pytest.mark.parametrize("pair", DEVS, ids=["dev%d%d" % p for p in DEVS])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_sequences(seed, pair):
    tw = Twins(500 + seed, (0, 1, 0) if seed != 1 else (0, 1, 2), _devices(pair), sizes=(200, 150, 80))
    rng = np.random.default_rng(900 + seed)
    now = 0
    try:
        tw.tick()
        for step in range(14):
            op = rng.choice(["tick", "fire", "transfer", "retire", "cycle"])
            if op == "fire":
                now += int(rng.integers(10, 80))
                tw.fire(now)
                tw.tick()
            elif op == "transfer":
                s, t = (int(x) for x in rng.choice(3, size=2, replace=False))
                if t == 0:   # the 64-step class holds no cond or decision codes: move into it only runs that never had any
                    s, t = t, s
                n = tw.A.n[s]
                if n > 1:
                    tw.transfer(s, t, rng.choice(n, size=int(rng.integers(1, min(n, 30) + 1)), replace=False).astype(np.uint32))
                tw.tick()
            elif op == "retire":
                b = int(rng.integers(0, 3))
                n = tw.A.n[b]
                if n > 1:
                    tw.retire(b, rng.choice(n, size=int(rng.integers(1, min(n, 10) + 1)), replace=False).astype(np.uint32))
                tw.tick()
            elif op == "cycle":
                tw.tick()
                tw.schedule(now + 100)
                tw.commit()
            else:
                tw.tick()
            tw.compare("seed %d step %d (%s)" % (seed, step, op))
        tw.tick()
        tw.schedule(now + 100)
        tw.commit()
        tw.compare("seed %d end" % seed)
    finally:
        tw.close()
