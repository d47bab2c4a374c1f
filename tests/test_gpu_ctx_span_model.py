"""bf_resident_transfer_ctx and bf_resident_schedule_ctxs against the host models, on ctxs of device 0 (or of two devices when two
are visible), each ctx with its Stories put in its own order so that no slot map is the identity:
  - every (source, destination) side-area set pair against tests/lifecycle.py, refusals included;
  - the baseline mark the gather stages, the ticks after a move, the slot maps and every refusal against tests/transfer.py;
  - the gather at every launch shape (moved runs around CTA boundaries, timer slots past one lane sweep, state strides below and
    above one vector per lane) and at scale, against the same calls within one ctx;
  - the span schedule against one model schedule (tests/sched_resident.py) over every part of every ctx: table bases that wrap,
    negative and wrapping priorities, keys past the tables, limits that bind only across ctxs, and part layouts."""
import copy
import ctypes as C

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import resident_schedule_ctxs
from bobrapet_b200.records import make_layout, pack_state
from tests import randgen
from tests import redrive as RD
from tests import sched_resident as SRM
from tests import schedref as SR
from tests import timers as T
from tests.lifecycle import RUNCTL, SCHED, TIMERS, Refused, area_sets, records_of, subset_name, template_records
from tests.narrowing import baseline_runs, numpy_extent
from tests.seqrig import random_records, story_pool
from tests.test_gpu_ctx_span import Deployment, _devices, _eq
from tests.test_gpu_run_areas import FIELDS, MOVED, NOW, TABLES, Twin
from tests.transfer import TransferRig, fits, relay_state
from tests import reshape as RS

pytestmark = pytest.mark.gpu

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT
NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
DEVS = [(0, 0), (0, 1)]
DEV_IDS = ["dev%d%d" % p for p in DEVS]
SETS = area_sets()
SET_IDS = [subset_name(s, k) for s, k in SETS]
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


def _map(live_src, live_dst, length=None):
    """the slot map of two registries ({slot: Story}): each live source slot -> the destination slot of its Story"""
    at = {k: s for s, k in live_dst.items()}
    m = np.full(length or max(live_src) + 1, A.SLOT_NONE, np.uint32)
    for s, k in live_src.items():
        if k in at:
            m[s] = at[k]
    return m


def _refused(fn):
    with pytest.raises(A.FrontierError) as ei:
        fn()
    assert ei.value.status == A.BF_EINVAL
    return ei.value


# ================================================================================== 2. every side-area pair against lifecycle.py
class CtxEnv:
    """one ctx of the area rig: test_gpu_run_areas's two Stories, put after `spare` other topologies in `order`"""

    def __init__(self, fr, ts1, order, spare=()):
        self.fr = fr
        for t in spare:
            fr.put_topologies(t)
        self.slots = [0, 0]
        for k in order:
            self.slots[k] = int(fr.put_topologies(ts1[k])[0])
        self.live = {s: k for k, s in enumerate(self.slots)}
        self.L = make_layout(64, 0, FIELDS)
        self.S = [int(t.S[0]) for t in ts1]
        self.descs = {}
        for k in range(2):
            self.descs.update(SR.from_topology_set(ts1[k], [self.slots[k]]))
        self.templates = template_records(self.L, self.slots, self.S)

    def records(self, n):
        return records_of(self.templates, n)


def _area_envs(pair):
    d0, d1 = _devices(pair)
    ts1 = [randgen.random_topologies(np.random.default_rng(4242 + k), 1, 20, 24, parallel=False) for k in range(2)]
    spare = [randgen.random_topologies(np.random.default_rng(17), 1, 5, 8, parallel=False)]
    f0, f1 = Frontier(d0), Frontier(d1)
    return CtxEnv(f0, ts1, [0, 1]), CtxEnv(f1, ts1, [1, 0], spare)


def span_schedule(twins):
    """a dense tick of each batch, then one bf_resident_schedule_ctxs over those with limiter inputs, compared with the model"""
    twins = [t for t in twins if t.m.sched is not None]
    if not twins:
        return []
    cur = []
    for t in twins:
        st = np.ascontiguousarray(t.m.state[:t.n])
        res, _ = t.fr.resident_tick(t.h, t.m.L, t.n, NONE_D)
        cur.append((st, res))
    got = resident_schedule_ctxs([(t.fr, dict(handle=t.h, n_runs=t.n)) for t in twins], TABLES, NOW)
    want = SRM.schedule([(t.m.sched, t.n, st, res, t.env.descs) for t, (st, res) in zip(twins, cur)], TABLES, NOW)
    _compare_schedule(got, want)
    return [set(w["listed"].tolist()) for w in want["parts"]]


def _compare_schedule(got, want, what=""):
    for k in ("story_running", "queue_running", "queue_max_priority"):
        assert np.array_equal(got[k], want[k]), "%s %s: %s, want %s" % (what, k, got[k][:8], want[k][:8])
    assert got["global_running"] == want["global_running"], what
    assert len(got["parts"]) == len(want["parts"])
    for i, (g, w) in enumerate(zip(got["parts"], want["parts"])):
        assert np.array_equal(g["runs"], w["listed"]), "%s part %d lists %s, the model %s" % (what, i, g["runs"][:10].tolist(),
                                                                                             w["listed"][:10].tolist())
        hv = np.stack([g["heads"][f] for f in g["heads"].dtype.names], axis=1) if g["runs"].size else np.zeros((0, 4), np.uint32)
        assert np.array_equal(hv, w["heads"]) and np.array_equal(g["events"], w["events"]), "%s part %d" % (what, i)
        assert g["full"] == w["full"] and g["n_events"] == w["n_events"], "%s part %d" % (what, i)


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
@pytest.mark.parametrize("src_set", SETS, ids=SET_IDS)
def test_transfer_every_area_pair(pair, src_set):
    """test_gpu_run_areas.test_transfer_every_destination_set with the destination in another ctx: every destination set, K
    down and up, destinations with entries past their runs; each refusal with the model's unfit, BF_UNFIT_LAYOUT and both ctxs
    byte-identical; then both batches over their whole capacity, and a span schedule of both"""
    e0, e1 = _area_envs(pair)
    m01 = _map(e0.live, e1.live)
    assert not np.array_equal(m01, np.arange(m01.size))
    refused = set()
    try:
        for dst_set in SETS:
            a, b = Twin(e0, *src_set), Twin(e1, *dst_set, n=4, beyond=True)
            try:
                what = "%s -> %s" % (subset_name(*src_set), subset_name(*dst_set))
                moved = MOVED
                try:
                    a.m.transfer(b.m, b.n, moved, slot_map=m01)
                    want = None
                except Refused as e:
                    want = e
                if want is not None:
                    before = a.snapshot(), b.snapshot()
                    got = _refused(lambda: e0.fr.resident_transfer_ctx(e1.fr, a.h, b.h, a.n, b.n, moved, m01))
                    assert got.unfit == want.unfit, (what, got.unfit, want.unfit)
                    assert (a.snapshot(), b.snapshot()) == before, "%s: a refused transfer changed a ctx" % what
                    if want.unfit == A.EXTENT_NO_RUN:
                        assert got.unfit_reason == A.UNFIT_NONE, what
                        refused.add("sched")
                        continue
                    assert got.unfit_reason == A.UNFIT_LAYOUT, (what, got.unfit_reason)
                    r = moved[want.unfit]
                    armed = len(T.armed(a.m.timers[r])) if a.m.timers is not None else 0
                    msg = str(got)
                    assert ("%d timer slot(s) of the destination's %d" % (armed, b.m.K)) in msg, (what, msg)
                    assert ("run-control area" in msg) == ("runctl" in want.lost), (what, msg)
                    refused |= want.lost
                    moved = [r for r in MOVED if not a.m.lost_by(b.m, r)]
                    a.m.transfer(b.m, b.n, moved, slot_map=m01)
                src_n, dst_n = a.n + len(moved), b.n - len(moved)
                out = e0.fr.resident_transfer_ctx(e1.fr, a.h, b.h, src_n, dst_n, moved, m01)
                assert (out["src_n_runs"], out["dst_n_runs"]) == (a.n, b.n), what
                a.check(what + " (source)")
                b.check(what + " (destination)")
                listed = span_schedule([a, b])
                if b.m.sched is not None:   # the arrivals carry no schedule baseline
                    assert set(range(dst_n, b.n)) <= listed[-1], what
            finally:
                e0.fr.resident_destroy(a.h)
                e1.fr.resident_destroy(b.h)
    finally:
        e0.fr.close()
        e1.fr.close()
    src, k = src_set
    if src & TIMERS and k == 5:
        assert "timers" in refused
    if src & RUNCTL:
        assert "runctl" in refused
    if src & SCHED:
        assert "sched" in refused


# ================================================================================== 3 and 5. against tests/transfer.py
def _pool(rng):
    """Stories of 10-20 steps, their edits and spares of 5-12 steps, and a wide one of 56 steps (last)"""
    pool = story_pool(rng, 10, 20, 2, 3)
    for p in pool[6:]:
        assert p.S <= 40
    big = RD.packed_story(RD.random_story(rng, "wide-", 56, 2))
    return pool + [big]


class Pair:
    """two TransferRigs over one pool, on two ctxs; the second puts the Stories in another order"""

    def __init__(self, pair, seed, label):
        d0, d1 = _devices(pair)
        self.rng = np.random.default_rng(seed)
        self.pool = _pool(self.rng)
        self.r = []
        try:
            for c, d in enumerate((d0, d1)):
                self.r.append(TransferRig(Frontier(d), self.pool, label + " ctx%d" % c))
        except BaseException:
            self.close()
            raise
        for k in range(len(self.pool)):
            self.r[0].put(k)
        for k in self.rng.permutation(len(self.pool)):
            self.r[1].put(int(k))
        self.child = max(p.child_nibbles() for p in self.pool)
        self.Ls = make_layout(64, self.child, COND | DEC | CHILD | OUT)
        self.Ld = make_layout(24, self.child, COND | DEC | CHILD | OUT)
        self.Lg = make_layout(64, self.child, COND | DEC | CHILD)

    def slot_of(self, c, k):
        return next(s for s, j in self.r[c].reg.live.items() if j == k)

    def slot_map(self, length=None):
        return _map(self.r[0].reg.live, self.r[1].reg.live, length)

    def records(self, stories, c=0):
        """state records of runs of the given pool Stories in ctx c's slots, codes within each Story's steps"""
        slots = [self.slot_of(c, k) for k in stories]
        return relay_state(self.Lg, self.Ls, random_records(self.rng, self.Lg, [self.pool[k] for k in stories], slots))

    def blank(self, k, c=0):
        """the state record of a run of pool Story k in ctx c that has not started: every code 0"""
        W = 32 * self.Ls.words
        z = np.zeros((1, W), np.uint8)
        return pack_state(self.Ls, np.array([self.slot_of(c, k)], np.uint32), np.zeros(1, np.uint8), z, z, z)

    def close(self):
        for r in self.r:
            r.destroy()
            r.fr.close()


def _extent_counted(b, r, n_runs, T, counted):
    """the extent of run r alone with its current result record counted or not"""
    reg = b.reg
    S = {s: reg.stories[k].S for s, k in reg.live.items()}
    Cn = {s: reg.stories[k].child_nibbles() for s, k in reg.live.items()}
    names = [nm for nm, _ in RS.RESULT_FIELDS if getattr(T, nm) != A.OFF_NONE]
    return numpy_extent(b.L, b.state[r:r + 1], b.cur[r:r + 1], 1, S, Cn, names, {0} if counted else set())


STATES = ["changed", "touched", "uploaded", "rewritten"]


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
@pytest.mark.parametrize("state", STATES)
def test_baselines_and_ticks_after_a_move(pair, state):
    """runs leave a source in each baseline state: after a changed-only tick, after a touched tick, uploaded since the tick,
    and rewritten since the tick (by a delta; a commit's writes mark a run the same way, touched and not to be listed
    regardless), below and above its changed-only run count in one call.  The staged baseline mark decides whether a run's
    current result record counts in the fit: a run re-uploaded on a narrow Story over a record a wide Story left must fit
    (counted, it would not), a baseline run whose slot now holds a narrow Story must not (uncounted, it would).  In the
    rewritten state that run is in no changed-only baseline, so only its even touched mark keeps it in the baseline.  After
    each move, touched and changed-only ticks of both ctxs list what the model lists"""
    P = Pair(pair, 300 + STATES.index(state), "baselines %s" % state)
    r0, r1 = P.r
    wide = len(P.pool) - 1
    n0, n_up, n_dst = 40, 12, 9
    try:
        # A1 / B1 take touched ticks, A2 / B2 changed-only ones; the sources tick over their first n0 runs only
        A1, A2 = r0.create(P.Ls, 80), r0.create(P.Ls, 80)
        B1, B2 = r1.create(P.Ld, 80), r1.create(P.Ld, 80)
        n = n0 + n_up
        stories = [wide if r in (3, 4, 17, 21) else int(P.rng.integers(0, 6)) for r in range(n)]
        recs = P.records(stories)
        for r in (3, 4, 17, 21):   # not started: their state fits any width, their result records hold the wide Story's ready steps
            recs[r] = P.blank(wide)[0]
        drec = relay_state(P.Ls, P.Ld, P.records([int(x) for x in P.rng.integers(0, 6, n_dst)], 1))
        for r, b, kind, k in ((r0, A1, "changed" if state == "changed" else "touched", n0), (r0, A2, "changed", n0),
                              (r1, B1, "touched", n_dst), (r1, B2, "changed", n_dst)):
            r.upload(b, 0, recs if r is r0 else drec)
            r.tick(b, kind, k)
        if state == "uploaded":
            for a in (A1, A2):
                r0.upload(a, 10, P.records([2]))

        def move(runs):
            nonlocal n, n_dst
            for a, b in ((A1, B1), (A2, B2)):
                out = r0.transfer_ctx(r1, a, b, n, n_dst, runs, P.slot_map())
                assert out is not None and out["dst_n_runs"] == n_dst + len(runs)
            n, n_dst = n - len(runs), n_dst + len(runs)
            o = r1.tick(B1, "touched", n_dst)
            assert o["full"] == 0 and set(range(n_dst - len(runs), n_dst)) <= set(o["runs"].tolist())
            r0.tick(A1, "touched", n)
            r1.tick(B2, "changed", n_dst)
            r0.tick(A2, "changed", n)

        # (i) runs below and above the ticked ones in one call
        move([0, 30, 8, n0 + 2, n0 + 7])
        # (ii) a wide run re-uploaded on a narrow Story: uploaded since the tick, its wide result record must not count
        slot = lambda a, r: int(np.ascontiguousarray(a.state[r, 0:4]).view("<u4")[0])  # noqa: E731
        s_wide = P.slot_of(0, wide)
        w = [r for r in range(n) if slot(A1, r) == s_wide]
        assert len(w) >= 2 and all(slot(A2, r) == s_wide for r in w)
        for a in (A1, A2):
            r0.upload(a, w[0], P.records([1]))
        for a in (A1, A2):
            assert not fits(_extent_counted(a, w[0], n, P.Ld, True), P.Ld), "the case would not see a mark of 0"
            assert fits(_extent_counted(a, w[0], n, P.Ld, False), P.Ld)
        move([w[0], 1])
        # back into the source's layout
        r1.transfer_ctx(r0, B1, A1, n_dst, n, [n_dst - 1, 2], _map(r1.reg.live, r0.reg.live))
        r0.tick(A1, "touched", n + 2)
        r1.tick(B1, "touched", n_dst - 2)
        # (iii) the wide Story's slot dropped and put again for a narrow Story: a baseline run on it keeps its wide result
        # record, which counts, so it does not fit; uncounted it would
        narrow = next(k for k in range(6) if P.pool[k].S <= 24)
        r0.drop(s_wide)
        assert r0.put(narrow) == s_wide
        refused = []
        for a, b, na, nb in ((A1, B1, n + 2, n_dst - 2), (A2, B2, n, n_dst)):
            r = next(r for r in range(na) if slot(a, r) == s_wide)
            if state == "rewritten":
                # another run re-uploaded (no changed-only baseline is left), then run r rewritten: its mark is touched, even
                u = next(x for x in range(1, na) if x != r and slot(a, x) != s_wide)
                r0.upload(a, u, P.records([2]))
                d = np.zeros(1, Frontier.DELTA_DTYPE)
                d["run"], d["index"], d["field"], d["code"] = r, 0, A.DELTA_PHASE, A.PHASE_RUNNING
                r0.apply(a, d)
                assert not a.prev_valid and r in a.touched and r not in a.must
            if r in baseline_runs(a, na):
                assert fits(_extent_counted(a, r, na, P.Ld, False), P.Ld)
                assert not fits(_extent_counted(a, r, na, P.Ld, True), P.Ld)
            out = r0.transfer_ctx(r1, a, b, na, nb, [0, r], P.slot_map())
            refused.append(out is None)
        assert any(refused), "no baseline run keeps a record that counts: a mark of 3 would go unseen"
        if state == "rewritten":
            assert refused[0], "the rewritten run is not in the touched baseline: its even mark would go unseen"
    finally:
        P.close()


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
def test_slot_maps_and_refusals(pair):
    """slot maps longer than the source's slot table, entries no moved run uses (live source slot: checked; dead: ignored), a
    source slot dropped and reused by another Story, an arena compaction in either ctx before the call; every refusal of one
    ctx's transfer across two; unfit runs of different kinds at different positions.  Each call against the model, both ctxs
    compared with their models after it"""
    P = Pair(pair, 77, "slot maps")
    r0, r1 = P.r
    n, n_dst = 30, 5
    wide = len(P.pool) - 1
    try:
        a, b = r0.create(P.Ls, n + 4), r1.create(P.Ld, n_dst + 12)
        stories = [wide if r in (2, 9) else int(P.rng.integers(0, 6)) for r in range(n)]
        r0.upload(a, 0, P.records(stories))
        r1.upload(b, 0, relay_state(P.Ls, P.Ld, P.records([0] * n_dst, 1)))
        r0.tick(a, "touched", n)
        r1.tick(b, "touched", n_dst)
        m = P.slot_map()
        slot = lambda r: int(np.ascontiguousarray(a.state[r, 0:4]).view("<u4")[0])  # noqa: E731
        narrow = [r for r in range(n) if stories[r] != wide]
        u = next(r for r in narrow[3:] if slot(r) not in {slot(x) for x in narrow[:3]})
        # the wide runs (2, 9) do not fit 24 steps (BF_UNFIT_LAYOUT); run u's slot unmapped
        um = m.copy()
        um[slot(u)] = A.SLOT_NONE
        for runs, unfit, why in (([2, narrow[0], narrow[1], u], 0, A.UNFIT_LAYOUT), ([u, narrow[0], narrow[1], 9], 0, A.UNFIT_SLOT_UNMAPPED),
                                 ([narrow[0], narrow[1], narrow[2], 9, u], 3, A.UNFIT_LAYOUT),
                                 ([narrow[0], narrow[1], narrow[2], u, 2], 3, A.UNFIT_SLOT_UNMAPPED)):
            r0.transfer_ctx(r1, a, b, n, n_dst, runs, um)
            e = _refused(lambda: r0.fr.resident_transfer_ctx(r1.fr, r0.handles[a], r1.handles[b], n, n_dst, runs, um))
            assert (e.unfit, e.unfit_reason) == (unfit, why), (runs, e.unfit, e.unfit_reason)
        # past the end of the map, for the run at position 2
        cand = sorted(narrow, key=slot)
        assert slot(cand[-1]) > slot(cand[1])
        e = r0.transfer_ctx(r1, a, b, n, n_dst, [cand[0], cand[1], cand[-1]], m[:slot(cand[-1])])
        assert e is None
        # every refusal of the call itself: duplicates, a run at src_n_runs, the destination's capacity, src_n_runs past the
        # capacity, and a null map with n_slot_map > 0
        for runs, sn, dn in (([narrow[0], narrow[0]], n, n_dst), ([n], n, n_dst), (narrow[:3], n, b.cap - 2), (narrow[:2], a.cap + 1, n_dst)):
            r0.transfer_ctx(r1, a, b, sn, dn, runs, m)
        rs = np.asarray(narrow[:2], np.uint32)
        t = A.CtxTransfer(struct_size=C.sizeof(A.CtxTransfer), src_n_runs=n, dst_n_runs=n_dst, runs=rs.ctypes.data, n=2, slot_map=None,
                          n_slot_map=3)
        assert r0.fr._lib.bf_resident_transfer_ctx(r0.fr._ctx, r0.handles[a], r1.fr._ctx, r1.handles[b], C.byref(t)) == A.BF_EINVAL
        r0.sync()
        r1.sync()
        # a longer map, with entries past the source's slot table that name nothing live anywhere: ignored
        long = np.concatenate([m, np.array([A.SLOT_NONE, 3, 0xFFFF, 1], np.uint32)])
        out = r0.transfer_ctx(r1, a, b, n, n_dst, [narrow[0]], long)
        assert out is not None
        n, n_dst = n - 1, n_dst + 1
        # an entry of a live source slot no moved run uses, naming a dead destination slot: the whole call is refused
        spare = next(s for s in r0.reg.live if s not in {slot(r) for r in range(n)})
        bad = m.copy()
        bad[spare] = 0xFFFF
        r0.transfer_ctx(r1, a, b, n, n_dst, [narrow[1]], bad)
        e = _refused(lambda: r0.fr.resident_transfer_ctx(r1.fr, r0.handles[a], r1.handles[b], n, n_dst, [narrow[1]], bad))
        assert e.unfit == A.EXTENT_NO_RUN and e.unfit_reason == A.UNFIT_NONE
        # ... and one naming a live destination slot of another Story
        other = m.copy()
        other[spare] = P.slot_of(1, (r0.reg.live[spare] + 1) % 6)
        assert r1.reg.live[int(other[spare])] != r0.reg.live[spare]
        r0.transfer_ctx(r1, a, b, n, n_dst, [narrow[1]], other)
        # once that source slot is dead, its entry is ignored
        r0.drop(spare)
        assert r0.transfer_ctx(r1, a, b, n, n_dst, [narrow[1]], bad) is not None
        n, n_dst = n - 1, n_dst + 1
        # a source slot dropped and put again for another Story: the old map names the old Story's slot and is refused; the
        # map of the registries as they stand moves the run with its new Story's slot
        s_re = slot(narrow[2] if narrow[2] < n else 0)
        k_old = r0.reg.live[s_re]
        r0.drop(s_re)
        k_new = next(k for k in range(6) if k != k_old and P.pool[k].S <= P.pool[k_old].S)
        assert r0.put(k_new) == s_re
        stale = m.copy()
        run_re = next(r for r in range(n) if slot(r) == s_re)
        r0.transfer_ctx(r1, a, b, n, n_dst, [run_re], stale)
        assert r0.transfer_ctx(r1, a, b, n, n_dst, [run_re], P.slot_map()) is not None
        n, n_dst = n - 1, n_dst + 1
        got = r1.fr.resident_download(r1.handles[b], n_dst - 1, 1, P.Ld.state_stride)
        assert int(got[0, :4].view(np.uint32)[0]) == P.slot_of(1, k_new)
        # an arena compaction in each ctx: many wide topologies put and dropped, then one more put re-packs the live records
        for c, r in enumerate((r0, r1)):
            fill = randgen.random_topologies(np.random.default_rng(900 + c), 1500, 200, 256, parallel=False)
            while r.reg.free:
                r.put(0)
            got_slots = [int(s) for s in r.fr.put_topologies(fill)]
            assert got_slots == list(range(r.reg.n_index, r.reg.n_index + len(got_slots)))
            for s in got_slots:
                r.fr.drop_topology(s)
            # the registry follows: the slots were new (or reused from the free list in its order), then dropped in order
            r.reg.n_index += len(got_slots)
            for s in got_slots:
                r.reg.free.append(s)
                r.reg.changes += 1
            before = r.fr.stats()["arena_compactions"]
            r.put(7 + c)
            assert r.fr.stats()["arena_compactions"] == before + 1
        runs = [r for r in range(n) if r0.reg.live.get(slot(r)) is not None and r0.reg.stories[r0.reg.live[slot(r)]].S <= P.Ld.steps_max][:4]
        assert r0.transfer_ctx(r1, a, b, n, n_dst, runs, P.slot_map()) is not None
        r0.tick(a, "touched", n - len(runs))
        r1.tick(b, "touched", n_dst + len(runs))
    finally:
        P.close()


# ================================================================================== 4. the gather at every launch shape, at scale
class GatherTwins:
    """deployment A (source and destination batch in one ctx) and B (the same two batches in two ctxs, the Stories put in other
    orders), with every side area; the same calls to both, compared with slots read as the Story they hold"""

    def __init__(self, pair, seed, S, fields, K, n_src, n_dst, s_lo, s_hi):
        d0, d1 = _devices(pair)
        self.rng = rng = np.random.default_rng(seed)
        self.pool = story_pool(rng, s_lo, s_hi, 2 if fields & CHILD else 0, 3, n_spare=0)
        self.K = K
        self.cap = [n_src + 8, n_dst + n_src]
        self.n_timers = 0
        self.deps = ()
        try:
            self.A = Deployment([d0], [0, 0], self.pool, rng)
            self.deps = (self.A,)
            self.B = Deployment([d0, d1], [0, 1], self.pool, rng)
            self.deps = (self.A, self.B)
            self._fill(S, fields, n_src, n_dst)
        except BaseException:
            self.close()
            raise

    def _fill(self, S, fields, n_src, n_dst):
        rng, K = self.rng, self.K
        child = max(p.child_nibbles() for p in self.pool) if fields & CHILD else 0
        self.L = L = make_layout(S, child, fields)
        Lg = make_layout(S, child, fields & (COND | CHILD))
        for b, n in ((0, n_src), (1, n_dst)):
            story = rng.integers(0, len(self.pool), n)
            recs = relay_state(Lg, L, random_records(rng, Lg, [self.pool[k] for k in story], story))
            timers = self._timers(story) if n else np.zeros(0, Frontier.TIMER_DTYPE)
            self.n_timers = max(self.n_timers, len(timers))
            sched = SRM.defaults(n)
            sched["run"], sched["story_key"], sched["queue_key"] = np.arange(n), story, rng.integers(0, 3, n)
            sched["priority"], sched["run_phase"] = rng.integers(-2, 4, n), 2
            ctl = np.zeros(n // 4, Frontier.RUNCTL_PUT_DTYPE)
            ctl["run"] = rng.choice(n, size=n // 4, replace=False) if n else []
            ctl["story_deadline"], ctl["drain_deadline"] = rng.integers(500, 900, n // 4), A.TIMER_NONE
            for d in self.deps:
                d.create(L, self.cap[b])
                fr, h = d.fr(b), d.h[b]
                if n:
                    fr.resident_upload(h, 0, d.records(b, recs))
                fr.resident_timers(h, K)
                if len(timers):
                    fr.resident_timers_arm(h, timers)
                fr.resident_sched(h)
                if n:
                    fr.resident_sched_put(h, sched)
                fr.resident_runctl(h)
                if len(ctl):
                    fr.resident_runctl_put(h, ctl)
                fr.resident_commit_marks(h)
                d.n[b] = n

    def _timers(self, story):
        """up to K armed slots on a third of the runs: as many steps as the Story has, from step 0"""
        out = []
        for r in range(0, len(story), 3):
            for s in range(min(self.K, self.pool[int(story[r])].S)):
                out.append((r, s, A.DEC_PENDING, 0, 1000 + s, 0))
        return np.array(out, Frontier.TIMER_DTYPE)

    def snapshot(self, d, b):
        fr, h, cap = d.fr(b), d.h[b], self.cap[b]
        st = fr.resident_download(h, 0, cap, self.L.state_stride).copy()
        w = st[:, :4].view(np.uint32)
        w[:d.n[b], 0] = [d.story[d.home[b]].get(int(s), 0xFFFF) for s in w[:d.n[b], 0]]
        return {"state": st, "timers": fr.resident_timers_download(h, 0, cap, self.K), "sched": fr.resident_sched_download(h, 0, cap),
                "runctl": fr.resident_runctl_download(h, 0, cap)}

    def compare(self, what):
        for b in (0, 1):
            assert self.A.n[b] == self.B.n[b]
            _eq(self.snapshot(self.A, b), self.snapshot(self.B, b), "%s: batch %d" % (what, b))

    def tick(self, what):
        outs = []
        for d in self.deps:
            o = [d.fr(b).resident_tick_touched(d.h[b], d.n[b], NONE_D, d.n[b], d.n[b] * 1024 + 1) for b in (0, 1)]
            for x in o:
                for k in ("runs", "head", "events"):
                    x[k] = x[k].copy()
            outs.append(o)
        _eq(outs[0], outs[1], "touched tick " + what)
        return outs[0]

    def transfer(self, s, t, runs):
        A_, B = self.A, self.B
        a = A_.fr(s).resident_transfer(A_.h[s], A_.h[t], A_.n[s], A_.n[t], runs)
        b = B.fr(s).resident_transfer_ctx(B.fr(t), B.h[s], B.h[t], B.n[s], B.n[t], runs, B.slot_map(B.home[s], B.home[t]))
        _eq(a, b, "transfer %d -> %d" % (s, t))
        for d in self.deps:
            d.n[s] -= len(runs)
            d.n[t] += len(runs)

    def close(self):
        for d in self.deps:
            d.close()


def _gather_case(pair, seed, S, fields, K, n_move, n_src, n_dst, s_lo, s_hi, outgrow=False):
    """outgrow: the staging of the move is asserted larger than every earlier call of the case could have left in either
    ctx's scratch (which grows to the largest call's inputs and outputs, and is not reported): the bytes of every record and
    request sent, every list a tick returned, and 1 MiB for the rest"""
    g = GatherTwins(pair, seed, S, fields, K, n_src, n_dst, s_lo, s_hi)
    try:
        g.compare("set-up")
        ticked = g.tick("set-up")
        if outgrow:
            L = g.L
            staging = n_move * (L.state_stride + L.result_stride + 8 * K)
            earlier = (n_src * (L.state_stride + 2 * 32) + 16 * g.n_timers + sum(8 * x["n_listed"] + 2 * x["n_events"] for x in ticked) +
                       (1 << 20))
            assert staging > earlier, (staging, earlier)
        # runs uploaded since the tick (mark 3) and above the ticked runs, mixed with baseline runs
        Lg = make_layout(S, g.L.child_nibbles, fields & (COND | CHILD))
        fresh = relay_state(Lg, g.L, random_records(g.rng, Lg, [g.pool[0]] * 2, [0] * 2))
        for d in g.deps:
            d.fr(0).resident_upload(d.h[0], 1, d.records(0, fresh))
        runs = g.rng.choice(n_src, size=n_move, replace=False).astype(np.uint32)
        g.transfer(0, 1, runs)
        g.compare("after %d runs moved" % n_move)
        g.tick("after the move")
        back = np.arange(n_dst, n_dst + n_move, dtype=np.uint32)   # the same runs, back
        g.transfer(1, 0, back)
        g.compare("after %d runs moved back" % len(back))
        g.tick("after the move back")
    finally:
        g.close()


FULL = COND | DEC | CHILD | OUT
SHAPES = [(n, 33, 1024, FULL) for n in (1, 7, 8, 9, 255, 256, 257)] + [(40, k, 1024, FULL) for k in (1, 32, 64)] + \
         [(257, 32, 32, 0), (9, 1, 32, 0)]


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=["n%d-K%d-S%d%s" % (n, k, s, "-planes" if f else "") for n, k, s, f in SHAPES])
def test_gather_launch_shapes(pair, shape):
    """n moved runs around the gather's 8-run CTAs; K timer slots (33 and 64 take a second lane sweep, armed from step 0 on
    Stories of 70-110 steps); 32-step records without planes (fewer than 32 vectors per run) and 1024-step records with cond,
    decision, child and output fields (several vectors per lane).  Both ways, against the same calls within one ctx"""
    n, K, S, fields = shape
    lo, hi = (70, 110) if S == 1024 else (8, 30)
    _gather_case(pair, 40 + n + K + S, S, fields, K, n, n + 30, 20, lo, hi)


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
def test_gather_at_scale(pair):
    """20 480 runs of a 1024-step batch with every area move in one call, a staging larger than any earlier call left in either
    ctx's scratch, and the same runs back again"""
    _gather_case(pair, 9, 1024, FULL, 8, 20480, 20600, 50, 1000, 1024, outgrow=True)


# ================================================================================== 6. the span schedule against the model
class Span:
    """resident batches with limiter inputs on several ctxs; parts are (ctx, handle, L, n, model, topo)"""

    def __init__(self, pair, n_ctx, seed):
        devs = _devices(pair)
        self.rng = rng = np.random.default_rng(seed)
        self.ts = [randgen.random_topologies(rng, 8, 4, 60, parallel=True), randgen.random_topologies(rng, 6, 100, 300, parallel=True)]
        spare = randgen.random_topologies(rng, 1, 3, 5, parallel=False)
        self.frs = []
        try:
            for c in range(n_ctx):
                self.frs.append(Frontier(devs[c % 2]))
        except BaseException:
            self.close()
            raise
        self.slots, self.descs = [], []
        for c, fr in enumerate(self.frs):
            if c % 2:
                fr.put_topologies(spare)
            sl = [fr.put_topologies(t) for t in self.ts]
            self.slots.append(sl)
            d = {}
            for t, s in zip(self.ts, sl):
                d.update(SR.from_topology_set(t, s))
            self.descs.append(d)
        self.parts = []

    def add(self, c, n, width, inputs):
        """a batch of n runs on ctx c over the topologies of width class `width`, its inputs from inputs(n, rng)"""
        fr = self.frs[c]
        L, state, topo = randgen.random_state(self.rng, self.ts[width], self.slots[c][width], max(n, 1), COND | DEC, phase_mix="progress")
        h = fr.resident_create(L, max(n, 1) + 4)
        m = SRM.Batch(L, max(n, 1) + 4)
        fr.resident_upload(h, 0, state[:max(n, 1)])   # a part without runs still holds one, ticked, past its n_runs
        fr.resident_sched(h)
        if n:
            p = inputs(n, self.rng)
            fr.resident_sched_put(h, p)
            m.put(p)
        self.parts.append({"c": c, "h": h, "L": L, "n": n, "m": m, "topo": topo[:n], "w": width})
        return len(self.parts) - 1

    def tick(self, i, deltas=NONE_D):
        p = self.parts[i]
        fr = self.frs[p["c"]]
        p["res"], _ = fr.resident_tick(p["h"], p["L"], max(p["n"], 1), deltas)
        p["res"] = p["res"][:p["n"]]
        p["state"] = fr.resident_download(p["h"], 0, p["n"], p["L"].state_stride) if p["n"] else np.zeros((0, p["L"].state_stride), np.uint8)

    def model(self, order, tables, now, models=None):
        ps = [self.parts[i] for i in order]
        ms = models or [p["m"] for p in ps]
        return SRM.schedule([(m, p["n"], p["state"], p["res"], self.descs[p["c"]]) for m, p in zip(ms, ps)], tables, now)

    def schedule(self, order, tables, now, what=""):
        got = resident_schedule_ctxs([(self.frs[self.parts[i]["c"]], dict(handle=self.parts[i]["h"], n_runs=self.parts[i]["n"]))
                                      for i in order], tables, now)
        want = self.model(order, tables, now)
        _compare_schedule(got, want, what)
        return got, want

    def per_ctx_launches(self, order, tables, now):
        """the steps that schedules of each ctx alone would launch (model copies; the batches keep their baselines)"""
        total = 0
        for c in range(len(self.frs)):
            mine = [i for i in order if self.parts[i]["c"] == c]
            if mine:
                ms = [copy.deepcopy(self.parts[i]["m"]) for i in mine]
                w = self.model(mine, tables, now, ms)
                total += sum(int(np.ascontiguousarray(x["records"][:, 0:4]).view("<u4").sum()) for x in w["parts"])
        return total

    def close(self):
        for fr in self.frs:
            fr.close()


def _launched(want):
    return sum(int(np.ascontiguousarray(x["records"][:, 0:4]).view("<u4").sum()) for x in want["parts"])


def _inputs(ns, nq, prio, since=None, queue=None, story=None, oor=0.05):
    """limiter puts: keys in range (a fraction oor past the tables), priorities from prio(n, rng), origins from since(n, rng)"""
    def make(n, rng):
        p = SRM.defaults(n)
        p["run"] = np.arange(n)
        p["story_key"] = story(n, rng) if story else rng.integers(0, ns, n)
        p["queue_key"] = queue(n, rng) if queue else rng.integers(0, nq, n)
        out = rng.random(n) < oor
        p["story_key"][out] = rng.choice([ns, ns + 1, 0xFFFFFFFF], size=int(out.sum()))
        out = rng.random(n) < oor
        p["queue_key"][out] = rng.choice([nq, nq + 7, 0xFFFFFFFE], size=int(out.sum()))
        p["priority"] = prio(n, rng)
        p["queued_since"] = since(n, rng) if since else np.where(rng.random(n) < 0.3, SRM.NONE, rng.integers(0, 1000, n))
        p["run_phase"] = rng.choice([1, 2, 2, 2, 14], size=n)
        return p
    return make


NOW_S = 1000
NS, NQ = 12, 4


def _tables(**kw):
    t = dict(story_limit=np.zeros(NS, np.int32), queue_limit=np.zeros(NQ, np.int32), queue_aging_s=np.array([0, 30, 7, 0], np.int32),
             global_limit=0)
    t.update(kw)
    return t


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
@pytest.mark.parametrize("given", ["null", "story", "queue", "global", "maxprio", "all"])
def test_span_schedule_bases(pair, given):
    """table bases given or NULL, near 2^32 on keys without a limit so that the sums over the ctxs wrap as the device's atomics
    do; small bases on limited keys; queue 3's priorities all negative and its demand on ctx 0 only, so that the maxima of
    the ctxs without it must start from INT32_MIN"""
    sp = Span(pair, 3, 500 + ["null", "story", "queue", "global", "maxprio", "all"].index(given))
    try:
        def queue(n, rng):
            return rng.integers(0, 3, n)
        for c in range(3):
            for w in (0, 1):
                sp.add(c, int(sp.rng.integers(150, 400)), w, _inputs(NS, NQ, lambda n, rng: rng.integers(-3, 6, n), queue=queue))
        sp.add(0, 200, 0, _inputs(NS, NQ, lambda n, rng: rng.integers(-9, -1, n), queue=lambda n, rng: np.full(n, 3)))
        kw = {}
        if given in ("story", "all"):
            sb = np.arange(NS, dtype=np.uint32) % 3
            sb[:4] = np.uint32(0xFFFFFFFF) - np.arange(4, dtype=np.uint32)   # stories 0-3: no limit
            kw["story_running_base"] = sb
        if given in ("queue", "all"):
            kw["queue_running_base"] = np.array([0xFFFFFFFE, 1, 2, 0xFFFFFFFF], np.uint32)
        if given in ("global", "all"):
            kw["global_running_base"] = 0xFFFFFFF0
        if given in ("maxprio", "all"):
            kw["queue_max_priority_base"] = np.array([INT32_MIN, 2, -50, INT32_MIN + 1], np.int32)
        sl = np.zeros(NS, np.int32)
        sl[4:] = [3, 1, 9, 20, 2, 5, 40, 1]
        ql = np.array([0, 0, 60, 0], np.int32) if given not in ("queue", "all") else np.array([0, 0, 0, 0], np.int32)
        tables = _tables(story_limit=sl, queue_limit=ql, **kw)
        for i in range(len(sp.parts)):
            sp.tick(i)
        order = list(range(len(sp.parts)))
        got, want = sp.schedule(order, tables, NOW_S, given)
        if given in ("null", "story", "queue", "global"):
            assert want["queue_max_priority"][3] < 0, "queue 3 has no negative maximum: INT32_MIN would not be seen"
            assert any(int(x["heads"][:, 0].sum()) for x in want["parts"][-1:]), "queue 3 launches nothing: its maximum is not seen"
        if "story_running_base" in kw:
            assert (want["story_running"][:4] < kw["story_running_base"][:4]).any(), "no story total wraps past 2^32"
        if "queue_running_base" in kw:
            assert want["queue_running"][0] < 0xFFFFFFFE and want["queue_running"][3] < 0xFFFFFFFF
        if "global_running_base" in kw:
            assert want["global_running"] < 0xFFFFFFF0
        # a second schedule after a tick that changed runs on one ctx only lists only those runs
        p = sp.parts[2]
        runs = sp.rng.choice(p["n"], size=9, replace=False)
        d = np.zeros(9, Frontier.DELTA_DTYPE)
        d["run"], d["field"], d["code"] = runs, A.DELTA_PHASE, 2
        d["index"] = [int(sp.ts[p["w"]].S[int(p["topo"][r])]) - 1 for r in runs]
        sp.tick(2, d)
        for i in order:
            if i != 2:
                sp.tick(i)
        got, want = sp.schedule(order, tables, NOW_S, given + " second")
        for i, x in enumerate(got["parts"]):
            assert set(x["runs"].tolist()) <= (set(runs.tolist()) if i == 2 else set()), i
    finally:
        sp.close()


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
def test_span_schedule_priorities_and_keys(pair):
    """priorities near INT32_MAX that wrap with aging, INT32_MIN, origins at and after now, keys past both tables"""
    sp = Span(pair, 2, 611)

    def prio(n, rng):
        return rng.choice(np.array([INT32_MAX, INT32_MAX - 1, INT32_MAX - 40, INT32_MIN, INT32_MIN + 1, -1, 0, 5], np.int64), size=n)

    def since(n, rng):
        return rng.choice(np.array([SRM.NONE, NOW_S, NOW_S + 1, NOW_S + 900, 0, NOW_S - 1, NOW_S - 300], np.int64), size=n).astype(np.uint32)
    try:
        for c in range(2):
            for w in (0, 1):
                sp.add(c, int(sp.rng.integers(200, 500)), w, _inputs(NS, NQ, prio, since, oor=0.15))
        for i in range(len(sp.parts)):
            sp.tick(i)
        tables = _tables(queue_aging_s=np.array([1, 30, 0, 7], np.int32))
        got, want = sp.schedule(list(range(4)), tables, NOW_S)
        # not vacuous: some run of a queue with aging has a positive priority whose effective priority wraps negative
        wrapped = 0
        for p in sp.parts:
            inp = p["m"].inputs[:p["n"]]
            qk = inp["queue_key"].astype(np.int64)
            aging = np.where(qk < NQ, tables["queue_aging_s"][np.minimum(qk, NQ - 1)], 0)
            eff = SR.effective_priority_rows(inp["priority"], SRM.elapsed(inp["queued_since"], NOW_S), aging)
            wrapped += int(((inp["priority"] > 0) & (eff < 0)).sum())
        assert wrapped, "no priority wraps with aging"
    finally:
        sp.close()


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
@pytest.mark.parametrize("limit", ["queue", "global", "priority"])
def test_span_schedule_limits_bind_across_ctxs(pair, limit):
    """a queue limit, a global limit or a higher priority whose blocking runs live on the other ctx: the span schedule launches
    what the model's one schedule launches, where schedules of each ctx alone would launch more"""
    sp = Span(pair, 2, 700 + len(limit))
    try:
        if limit == "priority":   # queue 1: ctx 0's runs outrank ctx 1's
            sp.add(0, 300, 0, _inputs(NS, NQ, lambda n, rng: np.full(n, 9), queue=lambda n, rng: np.full(n, 1), oor=0))
            sp.add(1, 300, 0, _inputs(NS, NQ, lambda n, rng: np.full(n, 2), queue=lambda n, rng: np.full(n, 1), oor=0))
        else:
            for c in range(2):
                sp.add(c, 300, c, _inputs(NS, NQ, lambda n, rng: np.zeros(n, np.int64), queue=lambda n, rng: np.full(n, 2), oor=0))
        for i in range(len(sp.parts)):
            sp.tick(i)
        order = [0, 1]
        free = sp.model(order, _tables(), NOW_S, [copy.deepcopy(p["m"]) for p in sp.parts])
        tables = _tables(queue_aging_s=np.zeros(NQ, np.int32))
        if limit == "queue":
            ql = np.zeros(NQ, np.int32)
            ql[2] = int(free["queue_running"][2]) + 1
            tables["queue_limit"] = ql
        elif limit == "global":
            tables["global_limit"] = int(free["global_running"]) + 1
        per_ctx = sp.per_ctx_launches(order, tables, NOW_S)
        got, want = sp.schedule(order, tables, NOW_S, limit)
        assert per_ctx > _launched(want), "the %s does not bind across ctxs: the case would pass vacuously" % limit
        if limit == "priority":
            assert want["parts"][1]["heads"][:, 0].sum() == 0 and want["parts"][1]["heads"][:, 2].sum() > 0
    finally:
        sp.close()


@pytest.mark.parametrize("pair", DEVS, ids=DEV_IDS)
@pytest.mark.parametrize("n_ctx", [1, 2, 3, 4])
def test_span_schedule_part_layouts(pair, n_ctx):
    """one to four ctxs, parts of one ctx interleaved in call order with another's, a ctx whose parts all have no runs, and a
    second schedule after a tick that changed runs on one ctx only"""
    sp = Span(pair, n_ctx, 800 + n_ctx)
    try:
        inp = _inputs(NS, NQ, lambda n, rng: rng.integers(-2, 5, n))
        for c in range(n_ctx):
            empty = n_ctx >= 3 and c == n_ctx - 1
            for w in (0, 1):
                sp.add(c, 0 if empty else int(sp.rng.integers(50, 300)), w, inp)
        # interleaved: ctx 0's first part, ctx 1's first, ctx 0's second, ...
        order = [i for w in (0, 1) for i in range(len(sp.parts)) if sp.parts[i]["w"] == w]
        for i in order:
            sp.tick(i)
        sl = np.zeros(NS, np.int32)
        sl[::2] = 4
        tables = _tables(story_limit=sl, queue_limit=np.array([0, 30, 0, 5], np.int32), global_limit=5000,
                         story_running_base=np.arange(NS, dtype=np.uint32) % 2, queue_running_base=np.array([0, 3, 0, 1], np.uint32),
                         queue_max_priority_base=np.array([INT32_MIN, 1, -4, INT32_MIN], np.int32), global_running_base=7)
        got, want = sp.schedule(order, tables, NOW_S, "first")
        assert all(x["full"] for x in got["parts"])
        changed = sp.parts.index(next(p for p in sp.parts if p["c"] == 0 and p["n"]))
        p = sp.parts[changed]
        runs = sp.rng.choice(p["n"], size=min(6, p["n"]), replace=False)
        d = np.zeros(len(runs), Frontier.DELTA_DTYPE)
        d["run"], d["field"], d["code"] = runs, A.DELTA_PHASE, 2
        d["index"] = [int(sp.ts[p["w"]].S[int(p["topo"][r])]) - 1 for r in runs]
        sp.tick(changed, d)
        for i in order:
            if i != changed and sp.parts[i]["c"] != 0:
                sp.tick(i)
        got, want = sp.schedule(order, tables, NOW_S, "second")
        pos = order.index(changed)
        for k, x in enumerate(got["parts"]):
            assert set(x["runs"].tolist()) <= (set(runs.tolist()) if k == pos else set()), k
    finally:
        sp.close()
