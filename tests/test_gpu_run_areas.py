"""Every per-run side area of a resident batch through every call that moves, resets or re-lays runs, for each of the 8 area
sets (step timers with K = 2 or 5, limiter inputs, run control, any mix) and, for bf_resident_transfer, every (source set,
destination set) pair.  Each batch starts with non-default entries in every area it has: armed timer slots, stopped runs with
their saved flags byte, story and drain deadlines, limiter inputs, and schedule baselines.  After each call the state records,
the timer slots, the run-control records and the limiter inputs of every batch are compared over the whole capacity with the
composed host model of tests/lifecycle.py, and a tick and a bf_resident_schedule then check which runs kept their schedule
baseline.  A refused call must change nothing."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import randgen
from tests import sched_resident as SRM
from tests import schedref as SR
from tests import timers as T
from tests.lifecycle import (MOVED, RUNCTL, SCHED, TIMERS, Refused, area_sets, beyond_requests, records_of, seeded,
                             subset_name, template_records)

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
N, CAP, NOW = 16, 24, 5000
FIELDS = A.F_COND | A.F_DECISION | A.F_OUT_FAIL | A.F_OUT_SKIP_DEP
# no limit anywhere: runs of one template that are not stopped get equal schedule records, so a baseline kept where it should
# have been dropped shows as a run not listed
TABLES = dict(story_limit=np.zeros(4, np.int32), queue_limit=np.zeros(2, np.int32), queue_aging_s=np.zeros(2, np.int32),
              global_limit=0)
SETS = area_sets()
SET_IDS = [subset_name(s, k) for s, k in SETS]


class Env:
    def __init__(self, fr):
        self.fr = fr
        rng = np.random.default_rng(4242)
        self.ts = randgen.random_topologies(rng, 2, 20, 24, parallel=False)
        self.slots = [int(s) for s in fr.put_topologies(self.ts)]
        self.descs = SR.from_topology_set(self.ts, self.slots)
        self.L = make_layout(64, 0, FIELDS)
        self.S = [int(x) for x in self.ts.S]
        self.templates = template_records(self.L, self.slots, self.S)
        self.S_of, self.has_if = {}, {}
        self.add(self.ts, self.slots)

    def add(self, ts, slots):
        """the S and the HAS_IF step mask of each slot, for the redrive's reset"""
        at = 0
        for i, slot in enumerate(slots):
            S = int(ts.S[i])
            fl = ts.step_flags[at:at + S]
            self.S_of[int(slot)] = S
            self.has_if[int(slot)] = sum(1 << j for j in range(S) if fl[j] & A.SF_HAS_IF)
            at += S

    def resets(self, rq, words):
        """the reset set R of each redrive request, as an int step mask, and its slot's HAS_IF steps"""
        out = []
        for q in rq:
            slot, step = int(q["slot"]), int(q["step"])
            if step == A.REDRIVE_ALL:
                out.append((1 << self.S_of[slot]) - 1)
            else:
                w = self.fr.closure([slot], [step], words)[0]
                out.append(int.from_bytes(w.astype("<u4").tobytes(), "little"))
        return out, [self.has_if[int(q["slot"])] for q in rq]

    def records(self, n):
        return records_of(self.templates, n)


@pytest.fixture(scope="module")
def env():
    f = Frontier(0)
    yield Env(f)
    f.close()


def _rows(a):
    """a structured array as one row of bytes per record"""
    return np.ascontiguousarray(a).view(np.uint8).reshape(a.shape[0], -1)


class Twin:
    """a device batch and its model (tests/lifecycle.AreaBatch)"""

    def __init__(self, env, subset, K, n=N, cap=CAP, beyond=False):
        """beyond: also entries in every area at the indices past the runs, which arrivals must overwrite"""
        fr, L = env.fr, env.L
        self.env, self.fr = env, fr
        recs = env.records(n)
        m, (p, arms, q) = seeded(L, cap, subset, K, recs, env.S[0] - 1, NOW)
        self.m = m
        self.h = fr.resident_create(L, cap)
        fr.resident_upload(self.h, 0, recs)
        if m.sched is not None:
            fr.resident_sched(self.h)
            fr.resident_sched_put(self.h, p)
        if m.K:
            fr.resident_timers(self.h, m.K)
            fr.resident_timers_arm(self.h, arms)
        if m.runctl is not None:
            fr.resident_runctl(self.h)
            fr.resident_runctl_put(self.h, q)
        if beyond:
            p, arms, q = beyond_requests(m, NOW)
            if m.sched is not None:
                fr.resident_sched_put(self.h, p)
                m.put_sched(p)
            if m.K:
                fr.resident_timers_arm(self.h, arms)
                assert m.arm(arms) == 0
            if m.runctl is not None:
                fr.resident_runctl_put(self.h, q)
                assert m.put_runctl(q)[0] == 0
        self.check("set-up")
        if m.sched is not None:
            schedule([self])

    @property
    def n(self):
        return self.m.n

    def check(self, what):
        fr, h, m = self.fr, self.h, self.m
        cap = m.cap
        got = fr.resident_download(h, 0, cap, m.L.state_stride)
        bad = np.nonzero((got != m.state).any(axis=1))[0]
        assert bad.size == 0, "%s: state records differ at runs %s" % (what, bad[:8].tolist())
        if m.timers is not None:
            t = fr.resident_timers_download(h, 0, cap, m.K).view(np.uint64).reshape(cap, m.K)
            bad = np.nonzero((t != m.timers).any(axis=1))[0]
            assert bad.size == 0, "%s: timer slots differ at runs %s" % (what, bad[:8].tolist())
        if m.runctl is not None:
            c = fr.resident_runctl_download(h, 0, cap)
            bad = np.nonzero((_rows(c) != _rows(m.runctl)).any(axis=1))[0]
            assert bad.size == 0, "%s: run-control records differ at runs %s" % (what, bad[:8].tolist())
        if m.sched is not None:
            s = fr.resident_sched_download(h, 0, cap)
            bad = np.nonzero((_rows(s) != _rows(m.sched.download(0, cap))).any(axis=1))[0]
            assert bad.size == 0, "%s: limiter inputs differ at runs %s" % (what, bad[:8].tolist())

    def snapshot(self):
        fr, h, m = self.fr, self.h, self.m
        out = [fr.resident_download(h, 0, m.cap, m.L.state_stride)]
        if m.timers is not None:
            out.append(fr.resident_timers_download(h, 0, m.cap, m.K))
        if m.runctl is not None:
            out.append(fr.resident_runctl_download(h, 0, m.cap))
        if m.sched is not None:
            out.append(fr.resident_sched_download(h, 0, m.cap))
        return [x.tobytes() for x in out]


def schedule(twins):
    """a dense tick of each batch, then one bf_resident_schedule over those with limiter inputs, compared with the model:
    totals, listed runs, heads and events.  -> per part: the model's schedule records, its listed runs, the tick's result records"""
    twins = [t for t in twins if t.m.sched is not None]
    if not twins:
        return []
    cur = []
    for t in twins:
        st = np.ascontiguousarray(t.m.state[:t.n])
        res, _ = t.fr.resident_tick(t.h, t.m.L, t.n, NONE_D)
        cur.append((st, res))
    fr = twins[0].fr
    got = fr.resident_schedule([dict(handle=t.h, n_runs=t.n) for t in twins], TABLES, NOW)
    want = SRM.schedule([(t.m.sched, t.n, st, res, t.env.descs) for t, (st, res) in zip(twins, cur)], TABLES, NOW)
    for k in ("story_running", "queue_running", "queue_max_priority"):
        assert np.array_equal(got[k], want[k]), k
    assert got["global_running"] == want["global_running"]
    out = []
    for i, (g, w) in enumerate(zip(got["parts"], want["parts"])):
        assert np.array_equal(g["runs"], w["listed"]), "part %d lists %s, the model %s" % (i, g["runs"].tolist(), w["listed"].tolist())
        hv = np.stack([g["heads"][f] for f in g["heads"].dtype.names], axis=1) if g["runs"].size else np.zeros((0, 4), np.uint32)
        assert np.array_equal(hv, w["heads"]) and np.array_equal(g["events"], w["events"]), i
        assert g["full"] == w["full"]
        out.append((w["records"], set(w["listed"].tolist()), cur[i][1]))
    return out


def baselines(tw):
    """the model's schedule records of a batch as they stand (None: no baseline)"""
    return [None if r is None else r.copy() for r in tw.m.sched.rec] if tw.m.sched is not None else None


def assert_sees_kept_baseline(before, records, listed, moved_to):
    """at least one run that lost its baseline at index `to` has the record the index held: a baseline kept there by mistake
    would leave it unlisted"""
    assert any(before[t] is not None and np.array_equal(before[t], records[t]) and t in listed for t in moved_to), \
        "no moved run has the record its new index held: a kept baseline would go unseen"


# ---------------------------------------------------------------------------------------------------- transfer
@pytest.mark.parametrize("src_set", SETS, ids=SET_IDS)
def test_transfer_every_destination_set(env, src_set):
    """bf_resident_transfer from a batch of src_set into one of every set, K down and up included: the refusals of the fit
    (armed slots past the destination's K, a run-control record without an area to arrive in, limiter inputs without an area),
    each leaving both batches byte-identical, then the transfer of the runs that fit"""
    fr = env.fr
    refused = set()
    for dst_set in SETS:
        a, b = Twin(env, *src_set), Twin(env, *dst_set, n=4, beyond=True)
        try:
            what = "%s -> %s" % (subset_name(*src_set), subset_name(*dst_set))
            moved = MOVED
            try:
                a.m.transfer(b.m, b.n, moved)
                want = None
            except Refused as e:
                want = e
            if want is not None:
                before = a.snapshot(), b.snapshot()
                with pytest.raises(A.FrontierError) as got:
                    fr.resident_transfer(a.h, b.h, a.n, b.n, moved)
                got = got.value
                assert got.status == A.BF_EINVAL and got.unfit == want.unfit, (what, got.unfit, want.unfit)
                assert (a.snapshot(), b.snapshot()) == before, "%s: a refused transfer changed a batch" % what
                if want.unfit == A.EXTENT_NO_RUN:
                    refused.add("sched")
                    continue
                r = moved[want.unfit]
                armed = len(T.armed(a.m.timers[r])) if a.m.timers is not None else 0
                # the refused run's extent word (its armed slots, and bit 31 for a lost run-control record) leaves the call only
                # through bf_last_error: bf_transfer.why has no field for it
                msg = str(got)
                assert ("%d timer slot(s) of the destination's %d" % (armed, b.m.K)) in msg, (what, msg)
                assert ("run-control area" in msg) == ("runctl" in want.lost), (what, msg)
                refused |= want.lost
                moved = [r for r in MOVED if not a.m.lost_by(b.m, r)]
                a.m.transfer(b.m, b.n, moved)
            src_n, dst_n = a.n + len(moved), b.n - len(moved)
            out = fr.resident_transfer(a.h, b.h, src_n, dst_n, moved)
            assert (out["src_n_runs"], out["dst_n_runs"]) == (a.n, b.n), what
            a.check(what + " (source)")
            b.check(what + " (destination)")
            schedule([a, b])
        finally:
            fr.resident_destroy(a.h)
            fr.resident_destroy(b.h)
    src, k = src_set
    if src & TIMERS and k == 5:
        assert "timers" in refused
    if src & RUNCTL:
        assert "runctl" in refused
    if src & SCHED:
        assert "sched" in refused


# ---------------------------------------------------------------------------------------------------- retire
@pytest.mark.parametrize("capacity", [0, CAP, 14], ids=["keep", "same", "smaller"])
@pytest.mark.parametrize("area_set", SETS, ids=SET_IDS)
def test_retire(env, area_set, capacity):
    """retire runs 1, 12 and 14 of 16: run 13 moves to 1 and run 15 to 12, indices 13-15 are vacated; a new capacity keeps the
    first `capacity` entries of every area"""
    tw = Twin(env, *area_set)
    try:
        before = baselines(tw)
        gone = [1, 12, 14]
        m, mv = tw.m.retire(N, gone, capacity)
        got = env.fr.resident_retire(tw.h, N, gone, capacity)
        assert got[0] == m and dict(zip(got[1].tolist(), got[2].tolist())) == mv
        tw.check("retire capacity %d" % capacity)
        for records, listed, _ in schedule([tw]):
            assert_sees_kept_baseline(before, records, listed, mv.values())
    finally:
        env.fr.resident_destroy(tw.h)


# ---------------------------------------------------------------------------------------------------- reshape and narrow
@pytest.mark.parametrize("kind", ["capacity", "words", "both"])
@pytest.mark.parametrize("area_set", SETS, ids=SET_IDS)
def test_reshape(env, area_set, kind):
    tw = Twin(env, *area_set)
    try:
        L = make_layout(96, 0, FIELDS) if kind != "capacity" else env.L
        cap = CAP + 8 if kind != "words" else CAP
        tw.m.reshape(L, cap)
        env.fr.resident_reshape(tw.h, L, cap)
        tw.check("reshape " + kind)
        for records, listed, _ in schedule([tw]):
            assert listed == (set(range(N)) if kind != "capacity" else set()), sorted(listed)
    finally:
        env.fr.resident_destroy(tw.h)


@pytest.mark.parametrize("kind", ["words", "same_words"])
@pytest.mark.parametrize("area_set", SETS, ids=SET_IDS)
def test_narrow(env, area_set, kind):
    tw = Twin(env, *area_set)
    try:
        L = make_layout(32, 0, FIELDS) if kind == "words" else make_layout(40, 0, FIELDS & ~A.F_OUT_SKIP_DEP)
        tw.m.narrow(L)
        env.fr.resident_narrow(tw.h, L, tw.n)
        tw.check("narrow " + kind)
        for records, listed, _ in schedule([tw]):
            assert listed == (set(range(N)) if kind == "words" else set()), sorted(listed)
    finally:
        env.fr.resident_destroy(tw.h)


# ---------------------------------------------------------------------------------------------------- migrate and redrive
@pytest.mark.parametrize("area_set", SETS, ids=SET_IDS)
def test_migrate(env, area_set):
    """the runs of template A move to a new topology of the same size that drops the last step: run 1's slot of that step is
    cancelled, and the migrated runs lose their schedule baseline"""
    fr = env.fr
    tw = Twin(env, *area_set)
    try:
        S = env.S[0]
        nt = randgen.random_topologies(np.random.default_rng(S), 1, S, S, parallel=False)
        new = int(fr.put_topologies(nt)[0])
        env.descs.update(SR.from_topology_set(nt, [new]))
        env.add(nt, [new])
        step_map = np.arange(S, dtype=np.uint16)
        step_map[S - 1] = T.MIGRATE_GONE
        runs = tw.m.migrate(env.slots[0], new, step_map)
        assert fr.resident_migrate(tw.h, env.slots[0], new, step_map, tw.n) == len(runs) > 0
        tw.check("migrate")
        for records, listed, _ in schedule([tw]):
            assert set(runs) <= listed
    finally:
        fr.resident_destroy(tw.h)


@pytest.mark.parametrize("step", [0, A.REDRIVE_ALL], ids=["step", "all"])
@pytest.mark.parametrize("area_set", SETS, ids=SET_IDS)
def test_redrive(env, area_set, step):
    """redrives of stopped runs (3: a timeout, 7: a cancel), of a run with armed slots and both deadlines kinds, and one
    request on the wrong slot, which changes nothing"""
    fr = env.fr
    tw = Twin(env, *area_set)
    try:
        rq = np.zeros(5, Frontier.REDRIVE_DTYPE)
        for i, r in enumerate([3, 7, 5, 13]):
            rq[i] = (r, env.slots[0], step, 0)
        rq[4] = (6, env.slots[0], step if step == A.REDRIVE_ALL else 0, 0)   # run 6 holds template B
        status, applied = fr.resident_redrive(tw.h, rq)
        assert status.tolist() == [1, 1, 1, 1, 0] and applied == 4
        tw.m.redrive(rq, status, *env.resets(rq, tw.m.L.words))
        tw.check("redrive")
        schedule([tw])
    finally:
        fr.resident_destroy(tw.h)
