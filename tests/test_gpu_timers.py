"""Step timers of a resident batch on the device (bf_resident_timers, _timers_arm, _fire, _timers_download) against the host model
tests/timers.py, byte for byte: the state records, the slots, the fired list, the counts and next_deadline.  Also: a fire followed
by a tick equals the written codes sent as BF_DELTA_DECISION deltas followed by the same tick; the edges of the slot area and of
the layout; refusals change nothing; every resident call that moves, re-indexes or resets runs re-keys the slots as the model
does; and a batch that never enables timers launches what it launched before."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import randgen
from tests import timers as T
from tests.test_gpu_reshape import _batch

pytestmark = pytest.mark.gpu

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def requests(rng, L, n_runs, k, cap=None, cancel=0.15, step_hi=None):
    """k random requests on distinct (run, step) pairs of runs [0, n_runs): codes that write only with decision planes"""
    step_hi = step_hi or L.steps_max
    pairs = set()
    while len(pairs) < k:
        pairs.add((int(rng.integers(0, n_runs)), int(rng.integers(0, step_hi))))
    rq = np.zeros(k, dtype=Frontier.TIMER_DTYPE)
    codes = [0, 1, 2, 3] if L.off_decision != A.OFF_NONE else [0]
    for i, (r, s) in enumerate(sorted(pairs, key=lambda _: rng.random())):
        dl = T.NONE if rng.random() < cancel else int(rng.integers(0, 1000))
        rq[i] = (r, s, int(rng.choice(codes)), 0, dl, 0)
    return rq


class Twin:
    """a device batch with a timer area and its model: the state records and the slots"""

    def __init__(self, fr, L, st, cap, K):
        self.fr, self.L, self.K = fr, L, K
        self.h = fr.resident_create(L, cap)
        fr.resident_upload(self.h, 0, st)
        fr.resident_timers(self.h, K)
        self.state = fr.resident_download(self.h, 0, cap, L.state_stride)
        self.area = T.empty_area(cap, K)

    @property
    def cap(self):
        return self.area.shape[0]

    def slots(self):
        return self.fr.resident_timers_download(self.h, 0, self.cap, self.K).view(np.uint64).reshape(self.cap, self.K)

    def check(self):
        assert np.array_equal(self.slots(), self.area), "timer slots differ from the model"
        assert np.array_equal(self.fr.resident_download(self.h, 0, self.cap, self.L.state_stride), self.state), "records differ"

    def arm(self, rq):
        rc, run = T.check_arm(self.area, self.L, rq)
        if rc:
            with pytest.raises(A.FrontierError) as e:
                self.fr.resident_timers_arm(self.h, rq)
            assert e.value.status == rc
            if rc == T.ENOMEM:
                assert ("run %d " % run) in str(e.value)
        else:
            self.fr.resident_timers_arm(self.h, rq)
            T.arm(self.area, self.L, rq)
        return rc

    def fire(self, n_runs, now, cap=None):
        got = self.fr.resident_fire(self.h, n_runs, now, fired_cap=cap)
        want = T.fire(self.area, self.L, self.state, n_runs, now)
        for k in ("n_fired", "n_written", "n_pruned", "next_deadline"):
            assert got[k] == want[k], (k, got[k], want[k])
        lst = [tuple(int(x) for x in e) for e in got["fired"]]
        assert lst == want["fired"][:len(lst)] and len(lst) == min(want["n_fired"], 4096 if cap is None else cap)
        return want


@pytest.mark.parametrize("S,fields,K", [(256, ALL, 4), (64, A.F_DECISION, 1), (1024, ALL, 8), (256, 0, 3)])
def test_random_arms_and_fires_match_the_model(fr, S, fields, K):
    rng = np.random.default_rng(S + K + fields)
    n = 700
    pt, L, st = _batch(fr, rng, S, fields, False, n)
    tw = Twin(fr, L, st, n + 9, K)
    now = 0
    for step in range(10):
        tw.arm(requests(rng, L, n + 9, int(rng.integers(1, 600)), step_hi=min(S, 40) if step % 2 else S))
        tw.check()
        now += int(rng.integers(0, 200))
        tw.fire(int(rng.integers(n // 2, n + 1)), now, cap=int(rng.choice([0, 7, 4096])))
        tw.check()


def _tick_pair(fr, L, st, n):
    hs = []
    for _ in range(2):
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, st)
        hs.append(h)
    return hs


@pytest.mark.parametrize("kind", ["touched", "changed_only"])
def test_a_fire_equals_its_codes_sent_as_deltas(fr, kind):
    rng = np.random.default_rng(7 if kind == "touched" else 8)
    n = 1500
    pt, L, st = _batch(fr, rng, 256, ALL, False, n)
    hA, hB = _tick_pair(fr, L, st, n)
    for h in (hA, hB):   # the first tick of each kind evaluates every run
        if kind == "touched":
            assert fr.resident_tick_touched(h, n, NONE, n, BIG)["full"] == 1
        else:
            fr.resident_tick_compact(h, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    fr.resident_timers(hA, 4)
    model = T.empty_area(n, 4)
    rq = requests(rng, L, n, 1200, cancel=0.0)
    rc, _ = T.check_arm(model, L, rq)
    while rc:   # keep within K per run
        rq = requests(rng, L, n, 1200, cancel=0.0)
        rc, _ = T.check_arm(model, L, rq)
    fr.resident_timers_arm(hA, rq)
    T.arm(model, L, rq)
    state = fr.resident_download(hA, 0, n, L.state_stride)
    out = T.fire(model, L, state, n, 500)
    assert out["n_written"] > 50
    got = fr.resident_fire(hA, n, 500)
    assert got["n_written"] == out["n_written"]
    d = T.as_deltas(out["fired"], Frontier.DELTA_DTYPE)
    if kind == "touched":
        a = fr.resident_tick_touched(hA, n, NONE, n, BIG)
        b = fr.resident_tick_touched(hB, n, d, n, BIG)
        for k in ("full", "n_evaluated", "n_listed", "n_events"):
            assert a[k] == b[k], k
        for k in ("runs", "head", "events"):
            assert np.array_equal(a[k], b[k]), k
        assert a["full"] == 0 and a["n_evaluated"] == len(out["touched"])
    else:
        a = fr.resident_tick_compact(hA, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        b = fr.resident_tick_compact(hB, n, d, BIG, flags=A.EVAL_CHANGED_ONLY)
        for x, y in zip(a, b):
            assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y)
    assert np.array_equal(fr.resident_download(hA, 0, n, L.state_stride), fr.resident_download(hB, 0, n, L.state_stride))


def test_edges(fr):
    rng = np.random.default_rng(11)
    n = 200
    pt, L, st = _batch(fr, rng, 1024, ALL, False, n)     # S = 1024: words = 32
    tw = Twin(fr, L, st, n, 1)
    last = n - 1
    for r in (0, last):   # make the steps the timers name non-terminal and pending
        T._set(tw.state[r], L.off_phase, L.words, 4, 1023, A.PHASE_RUNNING)
        T._set(tw.state[r], L.off_decision, L.words, 2, 1023, A.DEC_PENDING)
    fr.resident_upload(tw.h, 0, tw.state)
    rq = np.zeros(2, dtype=Frontier.TIMER_DTYPE)
    rq[0] = (last, 1023, A.DEC_TIMED_OUT, 0, T.NONE - 1, 0)
    rq[1] = (0, 1023, A.DEC_SUCCEED, 0, 0, 0)
    assert tw.arm(rq) == 0
    tw.check()
    full = np.zeros(1, dtype=Frontier.TIMER_DTYPE)
    full[0] = (last, 5, A.DEC_SUCCEED, 0, 3, 0)
    assert tw.arm(full) == T.ENOMEM   # K = 1 is full
    tw.check()
    out = tw.fire(n, 0)                # now = 0 fires deadline 0 only
    assert out["fired"] == [(0, 1023, A.DEC_SUCCEED, 1)] and out["next_deadline"] == T.NONE - 1
    tw.check()
    out = tw.fire(n, T.NONE - 1)
    assert out["fired"] == [(last, 1023, A.DEC_TIMED_OUT, 1)]
    tw.check()
    # no decision planes: wake-only timers only
    L0 = make_layout(64, 0, 0)
    st0 = np.zeros((8, L0.state_stride), np.uint8)
    tw0 = Twin(fr, L0, st0, 8, 2)
    bad = np.zeros(1, dtype=Frontier.TIMER_DTYPE)
    bad[0] = (1, 1, A.DEC_TIMED_OUT, 0, 5, 0)
    assert tw0.arm(bad) == T.EINVAL
    ok = np.zeros(2, dtype=Frontier.TIMER_DTYPE)
    ok[0], ok[1] = (1, 63, A.DEC_PENDING, 0, 5, 0), (7, 0, A.DEC_PENDING, 0, 6, 0)
    assert tw0.arm(ok) == 0
    out = tw0.fire(8, 5)
    assert out["fired"] == [(1, 63, 0, 0)] and out["next_deadline"] == 6
    tw0.check()


def test_refusals_change_nothing(fr):
    rng = np.random.default_rng(12)
    n = 64
    pt, L, st = _batch(fr, rng, 64, ALL, False, n)
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    one = np.zeros(1, dtype=Frontier.TIMER_DTYPE)
    one[0] = (0, 0, 1, 0, 5, 0)
    for call in (lambda: fr.resident_timers_arm(h, one), lambda: fr.resident_fire(h, n, 0),
                 lambda: fr.resident_timers_download(h, 0, 1, 1), lambda: fr.resident_timers(h, 0),
                 lambda: fr.resident_timers(h, 65)):
        with pytest.raises(A.FrontierError):
            call()
    tw = Twin(fr, L, st, n, 4)
    tw.arm(requests(rng, L, n, 120, cancel=0.0, step_hi=8))
    marks_probe = fr.resident_tick_touched(tw.h, n, NONE, n, BIG)
    assert marks_probe["full"] == 1
    for bad in ((n, 0, 1, 0, 5, 0), (0, L.steps_max, 1, 0, 5, 0), (0, 0, 4, 0, 5, 0), (0, 0, 1, 1, 5, 0), (0, 0, 1, 0, 5, 1)):
        rq = np.zeros(1, dtype=Frontier.TIMER_DTYPE)
        rq[0] = bad
        with pytest.raises(A.FrontierError) as e:
            fr.resident_timers_arm(tw.h, rq)
        assert e.value.status == A.BF_EINVAL
    dup = np.zeros(2, dtype=Frontier.TIMER_DTYPE)
    dup[0], dup[1] = (3, 2, 1, 0, 5, 0), (3, 2, 0, 0, T.NONE, 0)
    with pytest.raises(A.FrontierError):
        fr.resident_timers_arm(tw.h, dup)
    over = np.zeros(5, dtype=Frontier.TIMER_DTYPE)
    for i in range(5):
        over[i] = (9, 20 + i, 1, 0, 5, 0)
    tw.arm(over)   # 5 > K: ENOMEM naming run 9
    with pytest.raises(A.FrontierError):
        fr.resident_timers(tw.h, 3)   # K cannot shrink
    with pytest.raises(A.FrontierError):
        fr.resident_fire(tw.h, n + 1, 0)
    tw.check()
    t = fr.resident_tick_touched(tw.h, n, NONE, n, BIG)   # nothing was touched by the refusals or by arming
    assert t["full"] == 0 and t["n_evaluated"] == 0
    fr.resident_timers(tw.h, 6)   # grows K keeping the slots
    tw.area = T.grow(tw.area, 6)
    tw.K = 6
    tw.check()


def _slot_of(st, r):
    return int(st[r, :4].view(np.uint32)[0])


@pytest.mark.parametrize("cap_mode", ["keep", "new"])
def test_retire_moves_the_slots(fr, cap_mode):
    rng = np.random.default_rng(21 + (cap_mode == "new"))
    n = 900
    pt, L, st = _batch(fr, rng, 256, ALL, False, n)
    tw = Twin(fr, L, st, n + 20, 4)
    tw.arm(requests(rng, L, n + 20, 1500, cancel=0.0, step_hi=64))
    tw.arm(requests(rng, L, n + 20, 200))
    runs = rng.choice(n, size=300, replace=False).astype(np.uint32)
    m = n - 300
    capacity = 0 if cap_mode == "keep" else m + 5
    got_m, mf, mt = fr.resident_retire(tw.h, n, runs, capacity)
    assert got_m == m
    tw.area = T.retire(tw.area, n, runs, capacity)
    tw.state = fr.resident_download(tw.h, 0, tw.cap, L.state_stride)   # the records: tests/test_gpu_retire.py
    tw.check()
    tw.fire(m, 600)
    tw.check()


def test_transfer_moves_the_slots_and_refuses_a_run_that_does_not_fit(fr):
    rng = np.random.default_rng(31)
    n = 600
    pt, L, st = _batch(fr, rng, 256, ALL, False, n)
    src = Twin(fr, L, st, n, 4)
    Ld = make_layout(512, 0, ALL)
    dst = Twin(fr, Ld, np.zeros((0, Ld.state_stride), np.uint8), 400, 2)
    nk = fr.resident_create(Ld, 400)   # a destination without a timer area
    src.arm(requests(rng, L, n, 900, cancel=0.0))
    full = np.zeros(3 * 10, dtype=Frontier.TIMER_DTYPE)   # runs 0, 60, ..., 540 hold 3 or 4 armed timers
    for i in range(30):
        full[i] = (60 * (i // 3), 250 + i % 3, A.DEC_TIMED_OUT, 0, 50 + i, 0)
    src.arm(full)
    counts = np.array([len(T.armed(src.area[r])) for r in range(n)])
    fit = np.nonzero(counts <= 2)[0]
    bad = np.nonzero(counts > 2)[0]
    assert fit.size > 30 and bad.size > 0 and np.nonzero(counts)[0].size > 0
    # refusals: a run with 3+ armed slots into K = 2, any armed run into a batch without an area
    before_src, before_dst = src.slots().copy(), dst.slots().copy()
    for d, runs in ((dst.h, np.array([fit[0], bad[0]], np.uint32)), (nk, np.array([np.nonzero(counts)[0][0]], np.uint32))):
        with pytest.raises(A.FrontierError) as e:
            fr.resident_transfer(src.h, d, n, 0, runs)
        assert e.value.unfit == len(runs) - 1
    assert np.array_equal(src.slots(), before_src) and np.array_equal(dst.slots(), before_dst)
    src.check()
    runs = rng.choice(fit, size=min(100, fit.size), replace=False).astype(np.uint32)
    out = fr.resident_transfer(src.h, dst.h, n, 0, runs)
    assert out["src_n_runs"] == n - runs.size
    src.area, dst.area = T.transfer(src.area, dst.area, n, 0, runs)
    src.state = fr.resident_download(src.h, 0, src.cap, L.state_stride)
    dst.state = fr.resident_download(dst.h, 0, dst.cap, Ld.state_stride)
    src.check()
    dst.check()
    dst.fire(runs.size, 700)
    dst.check()


def test_migrate_re_indexes_the_slots(fr):
    rng = np.random.default_rng(41)
    n = 500
    ts = randgen.random_topologies(rng, 2, 60, 60, max_deg=3, parallel=False, fill=0.5)
    slots = fr.put_topologies(ts)
    L0, st0, topo = randgen.random_state(rng, ts, slots, n, A.F_DECISION, phase_mix="progress")
    L = make_layout(64, 0, L0.fields)
    from tests import reshape as RS
    st = RS.reshape_state(L0, L, st0, n)
    tw = Twin(fr, L, st, n, 6)
    tw.arm(requests(rng, L, n, 1500, cancel=0.0, step_hi=64))   # steps past S of the old slot too: cancelled by the migrate
    old, new = int(slots[0]), int(slots[1])
    S_old, S_new = int(ts.S[0]), int(ts.S[1])
    perm = rng.permutation(S_new)[:S_old].astype(np.uint16)
    perm[rng.random(S_old) < 0.2] = T.MIGRATE_GONE
    migrated = [r for r in range(n) if _slot_of(tw.state, r) == old]
    got = fr.resident_migrate(tw.h, old, new, perm, n)
    assert got == len(migrated) > 0
    tw.area = T.migrate(tw.area, migrated, perm)
    tw.state = fr.resident_download(tw.h, 0, n, L.state_stride)
    tw.check()


def test_redrive_empties_the_slots_of_applied_requests(fr):
    rng = np.random.default_rng(51)
    n = 400
    pt, L, st = _batch(fr, rng, 128, ALL, False, n)
    tw = Twin(fr, L, st, n, 3)
    tw.arm(requests(rng, L, n, 700, cancel=0.0, step_hi=16))
    live = sorted({_slot_of(tw.state, r) for r in range(n)})
    assert len(live) > 1
    runs = rng.choice(n, size=120, replace=False)
    rq = np.zeros(runs.size + 1, dtype=Frontier.REDRIVE_DTYPE)
    for i, r in enumerate(runs):
        s = _slot_of(tw.state, int(r))
        if i % 5 == 0:   # stale: another live slot than the run's
            s = live[(live.index(s) + 1) % len(live)]
        rq[i] = (int(r), s, A.REDRIVE_ALL if i % 2 else 0, 0)
    rq[-1] = rq[1]   # two requests of one run
    rq[-1]["step"] = 0
    status, applied = fr.resident_redrive(tw.h, rq)
    assert 0 < applied < rq.shape[0]
    tw.area = T.redrive(tw.area, rq, status)
    tw.state = fr.resident_download(tw.h, 0, n, L.state_stride)
    tw.check()


def test_reshape_extends_and_narrow_counts_the_slots(fr):
    rng = np.random.default_rng(61)
    n = 300
    pt, L, st = _batch(fr, rng, 256, A.F_DECISION | A.F_ALL_OUT, False, n)
    tw = Twin(fr, L, st, n, 2)
    tw.arm(requests(rng, L, n, 200, cancel=0.0, step_hi=200))
    Lb = make_layout(512, 0, L.fields)
    fr.resident_reshape(tw.h, Lb, n + 100)
    tw.L, tw.area = Lb, T.reshape(tw.area, n + 100)
    tw.state = fr.resident_download(tw.h, 0, n + 100, Lb.state_stride)
    tw.check()
    fr.resident_tick_touched(tw.h, n, NONE, n, BIG)
    e = fr.resident_extent(tw.h, n)
    steps, fields, widest = T.extent(tw.area)
    assert e["steps_max"] >= steps and (e["fields"] & fields) == fields
    # one armed timeout at step 400: no width below 401, and the decision planes stay
    rq = np.zeros(1, dtype=Frontier.TIMER_DTYPE)
    rq[0] = (n + 50, 400, A.DEC_TIMED_OUT, 0, 9, 0)
    tw.arm(rq)
    e = fr.resident_extent(tw.h, n)
    assert e["steps_max"] == 401 and e["widest_run"] == n + 50 and e["fields"] & A.F_DECISION
    with pytest.raises(A.FrontierError):
        fr.resident_narrow(tw.h, make_layout(400, 0, L.fields), n)
    with pytest.raises(A.FrontierError) as err:
        fr.resident_narrow(tw.h, make_layout(512, 0, A.F_ALL_OUT), n)
    assert err.value.extent["fields"] & A.F_DECISION
    tw.check()
    fr.resident_narrow(tw.h, make_layout(416, 0, L.fields), n)
    tw.L = make_layout(416, 0, L.fields)
    tw.state = fr.resident_download(tw.h, 0, n + 100, tw.L.state_stride)
    tw.check()


def _launches(fr):
    return fr.stats()["kernel_launches"]


def test_a_batch_without_timers_launches_what_it_did_before(fr):
    """the launch counts each call documents, on a batch that never enabled timers"""
    rng = np.random.default_rng(71)
    n = 300
    pt, L, st = _batch(fr, rng, 128, ALL, False, n)
    h = fr.resident_create(L, n + 10)
    h2 = fr.resident_create(make_layout(256, 0, ALL), n)
    fr.resident_upload(h, 0, st)

    def count(call):
        a = _launches(fr)
        call()
        return _launches(fr) - a

    assert count(lambda: fr.resident_tick_touched(h, n, NONE, n, BIG)) >= 1
    slot = _slot_of(st, 0)
    rq = np.zeros(1, dtype=Frontier.REDRIVE_DTYPE)
    rq[0] = (0, slot, A.REDRIVE_ALL, 0)
    assert count(lambda: fr.resident_redrive(h, rq)) == 1
    assert count(lambda: fr.resident_extent(h, n)) == 1
    assert count(lambda: fr.resident_retire(h, n, np.array([3, 7], np.uint32))) == 1
    assert count(lambda: fr.resident_retire(h, n - 2, np.zeros(0, np.uint32), n - 2)) == 0
    assert count(lambda: fr.resident_reshape(h, make_layout(256, 0, ALL), n + 20)) == 0   # reshape counts no launch
    assert count(lambda: fr.resident_transfer(h, h2, n - 2, 0, np.array([0, 1], np.uint32))) == 3
    with_t = fr.resident_create(L, n)
    fr.resident_timers(with_t, 2)
    assert count(lambda: fr.resident_reshape(with_t, L, n + 20)) == 1   # the timer area follows the capacity
    assert count(lambda: fr.resident_fire(with_t, n, 5)) == 2
