"""StoryRun stops and deadlines of a resident batch on the device (bf_resident_runctl, _runctl_put, _runctl_download and the run
level of bf_resident_fire) against the host model tests/runctl.py, byte for byte: the state records, the run-control records,
the timer slots, the limiter inputs, the fired list, the counts and next_deadline.  Also: the ticks after a stop evaluate and
list the stopped runs as touched runs, give them no events and group BF_GROUP_DONE, and agree with bf_eval_compact over the same
records; a schedule lists no launch for a stopped run and counts its Running steps; refusals change nothing; and a batch that
never enables run control launches what it launched before."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import runctl as R
from tests import timers as T
from tests.test_gpu_reshape import _batch
from tests.test_gpu_timers import requests as timer_requests

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def puts(rng, cap, k, p_stop=0.2, hi=1000):
    """k requests on distinct runs below cap: random deadlines (some none), some stops of random reasons"""
    runs = rng.choice(cap, size=min(k, cap), replace=False)
    q = np.zeros(len(runs), dtype=R.PUT_DTYPE)
    for i, r in enumerate(runs):
        sd = R.NONE if rng.random() < 0.3 else int(rng.integers(0, hi))
        dd = R.NONE if rng.random() < 0.6 else int(rng.integers(0, hi))
        st = int(rng.integers(1, 4)) if rng.random() < p_stop else 0
        q[i] = (int(r), sd, dd, st, (0, 0, 0))
    return q


class Twin:
    """a device batch with a run-control area (and optionally timers and limiter inputs) and its model"""

    def __init__(self, fr, L, st, cap, K=0, sched=False):
        self.fr, self.L, self.K = fr, L, K
        self.h = fr.resident_create(L, cap)
        if len(st):
            fr.resident_upload(self.h, 0, st)
        if K:
            fr.resident_timers(self.h, K)
        self.sched = None
        if sched:
            fr.resident_sched(self.h)
            self.sched = fr.resident_sched_download(self.h, 0, cap)
        fr.resident_runctl(self.h)
        fr.resident_runctl(self.h)   # again: nothing changes
        self.state = fr.resident_download(self.h, 0, cap, L.state_stride)
        self.timers = T.empty_area(cap, K) if K else None
        self.area = R.defaults(cap)

    @property
    def cap(self):
        return self.area.shape[0]

    def check(self):
        fr, h = self.fr, self.h
        assert fr.resident_runctl_download(h, 0, self.cap).tobytes() == self.area.tobytes(), "run-control records differ"
        assert np.array_equal(fr.resident_download(h, 0, self.cap, self.L.state_stride), self.state), "state records differ"
        if self.K:
            got = fr.resident_timers_download(h, 0, self.cap, self.K).view(np.uint64).reshape(self.cap, self.K)
            assert np.array_equal(got, self.timers), "timer slots differ"
        if self.sched is not None:
            assert fr.resident_sched_download(h, 0, self.cap).tobytes() == self.sched.tobytes(), "limiter inputs differ"

    def put(self, q):
        rc = R.check_put(self.area, q)
        if rc:
            with pytest.raises(A.FrontierError):
                self.fr.resident_runctl_put(self.h, q)
            return rc, set()
        self.fr.resident_runctl_put(self.h, q)
        return R.put(self.area, self.state, q, self.timers, self.sched)

    def arm(self, rq):
        if T.check_arm(self.timers, self.L, rq)[0] == 0:
            self.fr.resident_timers_arm(self.h, rq)
            T.arm(self.timers, self.L, rq)

    def fire(self, n_runs, now, cap=None):
        got = self.fr.resident_fire(self.h, n_runs, now, fired_cap=cap)
        want = R.fire(self.area, self.L, self.state, self.timers, n_runs, now, self.sched)
        for k in ("n_fired", "n_written", "n_pruned", "next_deadline"):
            assert got[k] == want[k], (k, got[k], want[k])
        lst = [tuple(int(x) for x in e) for e in got["fired"]]
        assert lst == want["fired"][:len(lst)] and len(lst) == min(want["n_fired"], 4096 if cap is None else cap)
        return want

    def flags_deltas(self, rng, k):
        d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
        runs = rng.choice(self.cap, size=k, replace=False)
        for i, r in enumerate(runs):
            d[i] = (int(r), 0, A.DELTA_RUN_FLAGS, int(rng.choice([0, 1, 2, 3, 5])))
        self.fr.resident_apply(self.h, d)
        for x in R.deltas(self.area, self.state, d):
            self.state[int(x["run"])][4] = x["code"]


# (S, fields, K, limiter inputs, runs)
CASES = [(64, ALL, 4, True, 700), (256, A.F_DECISION, 0, False, 30_000), (1024, ALL, 2, True, 300), (256, 0, 3, False, 1),
         (64, A.F_DECISION | A.F_ALL_OUT, 0, True, 5000)]


@pytest.mark.parametrize("S,fields,K,sched,n", CASES)
def test_random_puts_and_fires_match_the_model(fr, S, fields, K, sched, n):
    rng = np.random.default_rng(S + K + n)
    pt, L, st = _batch(fr, rng, S, fields, False, n)
    tw = Twin(fr, L, st, n + 9, K, sched)
    now = 0
    for step in range(8):
        tw.put(puts(rng, tw.cap, int(rng.integers(1, max(2, tw.cap // 3))), p_stop=0.05))
        tw.check()
        if K:
            tw.arm(timer_requests(rng, L, tw.cap, int(rng.integers(1, tw.cap)), step_hi=min(S, 40)))
        if step % 3 == 1:
            tw.flags_deltas(rng, min(tw.cap, 50))
        now += int(rng.integers(0, 200))
        tw.fire(int(rng.choice([0, n, tw.cap, max(0, n // 2)])), now, cap=int(rng.choice([0, 5, 4096, 100_000])))
        tw.check()
    # one more fire far ahead: every story and drain deadline of the runs fired is gone or dormant
    tw.fire(tw.cap, R.NONE - 1, cap=200_000)
    tw.check()


def test_batch_sizes_and_a_batch_without_timers(fr):
    """K = 0 with run control; n_runs 0, 1 and one past a CTA"""
    rng = np.random.default_rng(5)
    for n in (1, 257, 2049):
        pt, L, st = _batch(fr, rng, 64, A.F_DECISION, False, n)
        tw = Twin(fr, L, st, n)
        q = puts(rng, n, n, p_stop=0.1, hi=50)
        tw.put(q)
        assert tw.fire(0, 100)["n_fired"] == 0
        tw.fire(n, 25)
        tw.fire(n, 100)
        tw.check()
        fr.resident_destroy(tw.h)


def _stopped_batch(fr, rng, n, S=256):
    pt, L, st = _batch(fr, rng, S, ALL, False, n)
    return pt, L, st


def test_ticks_after_stops(fr):
    rng = np.random.default_rng(77)
    n = 3000
    pt, L, st = _stopped_batch(fr, rng, n)
    tw = Twin(fr, L, st, n, K=2)
    first = fr.resident_tick_touched(tw.h, n, NONE_D, n, BIG)
    assert first["full"] == 1
    q = puts(rng, n, 600, p_stop=0.5, hi=100)
    _, touched = tw.put(q)
    out = tw.fire(n, 60)
    touched |= out["touched"]
    assert len(touched) > 200
    t = fr.resident_tick_touched(tw.h, n, NONE_D, n, BIG)
    assert t["full"] == 0 and t["n_evaluated"] == len(touched)
    listed = set(int(x) for x in t["runs"])
    assert listed <= touched
    for r, hd in zip(t["runs"], t["head"]):
        assert tw.area["stop"][r]
        assert int(hd) & A.SUM_GROUP_MASK == 3 and int(hd) >> A.HEAD_COUNT_SHIFT == 0
    # dense, compact and changed-only agree with bf_eval_compact over the same records (the pass the host path runs)
    head, ev, ne, _ = fr.eval_compact(L, tw.state, BIG)
    h2, ev2, ne2, _, _ = fr.resident_tick_compact(tw.h, n, NONE_D, BIG)
    assert np.array_equal(head & ~np.uint32(A.HEAD_LISTED), h2 & ~np.uint32(A.HEAD_LISTED)) and ne == ne2
    assert np.array_equal(ev, ev2)
    stopped = np.nonzero(tw.area["stop"][:n])[0]
    assert np.all((h2[stopped] & A.SUM_GROUP_MASK) == 3) and np.all((h2[stopped] >> A.HEAD_COUNT_SHIFT) == 0)
    ref = fr.resident_create(L, n)
    fr.resident_upload(ref, 0, tw.state)
    assert np.array_equal(fr.resident_tick(tw.h, L, n, NONE_D)[0], fr.resident_tick(ref, L, n, NONE_D)[0])
    a = fr.resident_tick_compact(tw.h, n, NONE_D, BIG, flags=A.EVAL_CHANGED_ONLY)
    b = fr.resident_tick_compact(ref, n, NONE_D, BIG, flags=A.EVAL_CHANGED_ONLY)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    tw.check()


def test_a_schedule_lists_no_launch_of_a_stopped_run(fr):
    rng = np.random.default_rng(79)
    n = 2000
    pt, L, st = _stopped_batch(fr, rng, n, S=128)
    tw = Twin(fr, L, st, n, sched=True)
    inputs = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
    inputs["run"] = np.arange(n)
    inputs["story_key"] = rng.integers(0, 4, n)
    inputs["queue_key"] = rng.integers(0, 3, n)
    inputs["priority"] = rng.integers(0, 5, n)
    inputs["queued_since"] = A.SCHED_NONE
    inputs["run_phase"] = A.PHASE_RUNNING
    fr.resident_sched_put(tw.h, inputs)
    tw.sched = fr.resident_sched_download(tw.h, 0, n)
    _, touched = tw.put(puts(rng, n, 500, p_stop=0.6, hi=10))
    tw.fire(n, 5)
    tw.check()
    # the same records and inputs in a batch without run control: the schedule must be identical
    ref = fr.resident_create(L, n)
    fr.resident_upload(ref, 0, tw.state)
    fr.resident_sched(ref)
    ri = tw.sched.copy()
    ri["run"] = np.arange(n)
    fr.resident_sched_put(ref, ri)
    tables = dict(story_limit=[3, 5, 1000, 2], queue_limit=[4, 1000, 7], queue_aging_s=[0, 60, 10], global_limit=5000)
    got = []
    for h in (tw.h, ref):
        fr.resident_tick_compact(h, n, NONE_D, BIG)
        got.append(fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], tables, 100))
    a, b = got
    for k in ("story_running", "queue_running", "queue_max_priority", "global_running"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    pa, pb = a["parts"][0], b["parts"][0]
    for k in ("runs", "heads", "events"):
        assert np.array_equal(np.asarray(pa[k]), np.asarray(pb[k])), k
    stopped = set(np.nonzero(tw.area["stop"][:n])[0].tolist())
    assert stopped
    for r, hd in zip(pa["runs"], pa["heads"]):
        if int(r) in stopped:
            assert int(hd["n_launch"]) == 0


def test_refusals_change_nothing(fr):
    rng = np.random.default_rng(81)
    n = 300
    pt, L, st = _batch(fr, rng, 64, ALL, False, n)
    bare = fr.resident_create(L, n)
    fr.resident_upload(bare, 0, st)
    with pytest.raises(A.FrontierError):
        fr.resident_runctl_put(bare, puts(rng, n, 3))
    with pytest.raises(A.FrontierError):
        fr.resident_runctl_download(bare, 0, 1)
    with pytest.raises(A.FrontierError):
        fr.resident_fire(bare, n, 5)
    tw = Twin(fr, L, st, n, K=2)
    tw.put(puts(rng, n, 100, p_stop=0.3))
    tw.check()
    for bad in ("dup", "stop", "reserved", "run"):
        q = puts(rng, n, 5)
        if bad == "dup":
            q[1]["run"] = q[0]["run"]
        elif bad == "stop":
            q[2]["stop"] = 4
        elif bad == "reserved":
            q[3]["reserved"][1] = 1
        else:
            q[4]["run"] = n
        assert tw.put(q)[0] == R.EINVAL
        tw.check()
    with pytest.raises(A.FrontierError):
        fr.resident_runctl_download(tw.h, n - 1, 2)
    # a transfer into a batch without an area refuses a run with a non-default record: both batches byte-identical
    moved = int(np.nonzero(tw.area["stop"])[0][0])
    fr.resident_reshape(bare, L, n + 10)
    before = fr.resident_download(bare, 0, n + 10, L.state_stride)
    with pytest.raises(A.FrontierError) as e:
        fr.resident_transfer(tw.h, bare, n, n, [moved])
    assert "run-control" in str(e.value)
    tw.check()
    assert np.array_equal(fr.resident_download(bare, 0, n + 10, L.state_stride), before)


def _launches(fr, call):
    before = fr.stats()["kernel_launches"]
    call()
    return fr.stats()["kernel_launches"] - before


def test_launch_counts(fr):
    """a batch without run control launches what each call documents; with it, the upload adds its re-stop launch and nothing
    else changes; a put launches one kernel, a fire two"""
    rng = np.random.default_rng(83)
    n = 300
    pt, L, st = _batch(fr, rng, 64, ALL, False, n)
    counts = []
    for with_area in (False, True):
        h = fr.resident_create(L, n + 20)
        fr.resident_upload(h, 0, st)
        fr.resident_timers(h, 2)
        if with_area:
            fr.resident_runctl(h)
            assert _launches(fr, lambda: fr.resident_runctl_put(h, puts(rng, n, 20, p_stop=0.5))) == 1
        d = np.zeros(3, dtype=Frontier.DELTA_DTYPE)
        d[0] = (1, 0, A.DELTA_RUN_FLAGS, 1)
        seq = [_launches(fr, lambda: fr.resident_upload(h, 5, st[5:9])),
               _launches(fr, lambda: fr.resident_apply(h, d[:1])),
               _launches(fr, lambda: fr.resident_fire(h, n, 10)),
               _launches(fr, lambda: fr.resident_redrive(h, np.array([(2, int(st[2][:4].view("<u4")[0]), A.REDRIVE_ALL, 0)],
                                                                      dtype=Frontier.REDRIVE_DTYPE))),
               _launches(fr, lambda: fr.resident_retire(h, n, [0, 7])),
               _launches(fr, lambda: fr.resident_reshape(h, L, n + 40))]
        counts.append(seq)
        fr.resident_destroy(h)
    assert counts[0] == [1, 1, 2, 1, 1, 1], counts[0]
    assert counts[1] == [2, 1, 2, 1, 1, 1], counts[1]
