"""The composed side-area model of tests/lifecycle.py on its own, without a GPU.  The directed area-set matrix of
tests/test_gpu_run_areas.py must reach every fit rule of a transfer (so that its device comparisons cannot pass vacuously), an
arrival takes the defaults of each area its source lacks, a retire to a smaller capacity keeps every area's prefix, and a fire
equals its written codes sent as decision deltas plus its story timeouts sent as stops, areas aside."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import make_layout
from tests import runctl as R
from tests import sched_resident as SRM
from tests import timers as T
from tests.lifecycle import (MOVED, RUNCTL, SCHED, TIMERS, Refused, area_sets, beyond_requests, records_of, seeded,
                             template_records)

FIELDS = A.F_COND | A.F_DECISION | A.F_OUT_FAIL | A.F_OUT_SKIP_DEP
L = make_layout(64, 0, FIELDS)
S = [22, 20]
N, CAP, NOW = 16, 24, 5000
SETS = area_sets()
DELTA = np.dtype([("run", "<u4"), ("index", "<u2"), ("field", "u1"), ("code", "u1")])   # bf_delta


def batch(subset, K, n=N):
    return seeded(L, CAP, subset, K, records_of(template_records(L, [0, 1], S), n), S[0] - 1, NOW)[0]


def outcome(src, dst):
    a, b = batch(*src), batch(*dst, n=4)
    p, arms, q = beyond_requests(b, NOW)
    if b.sched is not None:
        b.put_sched(p)
    if b.K:
        assert b.arm(arms) == 0
    if b.runctl is not None:
        assert b.put_runctl(q)[0] == 0
    try:
        a.transfer(b, b.n, MOVED)
        return "ok", a, b
    except Refused as e:
        return (e.unfit, frozenset(e.lost) or frozenset({"sched"})), a, b


def test_transfer_matrix_reaches_every_fit_rule():
    seen = {}
    for src in SETS:
        for dst in SETS:
            seen[(src, dst)] = outcome(src, dst)[0]
    # a destination without limiter inputs refuses a source that has them, before any run is looked at
    for (src, dst), o in seen.items():
        if src[0] & SCHED and not dst[0] & SCHED:
            assert o == (A.EXTENT_NO_RUN, frozenset({"sched"}))
    # K down: run 5's four armed slots do not fit K = 2; K up: two fit K = 5
    assert seen[((TIMERS | SCHED, 5), (TIMERS | SCHED, 2))] == (2, frozenset({"timers"}))
    assert seen[((TIMERS | SCHED, 2), (TIMERS | SCHED, 5))] == "ok"
    # no timer area: run 6's one armed slot is the first that does not fit
    assert seen[((TIMERS, 2), (0, 0))] == (1, frozenset({"timers"}))
    # a lost run-control record (run 5's story deadline), alone and with too many armed slots
    assert seen[((RUNCTL, 0), (0, 0))] == (2, frozenset({"runctl"}))
    assert seen[((TIMERS | RUNCTL, 5), (TIMERS, 2))] == (2, frozenset({"timers", "runctl"}))
    # every rule decides some pair, and some pairs of every kind are accepted
    lost = set().union(*(o[1] for o in seen.values() if o != "ok"))
    assert lost == {"timers", "runctl", "sched"}
    assert sum(o == "ok" for o in seen.values()) >= 20


def test_arrivals_take_the_defaults_of_areas_the_source_lacks():
    for src in SETS:
        for dst in SETS:
            o, a, b = outcome(src, dst)
            if o != "ok":
                continue
            a0 = batch(*src)
            for i, r in enumerate(MOVED):
                to = 4 + i
                assert np.array_equal(b.state[to], a0.state[r])
                if b.timers is not None:
                    want = T.canonical({} if a0.timers is None else {s: (d, c) for s, d, c in T.armed(a0.timers[r])}, b.K)
                    assert np.array_equal(b.timers[to], want)
                if b.runctl is not None:
                    want = R.defaults(1)[0] if a0.runctl is None else a0.runctl[r]
                    assert b.runctl[to].tobytes() == want.tobytes()
                if b.sched is not None:
                    want = SRM.defaults(1)[0] if a0.sched is None else a0.sched.inputs[r]
                    assert b.sched.inputs[to].tobytes() == want.tobytes() and b.sched.rec[to] is None


def test_retire_to_a_smaller_capacity_keeps_every_prefix():
    b = batch(TIMERS | SCHED | RUNCTL, 5)
    full = batch(TIMERS | SCHED | RUNCTL, 5)
    full.retire(N, [1, 12, 14])
    m, mv = b.retire(N, [1, 12, 14], 14)
    assert (m, mv) == (13, {13: 1, 15: 12})
    assert b.cap == 14 and np.array_equal(b.state, full.state[:14])
    assert np.array_equal(b.timers, full.timers[:14])
    assert b.runctl.tobytes() == full.runctl[:14].tobytes()
    assert b.sched.inputs.tobytes() == full.sched.inputs[:14].tobytes()
    # the moved runs carry their entries: run 15 was stopped, run 13 armed
    assert b.runctl["stop"][12] and T.armed(b.timers[1])
    assert all(b.runctl[i].tobytes() == R.defaults(1)[0].tobytes() for i in (13,))


def test_fire_equals_its_codes_as_deltas_and_its_timeouts_as_stops():
    for now in (NOW + 100, NOW + 110, NOW + 205, NOW + 400):
        fired = batch(TIMERS | RUNCTL, 5)
        sent = batch(TIMERS | RUNCTL, 5)
        out = R.fire(fired.runctl, L, fired.state, fired.timers, N, now)
        for d in T.as_deltas([e for e in out["fired"] if e[1] < R.FIRED_DRAIN], DELTA):
            assert d["field"] == A.DELTA_DECISION
            T._set(sent.state[int(d["run"])], L.off_decision, L.words, 2, int(d["index"]), int(d["code"]))
        stops = [e[0] for e in out["fired"] if e[1] == R.FIRED_STORY]
        q = np.zeros(len(stops), R.PUT_DTYPE)
        for i, r in enumerate(stops):
            q[i] = (r, sent.runctl["story_deadline"][r], sent.runctl["drain_deadline"][r], R.STOP_TIMEOUT, (0, 0, 0))
        assert sent.put_runctl(q)[0] == 0
        assert np.array_equal(fired.state, sent.state), now
        assert out["n_written"] == sum(1 for e in out["fired"] if e[3])
