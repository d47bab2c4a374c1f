"""The host model of resident schedules (tests/sched_resident.py) pinned on the CPU: elapsed time from the stored queue origin,
shared totals across batches, the listing rule after each kind of lifecycle call, the defaults and the put refusals."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from oracle import limiters as LM
from tests import randgen
from tests import sched_resident as SRM
from tests import schedref as SR

NONE = A.SCHED_NONE


def _batch(rng, n, smax, smin=1, count=12, parallel=True):
    ts = randgen.random_topologies(rng, count, smin, smax, parallel=parallel)
    slots = np.arange(ts.count, dtype=np.uint32)
    L, state, _ = randgen.random_state(rng, ts, slots, n, A.F_COND | A.F_DECISION, phase_mix="progress")
    result = rng.integers(0, 256, size=(n, L.result_stride), dtype=np.uint8)
    return L, state, result, SR.from_topology_set(ts, slots)


def _inputs(rng, n, ns, nq, now):
    p = SRM.defaults(n)
    p["run"] = np.arange(n)
    p["story_key"] = rng.integers(0, ns + 1, size=n)
    p["queue_key"] = rng.integers(0, nq + 1, size=n)
    p["priority"] = rng.integers(-3, 6, size=n)
    p["queued_since"] = np.where(rng.random(n) < 0.3, NONE, rng.integers(0, now + 100, size=n))
    p["run_phase"] = rng.integers(0, 16, size=n)
    return p


def test_elapsed_from_the_queue_origin():
    now = 1000
    got = SRM.elapsed([NONE, 1001, 1000, 999, 0, 940], now)
    assert got.tolist() == [NONE, 0, 0, 1, 1000, 60]
    # aging boundaries at 60 s: 59 keeps the base, 60 and 119 add one step, 120 adds two
    el = SRM.elapsed([1000 - 59, 1000 - 60, 1000 - 119, 1000 - 120], now)
    assert SR.effective_priority_rows([5] * 4, el, [60] * 4).tolist() == [5, 6, 6, 7]
    # past INT32_MAX units the elapsed time is clamped, and the int32 sum wraps
    el = SRM.elapsed([0, 0], 0xFFFFFFFE)
    assert el.tolist() == [0xFFFFFFFE, 0xFFFFFFFE]
    assert SR.effective_priority_rows([0, SR.INT32_MAX], el, [1, 1]).tolist() == [SR.INT32_MAX, -2]
    # an origin at or past now is Go's elapsed <= 0: the base priority
    assert SR.effective_priority_rows([3, 3], SRM.elapsed([5, 6], 5), [1, 1]).tolist() == [3, 3]


@pytest.mark.parametrize("seed", range(3))
def test_two_batches_share_their_totals(seed):
    """the records and totals of two batches limited together equal schedref.expected over their concatenation"""
    rng = np.random.default_rng(40 + seed)
    L, state, result, descs = _batch(rng, 600, 90)
    now = 5000
    inputs = _inputs(rng, 600, 20, 4, now)
    tables = SR.random_tables(rng, 20, 4, 600, maxprio_base=bool(seed % 2))
    a, b = SRM.Batch(L, 400), SRM.Batch(L, 200)
    a.put(inputs[:400])
    q = inputs[400:].copy()
    q["run"] -= 400
    b.put(q)
    got = SRM.schedule([(a, 400, state[:400], result[:400], descs), (b, 200, state[400:], result[400:], descs)], tables, now)
    want = SR.expected(L, state, result, descs, SRM.sched_runs(inputs, now), tables)
    recs = np.concatenate([p["records"] for p in got["parts"]])
    SR.assert_schedule({**got, "records": recs}, want, "two batches")
    assert all(p["full"] for p in got["parts"])


def test_widths_share_their_totals():
    """batches of different widths: each run's record is bf_schedule's for its batch with the other batch's counts as bases"""
    rng = np.random.default_rng(7)
    L1, s1, r1, d1 = _batch(rng, 300, 60)
    L2, s2, r2, d2 = _batch(rng, 200, 700, smin=300)
    now = 900
    tables = SR.random_tables(rng, 10, 3, 500, maxprio_base=True)
    a, b = SRM.Batch(L1, 300), SRM.Batch(L2, 200)
    i1, i2 = _inputs(rng, 300, 10, 3, now), _inputs(rng, 200, 10, 3, now)
    a.put(i1)
    b.put(i2)
    got = SRM.schedule([(a, 300, s1, r1, d1), (b, 200, s2, r2, d2)], tables, now)
    for (L, st, res, ds, inp, part), (Lo, sto, reso, dso, inpo) in (
            ((L1, s1, r1, d1, i1, got["parts"][0]), (L2, s2, r2, d2, i2)), ((L2, s2, r2, d2, i2, got["parts"][1]), (L1, s1, r1, d1, i1))):
        other = SR.expected(Lo, sto, reso, dso, SRM.sched_runs(inpo, now), {**tables, "global_limit": 0})
        t = dict(tables)
        t["story_running_base"] = other["story_running"]
        t["queue_running_base"] = other["queue_running"]
        t["global_running_base"] = other["global_running"]
        t["queue_max_priority_base"] = other["queue_max_priority"]
        want = SR.expected(L, st, res, ds, SRM.sched_runs(inp, now), t)
        assert np.array_equal(part["records"], want["records"])
        assert np.array_equal(got["story_running"], want["story_running"]) and got["global_running"] == want["global_running"]


def _listed(batch, n, state, result, descs, tables, now):
    return SRM.schedule([(batch, n, state, result, descs)], tables, now)["parts"][0]


def test_listing_after_each_lifecycle_call():
    rng = np.random.default_rng(3)
    L, state, result, descs = _batch(rng, 256, 64)
    tables = SR.random_tables(rng, 8, 2, 256, edges=False)
    now = 100
    b = SRM.Batch(L, 256)
    b.put(_inputs(rng, 200, 8, 2, now))
    listed = lambda n: _listed(b, n, state[:n], result[:n], descs, tables, now)  # noqa: E731
    first = listed(200)
    assert first["full"] == 1 and first["listed"].size == 200
    assert listed(200)["listed"].size == 0                              # nothing changed: nothing listed
    b.upload(10, 3)
    assert listed(200)["listed"].tolist() == [10, 11, 12]
    assert listed(210)["listed"].tolist() == list(range(200, 210))      # past the previous n_runs
    assert listed(205)["listed"].size == 0
    assert listed(210)["listed"].tolist() == list(range(205, 210))      # past the previous schedule's n_runs again
    moves = b.retire(210, [0, 5, 209])
    assert moves == [(207, 0), (208, 5)] and b.base_runs == 207
    assert listed(207)["listed"].tolist() == [0, 5]                     # the movers' targets (the records did not move here)
    b.receive(207, SRM.defaults(3))
    assert listed(210)["listed"].tolist() == [207, 208, 209]
    b.relayout(L)                                                       # same words: baselines kept
    assert listed(210)["listed"].size == 0
    b.lose_baseline([3, 9])                                             # migrated runs
    assert listed(210)["listed"].tolist() == [3, 9]
    b.relayout(A.Layout(**{**L.as_dict(), "words": L.words + 1}))
    assert b.base_runs == 0


def test_aging_lists_runs_without_puts():
    """the host writes nothing as time passes; a later `now` may still change (and list) runs whose priority ages"""
    rng = np.random.default_rng(11)
    L, state, result, descs = _batch(rng, 300, 40)
    tables = SR.random_tables(rng, 4, 2, 300, edges=False)
    tables["queue_aging_s"] = np.array([1, 1], np.int32)
    b = SRM.Batch(L, 300)
    inp = _inputs(rng, 300, 4, 2, 100)
    inp["queued_since"] = np.where(np.arange(300) % 2, 50, NONE)
    b.put(inp)
    _listed(b, 300, state, result, descs, tables, 50)     # the queued runs' origin: no aging yet
    before = [r.copy() for r in b.rec]
    later = _listed(b, 300, state, result, descs, tables, 100 + 10_000_000)
    ref = SR.expected(L, state, result, descs, SRM.sched_runs(inp, 100 + 10_000_000), tables)
    assert np.array_equal(later["records"], ref["records"])
    changed = [r for r in range(300) if not np.array_equal(before[r], ref["records"][r])]
    assert changed and later["listed"].tolist() == changed          # aging alone changed these records, and only these are listed


def test_defaults_and_put_refusals():
    b = SRM.Batch(A.Layout(words=1), 8)
    d = b.download(0, 8)
    assert (d["story_key"] == NONE).all() and (d["queue_key"] == NONE).all() and (d["queued_since"] == NONE).all()
    assert (d["priority"] == 0).all() and (d["run_phase"] == 0).all() and d["run"].tolist() == list(range(8))
    for bad in ([(8, 0, 0, 0, 0, 0, (0, 0))], [(1, 0, 0, 0, 0, 0, (0, 1))], [(1, 0, 0, 0, 0, 0, (0, 0)), (1, 2, 0, 0, 0, 0, (0, 0))]):
        with pytest.raises(SRM.PutRefused):
            b.put(np.array(bad, SRM.PUT_DTYPE))
        assert np.array_equal(b.download(0, 8), d)    # a refused put changes nothing
    b.put(np.array([(3, 1, 2, -7, 40, 2, (0, 0))], SRM.PUT_DTYPE))
    assert b.download(3, 1)[0].tolist()[:6] == (3, 1, 2, -7, 40, 2)


def test_decode_round_trip():
    rng = np.random.default_rng(5)
    L, state, result, descs = _batch(rng, 100, 200)
    tables = SR.random_tables(rng, 4, 2, 100, edges=False)
    b = SRM.Batch(L, 100)
    b.put(_inputs(rng, 100, 4, 2, 10))
    p = _listed(b, 100, state, result, descs, tables, 10)
    assert np.array_equal(SRM.decode(L.words, 100, p["listed"], p["heads"], p["events"]), p["records"])
    assert LM.NONE_U32 == NONE
