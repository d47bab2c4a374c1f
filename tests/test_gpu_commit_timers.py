"""Tick commits that arm step timers (bf_resident_commit_timed, bf_topology_timings) on the device, against the host model
tests/commit_timers.py byte for byte: state records, timer slots, counts, n_armed and next_deadline, over random batches with and
without a limiter area, K = 1, 2 and 8, stopped runs and a dead slot.  Also every refusal (records and slots unchanged), the
timings call, the steady-state loop against commit + bf_resident_timers_arm, a Story end to end, and a plain commit on a batch
with timings (arms nothing)."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import make_layout, pack_state, unpack_result
from tests import commit as M
from tests import commit_timers as CT
from tests import runctl as R
from tests import timers as T
from tests.test_gpu_commit import ALL, NONE_D, Twin, _batch, entries_for

pytestmark = pytest.mark.gpu

CODES = {A.STEP_SLEEP: (A.DEC_SUCCEED, A.DEC_FAIL), A.STEP_GATE: (A.DEC_TIMED_OUT, A.DEC_FAIL),
         A.STEP_WAIT: (A.DEC_TIMED_OUT, A.DEC_PENDING, A.DEC_FAIL)}


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def random_timings(rng, ts, slots, p=0.7, pending_only=False):
    """a timing for about p of the sleep / gate / wait steps of every other topology -> {slot: {step: (code, delay)}}"""
    out, s0 = {}, 0
    for i in range(ts.count):
        S = int(ts.S[i])
        types = ts.step_flags[s0:s0 + S] & A.SF_TYPE_MASK
        s0 += S
        if i % 2:
            continue
        t = {}
        for s in range(S):
            if int(types[s]) in CODES and rng.random() < p:
                codes = (A.DEC_PENDING,) if pending_only and int(types[s]) == A.STEP_WAIT else CODES[int(types[s])]
                if pending_only and int(types[s]) != A.STEP_WAIT:
                    continue
                t[s] = (int(rng.choice(codes)), int(rng.choice([0, 1, 3, 20, 0xFFFFFFFF])))
        out[int(slots[i])] = t
    return out


def put_all(fr, timings):
    for slot, t in timings.items():
        fr.put_timings(slot, [(s, c, d) for s, (c, d) in t.items()])


def commit_both(fr, tw, area, timings, res, ents, n, now):
    """one timed commit on the device and in the model; a refusal must leave records and slots as they were -> the model's tuple"""
    K = area.shape[1]
    want = CT.commit_timed(tw.L, tw.topo, timings, tw.state, res, tw.sched, n, ents, area, now, tw.L.off_decision != A.OFF_NONE)
    if want[0]:
        with pytest.raises(A.FrontierError) as e:
            fr.resident_commit(tw.h, n, ents, now=now)
        assert (e.value.status, e.value.bad_run, e.value.bad_step) == want[:3], (str(e.value), want[:3])
    else:
        got = fr.resident_commit(tw.h, n, ents, now=now)
        assert got == dict(want[3], n_armed=want[5], next_deadline=want[6]), (got, want)
    tw.check()
    assert np.array_equal(fr.resident_timers_download(tw.h, 0, area.shape[0], K).view("<u8"), area)
    return want


def fire_both(fr, tw, area, n, now):
    want = T.fire(area, tw.L, tw.state, n, now)
    got = fr.resident_fire(tw.h, n, now)
    assert (got["n_fired"], got["n_written"], got["n_pruned"], got["next_deadline"]) == \
        (want["n_fired"], want["n_written"], want["n_pruned"], want["next_deadline"])
    assert [tuple(int(x) for x in f) for f in got["fired"]] == want["fired"]
    return got


# (S, fields, K, limiter area, run control, runs)
CASES = [(64, ALL, 1, False, False, 800), (64, A.F_DECISION | A.F_ALL_OUT, 2, True, False, 3000), (256, ALL, 2, False, True, 20_000),
         (256, ALL, 8, True, True, 4000), (1024, ALL, 8, True, False, 300), (1024, ALL, 1, False, True, 60)]


@pytest.mark.parametrize("S,fields,K,sched,runctl,n", CASES)
def test_timed_commits_match_the_model(fr, S, fields, K, sched, runctl, n):
    rng = np.random.default_rng(S * 7 + K + n)
    ts, slots, L, st = _batch(fr, rng, S, fields, True, n)
    cap = n + 5
    tw = Twin(fr, ts, slots, L, st, cap, sched, runctl)
    fr.resident_timers(tw.h, K)
    area = T.empty_area(cap, K)
    timings = random_timings(rng, ts, slots)
    put_all(fr, timings)
    dead = int(slots[0])   # a dead slot: its runs have no masks and arm nothing
    fr.drop_topology(dead)
    tw.topo.drop(dead)
    timings.pop(dead, None)
    if runctl:
        q = np.zeros(min(n, 40), dtype=R.PUT_DTYPE)
        q["run"] = rng.choice(n, size=q.shape[0], replace=False)
        q["story_deadline"] = R.NONE
        q["drain_deadline"] = R.NONE
        q["stop"] = 2
        fr.resident_runctl_put(tw.h, q)
        R.put(tw.area, tw.state, q)
        area[q["run"]] = T.EMPTY
    armed_total = 0
    for rnd in range(5):
        now = 100 + 7 * rnd
        fire_both(fr, tw, area, n, now)
        res = tw.tick(now)
        ents = entries_for(rng, L, tw.topo, tw.state, res, tw.sched, n)
        want = commit_both(fr, tw, area, timings, res, ents, n, now)
        while want[0] == CT.ENOMEM:   # grow K and repeat the same commit: its preconditions still hold
            K = min(2 * K + 2, A.TIMER_MAX_SLOTS)
            fr.resident_timers(tw.h, K)
            area = T.grow(area, K)
            want = commit_both(fr, tw, area, timings, res, ents, n, now)
        assert want[0] in (0, M.EINVAL)
        armed_total += want[5]
    if n >= 300:
        assert armed_total > 0
    if runctl:
        stopped = np.nonzero(tw.area["stop"][:n])[0]
        assert all(not T.armed(area[r]) for r in stopped)


def test_refusals_change_nothing(fr):
    rng = np.random.default_rng(5)
    n = 1200
    ts, slots, L, st = _batch(fr, rng, 128, A.F_ALL_OUT, True, n)   # no decision planes
    tw = Twin(fr, ts, slots, L, st, n)
    res = tw.tick()
    with pytest.raises(A.FrontierError) as e:   # no timer area
        fr.resident_commit(tw.h, n, entries_for(rng, L, tw.topo, tw.state, res, None, n, p_error=0), now=5)
    assert (e.value.status, e.value.bad_run, e.value.bad_step) == (A.BF_EINVAL, M.NONE, M.NONE)
    fr.resident_timers(tw.h, 8)
    area = T.empty_area(n, 8)
    timings = random_timings(rng, ts, slots, p=1.0)
    put_all(fr, timings)
    ents = entries_for(rng, L, tw.topo, tw.state, res, None, n, p_error=0, p_hold=0.1)
    with pytest.raises(A.FrontierError) as e:   # now = BF_TIMER_NONE
        fr.resident_commit(tw.h, n, ents, now=A.TIMER_NONE)
    assert (e.value.status, e.value.bad_run, e.value.bad_step) == (A.BF_EINVAL, M.NONE, M.NONE)
    out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
    arm = A.CommitArm(struct_size=ctypes.sizeof(A.CommitArm) + 4, now=5)
    assert fr._lib.bf_resident_commit_timed(fr._ctx, tw.h, n, None, 0, ctypes.byref(out), ctypes.byref(arm)) == A.BF_EINVAL
    tw.check()
    # a code that writes on a batch without decision planes: refused at the lowest (run, step), as the model says
    want = commit_both(fr, tw, area, timings, res, ents, n, 5)
    assert want[0] == M.EINVAL and want[1] is not None
    # an entry offence below it wins
    r0 = want[1]
    bad = np.concatenate([ents, np.array([(0, L.steps_max - 1, M.HOLD, 0)], dtype=Frontier.COMMIT_DTYPE)]) if r0 > 0 else ents
    commit_both(fr, tw, area, timings, res, bad, n, 5)
    # wake-only timings alone arm on the same batch
    timings = random_timings(rng, ts, slots, p=1.0, pending_only=True)
    put_all(fr, timings)
    want = commit_both(fr, tw, area, timings, res, ents, n, 5)
    assert want[0] == 0 and want[5] > 0
    assert tw.touched_tick()["n_evaluated"] == want[3]["n_runs_written"]


def test_timings_call(fr):
    ts = TopologySet([4, 2], [0, 0], np.zeros(8, np.uint32), np.zeros(0, np.uint16),
                     np.array([A.STEP_SLEEP, A.STEP_GATE, A.STEP_WAIT, A.STEP_ENGRAM, A.STEP_SLEEP, A.STEP_STOP], np.uint8),
                     [0, 0], np.zeros(0, dtype=[("step", "<u2"), ("branches", "<u2"), ("allow_first", "<u4")]))
    slots = fr.put_topologies(ts)
    s = int(slots[0])
    ok = [(0, A.DEC_SUCCEED, 1), (1, A.DEC_TIMED_OUT, 2), (2, A.DEC_PENDING, 3)]
    fr.put_timings(s, ok)
    fr.put_timings(s, [(2, A.DEC_FAIL, 0), (0, A.DEC_FAIL, 9)])   # any order, replaces the set
    fr.put_timings(s, None)
    for bad in ([(4, A.DEC_SUCCEED, 1)], [(3, A.DEC_SUCCEED, 1)], [(0, A.DEC_TIMED_OUT, 1)], [(0, A.DEC_PENDING, 1)],
                [(1, A.DEC_SUCCEED, 1)], [(1, A.DEC_PENDING, 1)], [(2, A.DEC_SUCCEED, 1)], [(0, 4, 1)],
                [(0, A.DEC_SUCCEED, 1), (0, A.DEC_FAIL, 2)]):
        with pytest.raises(A.FrontierError) as e:
            fr.put_timings(s, bad)
        assert e.value.status == A.BF_EINVAL
    t = np.zeros(1, Frontier.TIMING_DTYPE)
    t[0] = (0, A.DEC_SUCCEED, 1, 5)   # reserved != 0
    with pytest.raises(A.FrontierError):
        fr.put_timings(s, t)
    with pytest.raises(A.FrontierError):
        fr.put_timings(999, ok)
    assert fr._lib.bf_topology_timings(fr._ctx, s, None, 2) == A.BF_EINVAL
    # a drop discards the timings and a put that reuses the slot starts with none
    fr.put_timings(s, ok)
    fr.drop_topology(s)
    with pytest.raises(A.FrontierError):
        fr.put_timings(s, ok)
    again = fr.put_topologies(TopologySet([4], [0], np.zeros(5, np.uint32), np.zeros(0, np.uint16),
                                          np.array([A.STEP_SLEEP, A.STEP_GATE, A.STEP_WAIT, A.STEP_ENGRAM], np.uint8), [0],
                                          np.zeros(0, dtype=[("step", "<u2"), ("branches", "<u2"), ("allow_first", "<u4")])))
    assert int(again[0]) == s
    L = make_layout(4, 0, A.F_DECISION | A.F_ALL_OUT)
    h = fr.resident_create(L, 4)
    fr.resident_upload(h, 0, pack_state(L, np.full(4, s, np.uint32), np.zeros(4, np.uint8), np.zeros((4, 4), np.uint8)))
    fr.resident_timers(h, 4)
    fr.resident_tick(h, L, 4, NONE_D)
    got = fr.resident_commit(h, 4, now=10)
    assert got["n_launched"] == 16 and (got["n_armed"], got["next_deadline"]) == (0, A.TIMER_NONE)


def test_plain_commit_arms_nothing(fr):
    """bf_resident_commit on a batch with timings and a timer area writes and launches what it did before, and arms nothing"""
    rng = np.random.default_rng(9)
    n = 3000
    ts, slots, L, st = _batch(fr, rng, 64, ALL, True, n)
    a, b = Twin(fr, ts, slots, L, st, n), Twin(fr, ts, slots, L, st, n)
    fr.resident_timers(a.h, 4)
    put_all(fr, random_timings(rng, ts, slots, p=1.0))
    res = a.tick()
    assert np.array_equal(res, b.tick())
    ents = entries_for(rng, L, a.topo, a.state, res, None, n)
    before = fr.stats()["kernel_launches"]
    got = fr.resident_commit(a.h, n, ents)
    assert fr.stats()["kernel_launches"] - before == 2
    assert got == fr.resident_commit(b.h, n, ents)
    assert np.array_equal(fr.resident_download(a.h, 0, n, L.state_stride), fr.resident_download(b.h, 0, n, L.state_stride))
    assert (fr.resident_timers_download(a.h, 0, n, 4)["deadline"] == A.TIMER_NONE).all()


def test_loop_equals_commit_plus_arm(fr):
    """>= 20 ticks of Fire -> tick -> commit with an advancing now: the timed commit on one batch, bf_resident_commit and
    bf_resident_timers_arm (requests from the launches and the current slots) on its twin; identical after every tick"""
    rng = np.random.default_rng(21)
    n = 2500
    ts, slots, L, st = _batch(fr, rng, 96, ALL, True, n)
    a, b = Twin(fr, ts, slots, L, st, n), Twin(fr, ts, slots, L, st, n)
    K = A.TIMER_MAX_SLOTS   # no run overflows: the two forms refuse differently (the commit alone, or the arm after it)
    fr.resident_timers(a.h, K)
    fr.resident_timers(b.h, K)
    timings = random_timings(rng, ts, slots, p=0.9)
    for t in timings.values():   # short delays, so that timers fire during the loop
        for s, (c, d) in t.items():
            t[s] = (c, d % 4)
    put_all(fr, timings)
    armed = fired = 0
    for tick in range(24):
        now = 1000 + tick
        fa, fb = fr.resident_fire(a.h, n, now), fr.resident_fire(b.h, n, now)
        assert {k: v for k, v in fa.items() if k != "fired"} == {k: v for k, v in fb.items() if k != "fired"}
        assert np.array_equal(fa["fired"], fb["fired"])
        fired += fa["n_fired"]
        res = a.tick()
        assert np.array_equal(res, b.tick())
        state = fr.resident_download(a.h, 0, n, L.state_stride)
        ents = entries_for(rng, L, a.topo, state, res, None, n)
        area_b = fr.resident_timers_download(b.h, 0, n, K).view("<u8").copy()
        req = CT.arm_requests(L, a.topo, timings, state, res, None, n, ents, area_b, now, Frontier.TIMER_DTYPE)
        ga = fr.resident_commit(a.h, n, ents, now=now)
        gb = fr.resident_commit(b.h, n, ents)
        fr.resident_timers_arm(b.h, req)
        assert ga["n_armed"] == len(req) and {k: ga[k] for k in gb} == gb
        armed += ga["n_armed"]
        assert np.array_equal(fr.resident_download(a.h, 0, n, L.state_stride), fr.resident_download(b.h, 0, n, L.state_stride))
        assert np.array_equal(fr.resident_timers_download(a.h, 0, n, K), fr.resident_timers_download(b.h, 0, n, K))
    assert armed > 0 and fired > 0


def _story(fr, types, needs, flags=0):
    S = len(types)
    rp = np.zeros(S + 1, np.uint32)
    col = []
    for i in range(S):
        col += needs.get(i, [])
        rp[i + 1] = len(col)
    sf = np.array([t | (flags if t in (A.STEP_WAIT, A.STEP_GATE) else 0) for t in types], np.uint8)
    ts = TopologySet([S], [len(col)], rp, np.array(col, np.uint16), sf, [0],
                     np.zeros(0, dtype=[("step", "<u2"), ("branches", "<u2"), ("allow_first", "<u4")]))
    return int(fr.put_topologies(ts)[0])


@pytest.mark.parametrize("kind", ["sleep", "wait-skip", "gate"])
def test_end_to_end(fr, kind):
    """sleep "1s" -> engram: tick, timed commit at now = 100, Fire(100) fires nothing, Fire(101) writes, and the next tick has
    the engram ready; a wait with onTimeout skip ends Skipped, a gate timeout ends Timeout"""
    from tests.step_timings import step_timing
    ty, with_raw, flags = {"sleep": (A.STEP_SLEEP, '{"duration": "1s"}', 0),
                           "wait-skip": (A.STEP_WAIT, '{"until": "{{ inputs.ready }}", "timeout": "1s", "onTimeout": "skip"}',
                                         A.SF_ON_TIMEOUT_SKIP),
                           "gate": (A.STEP_GATE, '{"timeout": "1s"}', 0)}[kind]
    slot = _story(fr, [ty, A.STEP_ENGRAM], {1: [0]}, flags)
    code, delay = step_timing(ty, with_raw)
    fr.put_timings(slot, [(0, code, delay)])
    L = make_layout(2, 0, A.F_DECISION | A.F_ALL_OUT)
    h = fr.resident_create(L, 1)
    fr.resident_upload(h, 0, pack_state(L, np.array([slot], np.uint32), np.zeros(1, np.uint8), np.zeros((1, 2), np.uint8)))
    fr.resident_timers(h, 2)
    u = unpack_result(L, fr.resident_tick(h, L, 1, NONE_D)[0], 2)
    assert u["ready"][0].tolist() == [True, False]
    got = fr.resident_commit(h, 1, now=100)
    assert (got["n_launched"], got["n_armed"], got["next_deadline"]) == (1, 1, 101)
    assert fr.resident_fire(h, 1, 100)["n_fired"] == 0
    f = fr.resident_fire(h, 1, 101)
    assert (f["n_fired"], f["n_written"], f["next_deadline"]) == (1, 1, A.TIMER_NONE)
    u = unpack_result(L, fr.resident_tick(h, L, 1, NONE_D)[0], 2)
    want = {"sleep": A.PHASE_SUCCEEDED, "wait-skip": A.PHASE_SKIPPED, "gate": A.PHASE_TIMEOUT}[kind]
    assert int(u["phase_out"][0][0]) == want
    if kind == "sleep":
        assert u["ready"][0].tolist() == [False, True]
