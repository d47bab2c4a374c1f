"""The limiter reference itself, on the CPU: the numpy schedule (tests/schedref.schedule_fast) equals the loop definition
(oracle.limiters.schedule_packed) on random and extreme inputs; both oracle levels wrap the aged priority to int32 as Go
does; and the edges include/bobrafrontier.h pins (keys out of range, the low 4 bits of run_phase) hold in the definition."""
import numpy as np
import pytest

from oracle import limiters as LM
from tests import schedref as SR

INT32_MIN, INT32_MAX = SR.INT32_MIN, SR.INT32_MAX


def _both(args, **kw):
    a = LM.schedule_packed(*args, **kw)
    b = SR.schedule_fast(*args, **kw)
    for i, (x, y) in enumerate(zip(a, b)):
        if isinstance(x, np.ndarray):
            assert np.array_equal(np.asarray(x, np.int64), np.asarray(y, np.int64)), "output %d differs" % i
        else:
            assert int(x) == int(y), "output %d: %d != %d" % (i, x, y)
    return a


def _random_args(rng, n, W, ns, nq, oor=0.1):
    sched = SR.random_sched(rng, n, ns, nq, out_of_range=oor)
    t = SR.random_tables(rng, ns, nq, n, maxprio_base=bool(rng.integers(0, 2)))
    ready = rng.integers(0, 2**32, size=(n, W), dtype=np.uint64).astype(np.uint32)
    ready &= np.where(rng.random((n, W)) < 0.3, np.uint32(0), np.uint32(0xFFFFFFFF))   # empty words and empty rows
    ready[rng.random(n) < 0.1] = 0
    run_running = rng.choice([0, 0, 1, 2, 7, 40], size=n).astype(np.uint32)
    run_demand = (rng.random(n) < 0.4).astype(np.uint32)
    args = (run_running, run_demand, sched, ready, t["story_limit"], t["story_running_base"], t["queue_limit"], t["queue_aging_s"],
            t["queue_running_base"], t["global_limit"], t["global_running_base"])
    return args, t.get("queue_max_priority_base")


@pytest.mark.parametrize("seed", range(12))
def test_fast_equals_loop(seed):
    rng = np.random.default_rng(900 + seed)
    n = [300, 1, 0, 257, 500, 64, 1000, 33, 400, 200, 128, 700][seed]
    W = [1, 32, 3, 8, 2, 32, 4, 1, 16, 5, 32, 2][seed]
    ns, nq = [(5, 3), (1, 1), (0, 0), (40, 7), (0, 2), (3, 0), (100, 30), (2, 2), (9, 1), (1, 9), (6, 6), (300, 60)][seed]
    args, mb = _random_args(rng, n, W, ns, nq)
    _both(args, queue_maxprio_base=mb)


@pytest.mark.parametrize("seed", range(6))
def test_fast_equals_loop_partial_scheduling_cuts(seed):
    """global and queue limits a few slots above the running totals: many runs keep part of their ready set through either
    limit, and gslots == qslots ties (reason GLOBAL) occur beside both strict orders"""
    rng = np.random.default_rng(1700 + seed)
    n, W, ns, nq = 400, 3, 4, 6
    sched = np.zeros(n, LM.SCHED_RUN_DTYPE)
    sched["story_key"] = rng.integers(0, ns, size=n)
    sched["queue_key"] = rng.integers(0, nq, size=n)
    sched["queued_elapsed_s"] = LM.NONE_U32
    sched["run_phase"] = 2
    ready = rng.integers(0, 2**32, size=(n, W), dtype=np.uint64).astype(np.uint32)   # ~48 ready steps per run
    running = rng.choice([0, 1, 3, 9], size=n).astype(np.uint32)
    base = (running, np.zeros(n, np.uint32), sched, ready, np.zeros(ns, np.int32), np.zeros(ns, np.uint32))
    qb = rng.integers(0, 30, size=nq).astype(np.uint32)
    *_, qr, gr, _ = _both(base + (np.zeros(nq, np.int32), np.zeros(nq, np.int32), qb, 0, 17))
    seen = set()
    for k_global in (1, 5, 20, 33, 47):
        k_queue = rng.choice([1, 5, 20, 33, 47, 60, 0], size=nq)     # 0: no queue limit
        ql = np.where(k_queue > 0, qr + k_queue, 0).astype(np.int32)
        for gl in (int(gr) + k_global, 0):
            _, _, q_sched, info, *_ = _both(base + (ql, np.zeros(nq, np.int32), qb, gl, 17))
            cnt = SR.popcount(ready)
            kq = k_queue[sched["queue_key"]]
            partial = (info[:, 0] > 0) & (info[:, 2] > 0)
            for r in np.nonzero(partial)[0]:
                tie = gl > 0 and kq[r] == k_global
                seen.add((int(info[r, 3]), "tie" if tie else "strict"))
            # the kept prefix is exactly the smaller limit's slots
            lim = np.minimum(np.where(kq > 0, kq, cnt), k_global if gl > 0 else cnt)
            assert np.array_equal(info[:, 0], np.minimum(cnt, lim))
    assert {(LM.REASON_GLOBAL, "tie"), (LM.REASON_GLOBAL, "strict"), (LM.REASON_QUEUE, "strict")} <= seen, seen


@pytest.mark.parametrize("keep", [0, 1, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025])
def test_truncate_rows_on_word_boundaries(keep):
    rng = np.random.default_rng(keep)
    m = np.full((6, 32), 0xFFFFFFFF, np.uint32)
    m[1] = rng.integers(0, 2**32, size=32, dtype=np.uint64).astype(np.uint32)
    m[2, ::2] = 0
    m[3] = 0
    m[4, :] = 0x80000001
    m[5, 31] = 0x80000000
    got = SR.truncate_rows(m, np.full(6, keep))
    for r in range(6):
        assert np.array_equal(got[r], LM.truncate_mask(m[r], keep)), r
    assert SR.popcount(got[:1])[0] == min(keep, 1024)


def test_aged_priority_wraps_like_go():
    # Go: base + steps in int32 wraps; both oracle levels and the numpy rows must do the same
    now = 10_000_000_000.0
    for base in (INT32_MAX, INT32_MAX - 1, INT32_MAX - 5, INT32_MIN, -1, 0):
        for elapsed in (0, 1, 59, 60, 61, 3600, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE):
            for aging in (-5, 0, 1, 60, INT32_MAX):
                want = base
                if elapsed and aging > 0 and min(elapsed, INT32_MAX) // aging > 0:
                    want = ((base + min(elapsed, INT32_MAX) // aging + 2**31) % 2**32) - 2**31
                assert LM.effective_priority_packed(base, elapsed, aging) == want
                assert LM.effective_priority(base, (now - elapsed) if elapsed else now, aging, now) == want
                assert SR.effective_priority_rows([base], [elapsed], [aging])[0] == want
    assert LM.effective_priority_packed(INT32_MAX, 120, 60) == INT32_MIN + 1
    assert LM.effective_priority_packed(INT32_MAX, 0x7FFFFFFF, 1) == -2
    assert LM.effective_priority_packed(5, LM.NONE_U32, 1) == 5


def test_wrapped_priority_orders_the_queue():
    # run 0 at INT32_MAX has aged past the top: its effective priority wraps to INT32_MIN + 1, so it no longer outranks
    # run 1 (priority 0), and run 1 outranks it instead; the queue maximum is an int32
    sched = np.zeros(2, LM.SCHED_RUN_DTYPE)
    sched["priority"] = [INT32_MAX, 0]
    sched["queued_elapsed_s"] = [120, LM.NONE_U32]
    sched["run_phase"] = 1
    ready = np.array([[1], [1]], np.uint32)
    args = (np.zeros(2, np.uint32), np.zeros(2, np.uint32), sched, ready, np.zeros(1, np.int32), np.zeros(1, np.uint32),
            np.zeros(1, np.int32), np.array([60], np.int32), np.zeros(1, np.uint32), 0, 0)
    launch, _, q_sched, info, _, _, _, mp = _both(args)
    assert mp.dtype == np.int32 and mp[0] == 0
    assert info[:, 3].tolist() == [LM.REASON_PRIORITY, LM.REASON_NONE]
    assert launch[:, 0].tolist() == [0, 1] and q_sched[:, 0].tolist() == [1, 0]


def test_keys_out_of_range_are_counted_nowhere():
    sched = np.zeros(3, LM.SCHED_RUN_DTYPE)
    sched["story_key"] = [0, 1, 0xFFFFFFFF]
    sched["queue_key"] = [0, 1, 0x80000000]
    sched["priority"] = [0, 100, 100]
    sched["run_phase"] = 2
    ready = np.array([[0xF], [0xF], [0xF]], np.uint32)
    running = np.array([3, 5, 7], np.uint32)
    # one story (limit 4) and one queue (limit 5); global limit 100
    args = (running, np.zeros(3, np.uint32), sched, ready, np.array([4], np.int32), np.zeros(1, np.uint32),
            np.array([5], np.int32), np.array([0], np.int32), np.zeros(1, np.uint32), 100, 0)
    launch, q_story, q_sched, info, sr, qr, gr, mp = _both(args)
    assert sr.tolist() == [3] and qr.tolist() == [3] and gr == 15
    assert mp.tolist() == [0]                      # runs 1 and 2 (priority 100) are in no queue: they outrank nobody
    assert info[0].tolist() == [1, 3, 0, 0]        # story limit 4 - 3 running: one slot; queue 5 - 3: enough
    assert info[1].tolist() == [4, 0, 0, 0] and info[2].tolist() == [4, 0, 0, 0]   # no story, queue or priority limit
    # the global limit still applies to them
    args = args[:9] + (16, 0)
    _, _, _, info, *_ = _both(args)
    assert info[0].tolist() == [1, 3, 0, 0] and info[1].tolist() == [1, 0, 3, LM.REASON_GLOBAL] and info[2].tolist() == [1, 0, 3, LM.REASON_GLOBAL]


def test_only_low_four_bits_of_run_phase():
    rng = np.random.default_rng(5)
    args, _ = _random_args(rng, 200, 2, 4, 3, oor=0.0)
    low = args[2].copy()
    low["run_phase"] &= 0xF
    high = args[2].copy()
    high["run_phase"] = (high["run_phase"] & 0xF) | (rng.integers(1, 2**28, size=200, dtype=np.uint64).astype(np.uint32) << 4)
    a = _both(args[:2] + (low,) + args[3:])
    b = _both(args[:2] + (high,) + args[3:])
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_no_tables():
    rng = np.random.default_rng(3)
    args, _ = _random_args(rng, 100, 3, 0, 0, oor=0.0)
    launch, q_story, q_sched, info, sr, qr, gr, mp = _both(args)
    assert sr.size == 0 and qr.size == 0 and mp.size == 0 and not q_story.any()
