"""bfh_batch_retire in the C++ host mirror without a device: a retired mirror equals a mirror built by adding only the survivors,
in their new order, by the same bfh_* calls; the moves follow the rule of tests/retire.py; rejections change nothing."""
import ctypes as C

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import host as H
from tests import migration as M
from tests import retire as RT
from tests.test_host_reshape import _fill, _host_story

FIELDS = A.F_COND | A.F_DECISION | A.F_CHILD | A.F_ALL_OUT


def _runs(rng, n, share):
    """indices to retire out of [0, n) for a named share"""
    if share == "none":
        return np.zeros(0, np.uint32)
    if share == "one":
        return np.array([int(rng.integers(0, n))], np.uint32)
    if share == "tail":
        return np.arange(n - n // 5, n, dtype=np.uint32)
    if share == "head":
        return np.arange(0, n // 4, dtype=np.uint32)
    if share == "all":
        return rng.permutation(n).astype(np.uint32)
    return rng.choice(n, size=max(1, int(n * float(share))), replace=False).astype(np.uint32)   # scattered, any order


SHARES = ["none", "one", "tail", "head", "all", "0.1", "0.5", "0.9"]


@pytest.mark.parametrize("cap_mode", ["keep", "m", "between"])
@pytest.mark.parametrize("share", SHARES)
def test_retire_equals_a_mirror_of_the_survivors(share, cap_mode):
    rng = np.random.default_rng(SHARES.index(share) * 10 + ["keep", "m", "between"].index(cap_mode))
    steps = [M.random_story(rng, "s%d-" % k, 30, 2) for k in range(3)]
    stories = [M.story_from_steps(s) for s in steps]
    hs = [_host_story(s) for s in steps]
    child = max(p.child_nibbles() for p in stories)
    n, cap = 57, 64
    story = rng.integers(0, 3, n)
    states = [M.random_state(rng, stories[s]) for s in story]
    a = H.HostBatch(None, 32, child, FIELDS, cap)
    try:
        for r in range(n):
            assert a.add_run(hs[story[r]], 7 + story[r]) == r
            _fill(a, r, stories[story[r]], states[r], a.L)
        runs = _runs(rng, n, share)
        m, src, dst = RT.moves(n, runs)
        capacity = {"keep": 0, "m": m, "between": (m + cap + 1) // 2}[cap_mode]   # 0 keeps the capacity (also when m == 0)
        mf, mt = a.retire(runs, capacity)
        assert np.array_equal(mf, src) and np.array_equal(mt, dst)
        assert a.size() == m
        b = H.HostBatch(None, 32, child, FIELDS, capacity or cap)
        try:
            for j, r in enumerate(RT.order(n, runs)):
                assert b.add_run(hs[story[r]], 7 + story[r]) == j
                _fill(b, j, stories[story[r]], states[r], b.L)
            assert np.array_equal(a.state(), b.state())
            assert np.array_equal(a.result(), b.result())
            # both keep working alike: runs added into the vacated indices, setters on moved runs
            for x in (a, b):
                while x.size() < (capacity or cap):
                    x.add_run(hs[x.size() % 3], 7 + x.size() % 3)
                for r in list(dst[:3]) + [x.size() - 1]:
                    x.set_phase_code(int(r), 1, 3)
            assert np.array_equal(a.state(), b.state())
            with pytest.raises(A.FrontierError):   # the capacity is what the call left
                a.add_run(hs[0], 7)
        finally:
            b.close()
    finally:
        a.close()


def test_retire_rejections_leave_the_mirror_unchanged():
    rng = np.random.default_rng(5)
    steps = M.random_story(rng, "r-", 20, 1)
    ps, hs = M.story_from_steps(steps), _host_story(steps)
    b = H.HostBatch(None, 32, ps.child_nibbles(), FIELDS, 16)
    try:
        for r in range(10):
            b.add_run(hs, 3)
            _fill(b, r, ps, M.random_state(rng, ps), b.L)
        before = b.state().copy()
        for runs, cap in [([10], 0),          # not a run
                          ([3, 3], 0),        # twice
                          ([1, 2], 7),        # a capacity below the runs that stay
                          ([1, 2], 17),       # a capacity above the current one
                          (list(range(11)), 0)]:
            with pytest.raises(A.FrontierError) as e:
                b.retire(np.array(runs, np.uint32), cap)
            assert e.value.status == A.BF_EINVAL, (runs, cap)
            assert b.size() == 10 and np.array_equal(b.state(), before)
        lib = H.lib()
        assert lib.bfh_batch_retire(b._p, None, 2, 0, None, None) == A.BF_EINVAL   # null runs
        assert lib.bfh_batch_retire(None, None, 0, 0, None, None) == A.BF_EINVAL
        assert b.size() == 10 and np.array_equal(b.state(), before)
        mf, mt = b.retire(np.zeros(0, np.uint32))   # a no-op
        assert mf.size == 0 and mt.size == 0
        assert b.size() == 10 and np.array_equal(b.state(), before)
        # the valid call after all of them; moves_from / moves_to may be NULL
        runs = (C.c_uint32 * 2)(0, 4)
        assert lib.bfh_batch_retire(b._p, runs, 2, 0, None, None) == 2
        assert b.size() == 8
        assert np.array_equal(b.state(), RT.retire_records(before, 10, [0, 4], 8))
    finally:
        b.close()


@pytest.mark.parametrize("seed", range(40))
def test_moves_follow_the_rule(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(1, 200))
    runs = rng.choice(n, size=int(rng.integers(0, n + 1)), replace=False)
    m, src, dst = RT.moves(n, runs)
    # the rule's properties: at most len(runs) moves, targets below m and retired, sources at or above m and live, both ascending
    gone = np.zeros(n, bool)
    gone[runs] = True
    assert len(src) <= len(runs) and np.all(dst < m) and np.all(gone[dst]) and np.all(src >= m) and not gone[src].any()
    assert np.all(np.diff(dst.astype(np.int64)) > 0) and np.all(np.diff(src.astype(np.int64)) > 0)
    assert sorted(RT.order(n, runs).tolist()) == sorted(set(range(n)) - set(runs.tolist()))
    # the mirror computes the same moves
    steps = M.random_story(rng, "x-", 5, 0)
    hs = _host_story(steps)
    b = H.HostBatch(None, 8, 0, 0, n)
    try:
        for r in range(n):
            b.add_run(hs, r % 5)
        slots = np.ascontiguousarray(b.state()[:, 0:4]).view("<u4").reshape(n).copy()
        mf, mt = b.retire(runs.astype(np.uint32))
        assert np.array_equal(mf, src) and np.array_equal(mt, dst)
        kept = np.ascontiguousarray(b.state()[:, 0:4]).view("<u4").reshape(m)
        assert np.array_equal(kept, slots[RT.order(n, runs)])
    finally:
        b.close()
