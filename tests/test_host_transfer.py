"""bfh_batch_transfer in the C++ host mirror without a device: the destination's records equal a mirror that packed the same codes
at its layout from the start, the source equals bfh_batch_retire of the same runs, and every refusal leaves both mirrors
byte-identical.  (Pending deltas, which only resident mode logs, are covered by test_gpu_transfer.py.)"""
import ctypes as C

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import host as H
from bobrapet_b200.records import make_layout
from tests import migration as M
from tests import retire as RT
from tests.test_host_reshape import _fill, _host_story

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT

# (source steps_max, source fields, destination steps_max, destination fields): narrow -> wide with fields added, wide -> narrow
# with fields dropped, and equal layouts
PAIRS = {"64-to-256": (64, 0, 256, COND | DEC | CHILD | OUT),
         "256-to-1024": (256, COND | CHILD, 1024, COND | DEC | CHILD | A.F_OUT_FAIL),
         "1024-to-64": (1024, COND | DEC | CHILD | OUT, 64, CHILD | A.F_OUT_SKIP_DEP),
         "equal": (128, COND | DEC | CHILD | OUT, 128, COND | DEC | CHILD | OUT)}


def _stories(rng, k, S):
    steps = [M.random_story(rng, "s%d-" % j, S, 2) for j in range(k)]
    return [M.story_from_steps(s) for s in steps], [_host_story(s) for s in steps]


def _filled(L, both, stories, hs, story, states, cap, child):
    b = H.HostBatch(None, L[0], child if L[1] & CHILD else 0, L[1], cap)
    for r, s in enumerate(story):
        assert b.add_run(hs[s], 7 + s) == r
        _fill(b, r, stories[s], states[r], both)
    return b


@pytest.mark.parametrize("share", ["one", "0.3", "all"])
@pytest.mark.parametrize("pair", list(PAIRS))
def test_transfer_equals_packing_at_the_destination_and_retire_at_the_source(pair, share):
    s_src, f_src, s_dst, f_dst = PAIRS[pair]
    rng = np.random.default_rng(list(PAIRS).index(pair) * 10 + ["one", "0.3", "all"].index(share))
    stories, hs = _stories(rng, 3, 30)
    child = max(p.child_nibbles() for p in stories)
    both = make_layout(32, child, f_src & f_dst & (COND | DEC | CHILD))   # the fields both layouts hold codes in
    nS, nD, cap = 40, 9, 64
    story_s, story_d = rng.integers(0, 3, nS), rng.integers(0, 3, nD)
    st_s = [M.random_state(rng, stories[s]) for s in story_s]
    st_d = [M.random_state(rng, stories[s]) for s in story_d]
    runs = {"one": np.array([int(rng.integers(0, nS))]), "0.3": rng.choice(nS, 12, replace=False),
            "all": rng.permutation(nS)}[share].astype(np.uint32)
    src = _filled((s_src, f_src), both, stories, hs, story_s, st_s, cap, child)
    twin = _filled((s_src, f_src), both, stories, hs, story_s, st_s, cap, child)
    dst = _filled((s_dst, f_dst), both, stories, hs, story_d, st_d, cap, child)
    order = list(range(nD)) + [None] * len(runs)
    want = _filled((s_dst, f_dst), both, stories, hs, np.concatenate([story_d, story_s[runs]]),
                   st_d + [st_s[r] for r in runs], cap, child)
    try:
        mf, mt = src.transfer(dst, runs)
        # the source: bfh_batch_retire of the same runs, the same moves, the rule of tests/retire.py
        tf, tt = twin.retire(runs)
        m, wf, wt = RT.moves(nS, runs)
        assert np.array_equal(mf, tf) and np.array_equal(mt, tt) and np.array_equal(mf, wf) and np.array_equal(mt, wt)
        assert src.size() == twin.size() == m
        assert np.array_equal(src.state(), twin.state()) and np.array_equal(src.result(), twin.result())
        # the destination: the arrivals after its own runs, packed as at its layout from the start
        assert dst.size() == nD + len(runs) == len(order)
        assert np.array_equal(dst.state(), want.state()) and np.array_equal(dst.result(), want.result())
        # all three keep taking calls alike: a setter on an arrival, a run added after them
        for x in (dst, want):
            x.set_phase_code(nD, 1, A.PHASE_RUNNING)
            x.add_run(hs[0], 7)
        assert np.array_equal(dst.state(), want.state())
    finally:
        for b in (src, twin, dst, want):
            b.close()


def test_transfer_refusals_leave_both_mirrors_unchanged():
    rng = np.random.default_rng(17)
    wide_steps = M.random_story(rng, "w-", 70, 1)
    narrow_steps = M.random_story(rng, "n-", 20, 1)
    pw, pn = M.story_from_steps(wide_steps), M.story_from_steps(narrow_steps)
    hw, hn = _host_story(wide_steps), _host_story(narrow_steps)
    assert pw.S > 64
    child = max(pw.child_nibbles(), pn.child_nibbles())
    src = H.HostBatch(None, 128, child, COND | DEC | CHILD | OUT, 16)
    dst = H.HostBatch(None, 64, child, CHILD, 8)
    try:
        for r in range(10):
            ps, h = (pw, hw) if r == 4 else (pn, hn)
            src.add_run(h, 3)
            _fill(src, r, ps, M.random_state(rng, ps), make_layout(32, child, CHILD))
        for r in range(5):
            dst.add_run(hn, 3)
        src.set_cond(6, 1, A.COND_SKIP)   # a non-PASS cond code: the destination has no cond planes
        before = [(x.size(), x.state().copy(), x.result().copy()) for x in (src, dst)]

        def same():
            for x, (n, st, res) in zip((src, dst), before):
                assert x.size() == n and np.array_equal(x.state(), st) and np.array_equal(x.result(), res)
        for runs in ([4],            # the run's Story has more steps than the destination holds
                     [1, 6],         # a non-PASS cond code
                     [10],           # not a run
                     [2, 2],         # twice
                     [0, 1, 2, 3]):  # the destination holds 8 runs, 5 are taken
            with pytest.raises(A.FrontierError) as e:
                src.transfer(dst, np.array(runs, np.uint32))
            assert e.value.status == A.BF_EINVAL, runs
            same()
        lib = H.lib()
        assert lib.bfh_batch_transfer(src._p, src._p, (C.c_uint32 * 1)(0), 1, None, None) == A.BF_EINVAL   # to itself
        assert lib.bfh_batch_transfer(src._p, dst._p, None, 2, None, None) == A.BF_EINVAL                  # null runs
        assert lib.bfh_batch_transfer(None, dst._p, None, 0, None, None) == A.BF_EINVAL
        same()
        assert src.transfer(dst, np.zeros(0, np.uint32))[0].size == 0   # a no-op
        same()
        # the valid call after all of them; moves_from / moves_to may be NULL
        assert lib.bfh_batch_transfer(src._p, dst._p, (C.c_uint32 * 3)(0, 1, 9), 3, None, None) == 2
        assert src.size() == 7 and dst.size() == 8
    finally:
        src.close()
        dst.close()
