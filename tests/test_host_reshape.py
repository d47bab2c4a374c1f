"""bfh_batch_reshape in the C++ host mirror without a device: a mirror grown in place equals a mirror built at the new layout by
the same bfh_* calls, rejections change nothing, and a Story too large before the reshape fits after it."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import host as H
from bobrapet_b200.records import make_layout
from tests import migration as M
from tests import reshape as RS

OUT = A.F_ALL_OUT


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


def _fill(b, r, ps, st, L):
    """the state of run r through the mirror's setters, for the fields layout L has"""
    for i, nm in enumerate(ps.names):
        ph, cd, dc = st["codes"][nm]
        b.set_phase_code(r, i, ph)
        if L.off_cond != A.OFF_NONE:
            b.set_cond(r, i, cd)
        if L.off_decision != A.OFF_NONE:
            b.set_decision(r, i, dc)
    for q, stp in enumerate(ps.par_steps):
        on, kids = st["par"][ps.names[stp]]
        b.register_children(r, q, on)
        if L.off_child != A.OFF_NONE:
            for br, code in enumerate(kids):
                b.set_child_phase(r, q, br, A.PHASE_NAMES[min(code, 13)])


# (steps_max, child nibbles, fields, capacity): old -> new
CASES = [((31, 0, 0, 20), (33, 0, A.F_COND, 20)),
         ((64, 0, OUT, 20), (256, 0, OUT | A.F_DECISION, 40)),
         ((64, 40, A.F_CHILD, 20), (288, 52, A.F_CHILD | A.F_COND | A.F_DECISION | OUT, 41)),
         ((256, 0, A.F_COND, 20), (288, 0, A.F_COND | A.F_OUT_NEEDS_COND, 20)),
         ((40, 0, 0, 20), (544, 60, A.F_CHILD | A.F_COND | A.F_DECISION, 64))]


@pytest.mark.parametrize("old,new", CASES, ids=["%d-%d" % (o[0], n[0]) for o, n in CASES])
def test_reshape_equals_a_mirror_built_at_the_new_layout(old, new):
    rng = np.random.default_rng(old[0] * 1000 + new[0])
    n_par = 2 if old[2] & A.F_CHILD else 0
    steps = [M.random_story(rng, "s%d-" % k, min(old[0], 30), n_par) for k in range(2)]
    stories = [M.story_from_steps(s) for s in steps]
    hs = [_host_story(s) for s in steps]
    assert not old[2] & A.F_CHILD or max(p.child_nibbles() for p in stories) <= old[1]
    big = _host_story(M.random_story(rng, "big-", new[0], 0))
    a, b = H.HostBatch(None, *old), H.HostBatch(None, *new)
    try:
        n = old[3] - 3
        for r in range(n):
            st = M.random_state(rng, stories[r % 2])
            for x in (a, b):
                assert x.add_run(hs[r % 2], 5 + r % 2) == r
                _fill(x, r, stories[r % 2], st, a.L)   # the same calls on both: the fields of the tight layout
        with pytest.raises(A.FrontierError) as e:   # a Story larger than the tight layout
            a.add_run(big, 9)
        assert e.value.status == A.BF_EINVAL
        F = A.Layout.from_buffer_copy(a.L)
        before = a.state().copy()
        a.reshape(*new)
        assert a.L.as_dict() == make_layout(new[0], new[1], new[2]).as_dict()
        assert np.array_equal(a.state(), b.state())
        assert np.array_equal(a.state(), RS.reshape_state(F, a.L, before, n))
        assert np.array_equal(a.result(), b.result())
        # the mirror keeps working at the new layout: codes of the added fields, runs past the old capacity, a larger Story
        for r in range(0, n, 3):
            for x in (a, b):
                x.set_phase_code(r, 1, 3)
                if x.L.off_decision != A.OFF_NONE:
                    x.set_decision(r, 2, A.DEC_SUCCEED)
        for x in (a, b):
            while x.size() < new[3] - 1:
                x.add_run(hs[x.size() % 2], 5)
            assert x.add_run(big, 9) == new[3] - 1
            x.set_phase_code(new[3] - 1, new[0] - 1, 2)
        assert np.array_equal(a.state(), b.state())
    finally:
        a.close()
        b.close()


def test_reshape_rejections_leave_the_mirror_unchanged():
    E, PA = A.STEP_ENGRAM, A.STEP_PARALLEL
    hs = _host_story([dict(name=nm, group=0, type=t, needs=[], branches=br)
                      for nm, t, br in [("a", E, 0), ("p", PA, 3), ("b", E, 0), ("q", PA, 5)]])
    child, fields = 16, A.F_CHILD | A.F_COND | A.F_OUT_SKIP_DEP   # descs at nibbles 0 and 8: 13 nibbles
    b = H.HostBatch(None, 64, child, fields, 8)
    try:
        for r in range(5):
            b.add_run(hs, 3)
            b.set_phase_code(r, r % 4, 3)
            b.set_cond(r, (r + 1) % 4, 2)
            b.set_child_phase(r, 1, r % 5, "Running")
        before, layout = b.state().copy(), b.L.as_dict()
        for bad in [(64, child, fields, 7),                          # fewer runs
                    (32, child, fields, 8),                          # fewer steps
                    (64, child - 1, fields, 8),                      # a smaller child area
                    (64, child, fields & ~A.F_COND, 8),              # a dropped input field
                    (64, child, fields & ~A.F_OUT_SKIP_DEP, 8),      # a dropped output field
                    (64, 0, fields & ~A.F_CHILD, 8),                 # the child area dropped
                    (A.MAX_STEPS + 1, child, fields, 8)]:            # not a layout
            with pytest.raises(A.FrontierError) as e:
                b.reshape(*bad)
            assert e.value.status == A.BF_EINVAL, bad
            assert b.L.as_dict() == layout and b.size() == 5
            assert np.array_equal(b.state(), before)
        b.reshape(64, child, fields, 8)   # the same shape is a valid growth that changes nothing
        assert b.L.as_dict() == layout and np.array_equal(b.state(), before)
    finally:
        b.close()
