"""bfh_batch_narrow without a device: the C++ mirror re-lays its records at a smaller layout when its records, its runs' Stories
and its pending deltas allow it, and every rejection leaves it byte-identical."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import host as H
from tests import migration as M

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


def _fill(b, r, ps, st, cond=True, dec=True, child=True):
    for i, nm in enumerate(ps.names):
        ph, cd, dc = st["codes"][nm]
        b.set_phase_code(r, i, ph)
        if cond:
            b.set_cond(r, i, cd)
        if dec:
            b.set_decision(r, i, dc)
    for q, stp in enumerate(ps.par_steps):
        on, kids = st["par"][ps.names[stp]]
        b.register_children(r, q, on)
        for br, code in enumerate(kids if child else []):
            b.set_child_phase(r, q, br, A.PHASE_NAMES[min(code, 13)])


@pytest.mark.parametrize("cond,dec,child", [(True, True, True), (False, True, True), (True, False, False), (False, False, False)])
def test_narrowed_mirror_equals_one_built_at_the_narrow_layout(cond, dec, child):
    rng = np.random.default_rng(81 + 2 * cond + 4 * dec + child)
    steps = M.random_story(rng, "h-", 26, 2)
    ps = M.story_from_steps(steps)
    hs = _host_story(steps)
    c = ps.child_nibbles()
    keep = (COND if cond else 0) | (DEC if dec else 0) | (CHILD if child else 0)
    n = 40
    wide = H.HostBatch(None, 300, c + 40, COND | DEC | CHILD | OUT, n + 8)
    tight = H.HostBatch(None, 32, c, keep | A.F_OUT_SKIP_DEP, n + 8)
    try:
        states = [M.random_state(rng, ps) for _ in range(n)]
        for x in (wide, tight):
            for r in range(n):
                x.add_run(hs, 7)
                _fill(x, r, ps, states[r], cond, dec, child and c > 0)
        wide.narrow(32, c, keep | A.F_OUT_SKIP_DEP)
        assert wide.L.as_dict() == tight.L.as_dict()
        assert np.array_equal(wide.state(), tight.state()) and np.array_equal(wide.result(), tight.result())
        # the narrowed mirror takes the same calls as the tight one afterwards
        for x in (wide, tight):
            x.set_phase_code(3, 1, A.PHASE_RUNNING)
            x.add_run(hs, 7)
        assert np.array_equal(wide.state(), tight.state())
    finally:
        wide.close()
        tight.close()


def test_narrow_rejections_leave_the_mirror_unchanged():
    rng = np.random.default_rng(91)
    steps = M.random_story(rng, "r-", 40, 2)
    ps = M.story_from_steps(steps)
    assert ps.S > 32
    hs = _host_story(steps)
    c = ps.child_nibbles()
    n = 20
    b = H.HostBatch(None, 64, c + 16, COND | DEC | CHILD | OUT, n)
    try:
        for r in range(n):
            b.add_run(hs, 3)
            _fill(b, r, ps, M.random_state(rng, ps))
        b.set_cond(2, 1, A.COND_SKIP)
        b.set_decision(2, 1, A.DEC_FAIL)
        before = (b.L.as_dict(), b.state().copy(), b.result().copy())
        fields = b.L.fields
        for shape in [(32, c + 16, fields),             # the Story has more than 32 steps
                      (64, c + 16, fields & ~COND),     # a non-PASS cond code
                      (64, c + 16, fields & ~DEC),      # a non-PENDING decision code
                      (128, c + 16, fields),            # grows steps_max
                      (64, c + 24, fields),             # grows the child area
                      (64, c + 16, 0x8000 | fields)]:   # adds a field
            with pytest.raises(A.FrontierError) as e:
                b.narrow(*shape)
            assert e.value.status == A.BF_EINVAL, shape
            assert b.L.as_dict() == before[0]
            assert np.array_equal(b.state(), before[1]) and np.array_equal(b.result(), before[2])
        if c:
            with pytest.raises(A.FrontierError):
                b.narrow(64, c - 8, fields)   # the Story's parallel steps need the child area
        b.narrow(b.L.steps_max, b.L.child_nibbles, fields)   # the same layout: a no-op
        assert np.array_equal(b.state(), before[1])
        b.narrow(ps.S, c, fields & ~A.F_OUT_PHASE)           # output fields may always go
        assert b.L.steps_max == ps.S and b.L.off_phase_out == A.OFF_NONE
    finally:
        b.close()


def test_a_code_or_a_story_above_the_new_width_blocks_the_narrow():
    """a code at the last step blocks a narrow below it; once it is reset the run's Story still does (pending deltas, which only
    resident mode logs, are covered by the GPU tests)"""
    rng = np.random.default_rng(97)
    steps = M.random_story(rng, "p-", 20, 1)
    ps = M.story_from_steps(steps)
    hs = _host_story(steps)
    b = H.HostBatch(None, 64, 0, COND, 4)
    try:
        for r in range(4):
            b.add_run(hs, 1)
        b.set_phase_code(1, ps.S - 1, A.PHASE_SUCCEEDED)
        with pytest.raises(A.FrontierError):
            b.narrow(ps.S - 1, 0, COND)
        b.set_phase_code(1, ps.S - 1, 0)
        with pytest.raises(A.FrontierError):   # the run's Story still has S steps
            b.narrow(ps.S - 1, 0, COND)
        b.narrow(ps.S, 0, COND)
        assert b.L.steps_max == ps.S
    finally:
        b.close()
