"""Random sequences of resident-batch calls that mix bf_resident_narrow and bf_resident_extent with reshapes, deltas, uploads,
migrations, redrives, retirements and every tick kind, two batches on one ctx laid out wider than their Stories, checked after
every call against the host model (tests/resident_model.py, extended by the narrow in tests/narrowing.py): the device state,
every tick output and `full` flag, every extent, and which calls are refused."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests.narrowing import NarrowRig
from tests.seqrig import NONE, layout_for, story_pool
from tests.test_gpu_resident_sequences import N_BASE, Driver, assert_schedules_compared, close_with_schedules

pytestmark = pytest.mark.gpu

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT
# shape: (steps lo, hi, parallel steps per Story, layout fields, runs of batch A, runs of batch B, layout steps_max, spare child
# nibbles, cond / decision planes left all PASS / PENDING by the uploads)
SHAPES = {"w256": (20, 60, 2, COND | DEC | OUT | CHILD, 700, 200, 256, 16, False),
          "planes": (10, 30, 0, COND | DEC | OUT, 700, 200, 96, 0, True),
          "wide": (513, 600, 1, COND | OUT | CHILD, 300, 100, 800, 8, False)}
SEEDS = 4


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


class NarrowDriver(Driver):
    """the batcher of test_gpu_resident_sequences.py, whose batches are laid out wider than their Stories, and which now and then
    queries the extent and narrows"""

    def __init__(self, fr, rng, shape, seed):
        lo, hi, n_par, fields, nA, nB, s_wide, spare, self.zero_planes = SHAPES[shape]
        self.rng, self.fields, self.grow = rng, fields, None
        pool = story_pool(rng, lo, hi, n_par, N_BASE)
        self.rig = rig = NarrowRig(fr, pool, "narrow seed %d shape %s" % (seed, shape))
        self.base = [rig.put(k) for k in range(N_BASE)]
        self.edited, self.migrated = set(), set()
        L0 = layout_for(pool[:N_BASE], fields)
        L = make_layout(s_wide, L0.child_nibbles + spare if fields & CHILD else 0, fields)
        self.bs = []
        for n in (nA, nB):
            b = rig.create(L, n + n // 4)
            rig.upload(b, 0, self._fresh(L, n))
            self.bs.append([b, n])
        self.flags, self.max_iter, self.accepted = 0, 0, 0
        self.followed = set()

    def _fresh(self, L, n):
        recs = super()._fresh(L, n)
        if self.zero_planes:
            for off in (L.off_cond, L.off_decision):
                if off != A.OFF_NONE:
                    recs[:, off:off + 8 * L.words] = 0
        return recs

    def narrow(self):
        rng, rig = self.rng, self.rig
        bi = 0 if rng.random() < 0.75 else 1
        b, n = self.bs[bi]
        L = b.L
        nr = n if rng.random() < 0.8 else int(rng.integers(0, b.cap + 1))
        e = rig.extent(b, nr)
        if rng.random() < 0.7:   # a layout the extent allows, with some headroom and the droppable fields dropped now and then
            S = min(L.steps_max, e["steps_max"] + int(rng.choice([0, 0, 1, 7, 32])))
            f = L.fields
            for bit in (COND, DEC, CHILD, A.F_OUT_FAIL, A.F_OUT_NEEDS_COND, A.F_OUT_SKIP_DEP, A.F_OUT_PHASE):
                if f & bit and not e["fields"] & bit and rng.random() < 0.3:
                    f &= ~bit
            child = min(L.child_nibbles, e["child_nibbles"] + int(rng.choice([0, 0, 8]))) if f & CHILD else 0
        else:                    # anything no larger than the layout: often below the extent
            S = int(rng.integers(1, L.steps_max + 1))
            f = L.fields & ~int(rng.choice([0, 0, COND, DEC, CHILD, OUT]))
            child = int(rng.integers(0, L.child_nibbles + 1)) if f & CHILD else 0
        self.accepted += rig.narrow(b, make_layout(S, child, f), nr)
        self.follow(bi, "narrow")

    def step(self):
        u = self.rng.random()
        if u < 0.12:
            self.narrow()
        elif u < 0.15:
            b, n = self.bs[0]
            self.rig.extent(b, int(self.rng.integers(0, b.cap + 1)))
        else:
            super().step()


@pytest.mark.parametrize("seed", range(SEEDS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_random_sequences_with_narrows(fr, shape, seed):
    rng = np.random.default_rng(9500 + 100 * list(SHAPES).index(shape) + seed)
    dr = NarrowDriver(fr, rng, shape, seed)
    try:
        for b, n in dr.bs:
            dr.rig.extent(b, n)   # before the first tick: no result record counts
            dr.rig.tick(b, "touched", n)
        for _ in range(int(rng.integers(70, 111))):
            dr.step()
        for b, n in dr.bs:   # a closing tick of each kind over the batch as it ends
            dr.rig.tick(b, "touched", n, NONE, dr.flags, dr.max_iter)
            dr.rig.tick(b, "changed", n, NONE, dr.flags, dr.max_iter)
        close_with_schedules(dr)
    finally:
        dr.rig.destroy()
    assert dr.accepted > 0, "no narrow was accepted"
    assert_schedules_compared(dr)
