"""Random sequences of resident-batch calls over two batches of one ctx laid out differently (width classes), mixing
bf_resident_transfer in both directions with uploads, deltas, every tick kind, migrate, redrive, reshape, retire, narrow, extent and
slot churn, checked after every call against the host model (tests/resident_model.py, extended by the narrow in
tests/narrowing.py and the transfer in tests/transfer.py): the device state, every tick output and `full` flag, every move and
refusal."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests.seqrig import NONE, layout_for, random_records, story_pool
from tests.test_gpu_narrow_sequences import NarrowDriver
from tests.test_gpu_resident_sequences import N_BASE, assert_schedules_compared, close_with_schedules
from tests.transfer import TransferRig, fits, run_extent

pytestmark = pytest.mark.gpu

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT
# shape: (steps lo, hi, parallel steps per Story, fields of A, of B, runs of A, of B, steps_max of A, of B, cond / decision
# planes left all PASS / PENDING by the uploads).  Every steps_max holds the spare Stories (up to 40 steps) that slot churn
# re-points runs at.
SHAPES = {"64-256": (20, 60, 2, CHILD | A.F_OUT_SKIP_DEP, COND | DEC | CHILD | OUT, 700, 200, 64, 256, False),
          "planes": (10, 30, 0, COND | DEC | OUT, A.F_OUT_FAIL, 600, 300, 96, 64, True),
          "wide": (40, 60, 1, COND | CHILD | OUT, COND | CHILD, 300, 200, 800, 64, True)}
SEEDS = 4


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


class TransferDriver(NarrowDriver):
    """the batcher of test_gpu_narrow_sequences.py with two width classes: batch A and batch B differ in steps_max and fields,
    and runs move between them now and then"""

    def __init__(self, fr, rng, shape, seed):
        lo, hi, n_par, fA, fB, nA, nB, sA, sB, self.zero_planes = SHAPES[shape]
        self.rng, self.fields, self.grow = rng, fA, None
        pool = story_pool(rng, lo, hi, n_par, N_BASE)
        self.rig = rig = TransferRig(fr, pool, "transfer seed %d shape %s" % (seed, shape))
        # the base Stories, and a spare one that is never migrated or dropped, so that the ctx always holds a topology
        self.base = [rig.put(k) for k in range(N_BASE)] + [rig.put(len(pool) - 1)]
        self.edited, self.migrated = set(), set()
        child = layout_for(pool, CHILD).child_nibbles
        self.bs = []
        for n, s, f in ((nA, sA, fA), (nB, sB, fB)):
            L = make_layout(s, child + 8 if f & CHILD else 0, f)
            b = rig.create(L, n + n // 2)
            rig.upload(b, 0, self._fresh(L, n))
            self.bs.append([b, n])
        self.flags, self.max_iter, self.accepted, self.moved = 0, 0, 0, 0
        self.followed = set()

    def _fresh(self, L, n):
        """new runs on the live Stories the layout holds (a narrow may have taken a batch below some of them); runs on a slot no
        put created (dead) when it holds none"""
        reg = self.rig.reg
        live = [s for s in reg.live if (s in self.base or s in self.edited) and reg.story(s).S <= L.steps_max and
                (L.off_child == A.OFF_NONE or reg.story(s).child_nibbles() <= L.child_nibbles)]
        if not live:
            recs = np.zeros((n, L.state_stride), np.uint8)
            recs[:, 0:2] = 0xFF
            return recs
        slots = [int(self.rng.choice(live)) for _ in range(n)]
        recs = random_records(self.rng, L, [reg.story(s) for s in slots], slots)
        if self.zero_planes:
            for off in (L.off_cond, L.off_decision):
                if off != A.OFF_NONE:
                    recs[:, off:off + 8 * L.words] = 0
        return recs

    def transfer(self):
        rng, rig = self.rng, self.rig
        i = 0 if rng.random() < 0.5 else 1
        (a, na), (b, nb) = self.bs[i], self.bs[1 - i]
        if not na:
            return
        k = int(rng.integers(1, min(na, 60) + 1))
        runs = rng.choice(na, size=k, replace=False).astype(np.uint32)
        if rng.random() < 0.85:   # mostly runs the destination holds (deltas put codes anywhere in the source's width)
            runs = np.array([r for r in rng.permutation(na)[:200].tolist() if fits(run_extent(a, r, na, b.L), b.L)][:k], np.uint32)
            if not len(runs):
                return
        if rng.random() < 0.05:
            runs = np.concatenate([runs, runs[:1]])   # twice: refused
        if b.cap < nb + len(runs) and rng.random() < 0.7:   # the batcher reshapes the destination first
            rig.reshape(b, b.L, nb + len(runs) + 8)
        out = rig.transfer(a, b, na, nb, runs)
        if out is not None:
            self.bs[i][1], self.bs[1 - i][1] = out["src_n_runs"], out["dst_n_runs"]
            self.moved += len(runs)
        self.follow(1 - i, "transfer")

    def step(self):
        if self.rng.random() < 0.15:
            self.transfer()
        else:
            super().step()


@pytest.mark.parametrize("seed", range(SEEDS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_random_sequences_with_transfers(fr, shape, seed):
    rng = np.random.default_rng(9700 + 100 * list(SHAPES).index(shape) + seed)
    dr = TransferDriver(fr, rng, shape, seed)
    try:
        for b, n in dr.bs:
            dr.rig.tick(b, "touched", n)
        for _ in range(int(rng.integers(70, 111))):
            dr.step()
        for b, n in dr.bs:   # a closing tick of each kind over the batch as it ends
            dr.rig.tick(b, "touched", n, NONE, dr.flags, dr.max_iter)
            dr.rig.tick(b, "changed", n, NONE, dr.flags, dr.max_iter)
        close_with_schedules(dr)
    finally:
        dr.rig.destroy()
    assert dr.moved > 0, "no transfer was accepted"
    assert_schedules_compared(dr)
