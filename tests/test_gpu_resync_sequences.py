"""Random resyncs interleaved with the resident-batch calls of tests/test_gpu_resident_sequences.py (deltas, uploads, ticks of every
kind, touched ticks, migrations, redrives, reshapes, retirements, slot drops and reuses, schedules), two batches on one ctx.  Each
resync goes to the device and to the host models: tests/resync.py for its items and its repair, tests/resident_model.py for the
touch bookkeeping it leaves (written runs touched as by a delta, slot-drifted runs as by a migrate).  Every later call is compared
as the driver compares it: the device state after every call, every tick's lists and `full` flag, every accepted schedule."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from tests import resync as M
from tests.packing import topology_set
from tests.test_gpu_resident_sequences import SHAPES, Driver, assert_schedules_compared, close_with_schedules, fr  # noqa: F401
from tests.seqrig import NONE, random_records

pytestmark = pytest.mark.gpu

F = A.resync_field
FIELD_SETS = [A.RESYNC_ALL_FIELDS, F(A.DELTA_PHASE) | F(A.DELTA_RUN_FLAGS),
              F(A.DELTA_COND) | F(A.DELTA_DECISION) | F(A.DELTA_CHILD) | F(A.DELTA_REGISTERED)]


def _topos(reg):
    """the live slots of the ctx as the resync model takes them"""
    slots = sorted(reg.live)
    return M.Topos(topology_set([reg.stories[reg.live[s]] for s in slots]), slots)


def _perturbed(rng, reg, L, recs):
    """the records with a few codes changed: a phase, cond or decision bit, a child byte, the flags byte, a registered bit, or a
    live slot whose Story fits the layout (as the drivers' slot deltas draw them)"""
    out = recs.copy()
    W = L.words
    fits = [s for s, k in reg.live.items() if reg.stories[k].S <= L.steps_max and
            (L.off_child == A.OFF_NONE or reg.stories[k].child_nibbles() <= L.child_nibbles)]
    for r in rng.choice(out.shape[0], size=min(out.shape[0], int(rng.integers(0, 6))), replace=False):
        f = int(rng.integers(0, 7))
        if f == A.DELTA_COND and L.off_cond != A.OFF_NONE:
            out[r][L.off_cond + int(rng.integers(0, 8 * W))] ^= 1 << int(rng.integers(0, 8))
        elif f == A.DELTA_DECISION and L.off_decision != A.OFF_NONE:
            out[r][L.off_decision + int(rng.integers(0, 8 * W))] ^= 1 << int(rng.integers(0, 8))
        elif f == A.DELTA_CHILD and L.off_child != A.OFF_NONE and L.child_nibbles:
            out[r][L.off_child + int(rng.integers(0, (L.child_nibbles + 1) // 2))] ^= int(rng.integers(1, 256))
        elif f == A.DELTA_RUN_FLAGS:
            out[r][4] ^= 1 << int(rng.integers(0, 3))
        elif f == A.DELTA_REGISTERED:
            out[r][8 + int(rng.integers(0, 8))] ^= 1 << int(rng.integers(0, 8))
        elif f == A.DELTA_TOPO_SLOT and fits:
            out[r][:4] = np.frombuffer(np.uint32(int(rng.choice(fits))).tobytes(), np.uint8)
        else:
            out[r][L.off_phase + int(rng.integers(0, 16 * W))] ^= 1 << int(rng.integers(0, 8))
    return out


class ResyncDriver(Driver):
    def _fresh(self, L, n):
        """new runs on the base or edited Stories that fit L: after one batch grew, an edited Story may fit it and not the other"""
        reg = self.rig.reg
        live = [s for s in reg.live if (s in self.base or s in self.edited) and reg.story(s).S <= L.steps_max and
                (L.off_child == A.OFF_NONE or reg.story(s).child_nibbles() <= L.child_nibbles)]
        slots = [int(self.rng.choice(live)) for _ in range(n)]
        return random_records(self.rng, L, [reg.story(s) for s in slots], slots)

    def resync(self):
        rng, rig = self.rng, self.rig
        bi = 0 if rng.random() < 0.75 else 1
        b, n = self.bs[bi]
        h = rig.handles[b]
        runs = None if rng.random() < 0.4 else np.flatnonzero(rng.random(n) < rng.random()).astype(np.uint32)
        listed = np.arange(n, dtype=np.uint32) if runs is None else runs
        recs = _perturbed(rng, rig.reg, b.L, b.state[listed])
        fields = int(rng.choice(FIELD_SETS))
        check = rng.random() < 0.3
        rig.log.append("resync b%d %d runs fields %#x%s" % (h, listed.size, fields, " check" if check else ""))
        topos = _topos(rig.reg)
        items, drifted, state, _ = M.resync(b.L, topos, b.state, recs, n, runs=runs, fields=fields, check=check)
        got = rig.fr.resident_resync(h, n, recs, runs=runs, fields=fields, check=check, items_cap=max(items.size, 1))
        rig.check(got["items"].tobytes() == items.tobytes() and got["n_items"] == items.size, "resync items differ")
        rig.check(got["drifted"].tolist() == drifted.tolist(), "resync drifted runs differ")
        rig.check(got["n_written"] == (0 if check else drifted.size), "resync n_written")
        if not check and drifted.size:   # the model's bookkeeping of what the device wrote
            b._end_snapshot()
            b.state[:] = state
            slot = set(M.slot_drifted(items).tolist())
            b.touched |= set(drifted.tolist())
            b.must |= slot
        rig.sync()
        self.follow(bi, "resync")

    def step(self):
        if self.rng.random() < 0.25:
            self.resync()
        else:
            super().step()


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("shape", ["cfg4", "parallel", "cfg3"])
def test_random_resync_sequences(fr, shape, seed):  # noqa: F811
    rng = np.random.default_rng(7700 + 100 * list(SHAPES).index(shape) + seed)
    dr = ResyncDriver(fr, rng, shape, seed)
    try:
        for b, n in dr.bs:
            dr.rig.tick(b, "touched", n)
        for _ in range(int(rng.integers(60, 101))):
            dr.step()
        for b, n in dr.bs:
            dr.rig.tick(b, "touched", n, NONE, dr.flags, dr.max_iter)
            dr.rig.tick(b, "changed", n, NONE, dr.flags, dr.max_iter)
        close_with_schedules(dr)
    finally:
        dr.rig.destroy()
    assert_schedules_compared(dr)
    assert "resync" in dr.followed
