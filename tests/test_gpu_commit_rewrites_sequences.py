"""Rewriting tick commits (bf_resident_commit_rewrites) inside the random sequences of tests/test_gpu_resident_sequences.py: deltas,
uploads, every tick kind, migrations, redrives, reshapes, retirements, slot churn and schedules, two batches on one ctx, with a
rewriting commit drawn among them.  The commit follows a single-pass touched tick over the batch (the tick the call needs) and is
checked against tests/commit_rewrites.py over the model's records and result records: the device state (Rig.sync), the counts,
n_rewritten, the journal and its runs.  The commit's written runs are touched in the model, so the next touched tick (which the
rig checks against the model: its listed runs, heads and events) evaluates exactly them.  This is where the precondition of the
call is exercised: a result record left by an earlier tick, across moves, re-lays and slot changes, carries BF_SUM_PHASE_CHANGED
for every run whose stages rewrite."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from tests import commit as M
from tests import commit_rewrites as CR
from tests import resync as RS
from tests.seqrig import NONE
from tests.test_gpu_commit import entries_for
from tests.test_gpu_resident_sequences import OPS, SHAPES, Driver

pytestmark = pytest.mark.gpu


class _Topo:
    """tests/commit.py:Topologies of the registry's live slots"""

    def __init__(self, rig):
        self.by_slot = {}
        for slot, k in rig.reg.live.items():
            self.by_slot.update(M.Topologies(rig.ts1[k], [slot]).by_slot)


def _post(rig, L, rows):
    """tests/resync.py:post_phases of the rows over the registry's live slots"""
    out = [None] * len(rows)
    for slot, k in rig.reg.live.items():
        for i, p in enumerate(RS.post_phases(L, RS.Topos(rig.ts1[k], [slot]), rows)):
            if p is not None:
                out[i] = p
    return out


def rewriting_commit(rig, rng, b, n, counter):
    """a single-pass touched tick over [0, n) of b, then a rewriting commit checked against the model"""
    if n == 0:
        return
    rig.tick(b, "touched", n, NONE, 0, 0)
    h, L = rig.handles[b], b.L
    before = b.state.copy()
    res = b.cur[:n].copy()
    topo = _Topo(rig)
    ents = entries_for(rng, L, topo, before, res, None, n)
    want = before.copy()
    rc, _, _, counts, touched, n_rw, masked = CR.commit(L, topo, None, want, res, None, n, ents, post=_post(rig, L, list(before[:n])))
    rig.check(rc == 0, "the model refused the commit")
    rig.log.append("commit rewrites b%d n %d entries %d" % (h, n, len(ents)))
    got = rig.fr.resident_commit(h, n, ents, journal_cap=n * (32 * L.words + 64), rewrites=True)
    rig.check({k: got[k] for k in M.COUNT_KEYS} == counts and got["n_rewritten"] == n_rw,
              "counts %s, want %s / %d" % (got, counts, n_rw))
    items, runs = CR.journal(L, before, want, n, masked)
    from tests.commit_journal import as_tuples
    rig.check(as_tuples(got["items"]) == items and got["runs"].tolist() == runs == sorted(touched), "journal differs from the model")
    if touched:   # as a delta: the written runs are touched, the snapshot and the tick end
        b._end_snapshot()
        b.touched |= touched
        b.state[:] = want
        b.reg.last = None
    rig.sync()
    rig.tick(b, "touched", n, NONE, 0, 0)   # lists exactly the runs whose result changed, per the model
    counter["commits"] += 1
    counter["rewritten"] += n_rw


class CommitDriver(Driver):
    def __init__(self, *a):
        super().__init__(*a)
        self.counter = {"commits": 0, "rewritten": 0}

    def step(self):
        if self.rng.random() < 0.15:
            bi = 0 if self.rng.random() < 0.75 else 1
            b, n = self.bs[bi]
            rewriting_commit(self.rig, self.rng, b, n, self.counter)
        else:
            super().step()


@pytest.mark.parametrize("seed", range(2))
@pytest.mark.parametrize("shape", ["cfg4", "parallel", "wide", "grow"])
def test_rewriting_commits_in_random_sequences(fr, shape, seed):
    rng = np.random.default_rng(7100 + 100 * list(SHAPES).index(shape) + seed)
    dr = CommitDriver(fr, rng, shape, seed)
    try:
        for b, n in dr.bs:
            dr.rig.tick(b, "touched", n)
        for _ in range(int(rng.integers(60, 101))):
            dr.step()
        for b, n in dr.bs:
            rewriting_commit(dr.rig, rng, b, n, dr.counter)
    finally:
        dr.rig.destroy()
    assert dr.counter["commits"] > 0 and dr.counter["rewritten"] > 0


@pytest.fixture
def fr():
    from bobrapet_b200 import Frontier
    f = Frontier(0)
    yield f
    f.close()


assert "retire" in OPS and "migrate" in OPS and "redrive" in OPS and "reshape" in OPS
