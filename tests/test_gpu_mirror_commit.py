"""bfh_batch_commit: the C++ host mirror commits a tick on the device (bf_resident_commit_journal) and applies the journal to its
own records.  Random sequences of bfh_run_set_* -> bfh_batch_eval -> more sets -> bfh_batch_commit: after each commit and the
next eval the mirror's records equal the device's download, and bf_resident_resync with BF_RESYNC_CHECK over the mirror's
records reports no drift.  Deltas logged between the eval and the commit win over the commit's writes at their (run, field,
index), on both sides; a refused commit changes neither; outside resident mode the call is refused."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200 import host as H
from tests import commit as CM
from tests import migration as M
from tests.test_gpu_migrate import _host_story
from tests.test_gpu_reshape import _fill

pytestmark = pytest.mark.gpu

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT


@pytest.fixture
def fr():
    """a fresh ctx (the first mirror's resident batch is its handle 0); batches appended to fr.batches close before it, after
    the test's report, so that no array a failure shows points at freed records"""
    f = Frontier(0)
    f.batches = []
    yield f
    for b in f.batches:
        b.close()
    f.close()


def _entries(rng, b, n, types, p_hold=0.05, p_error=0.03):
    """HOLD / ERROR entries on random ready steps and a PHASE entry for every other ready stop step"""
    out = []
    for r in range(n):
        ready = [int(s) for s in b.ready(r)]
        if not ready:
            continue
        named = {}
        if rng.random() < p_error:
            named[int(rng.choice(ready))] = (CM.ERROR, 0)
        elif rng.random() < p_hold:
            named[int(rng.choice(ready))] = (CM.HOLD, 0)
        for s in ready:
            if types[r][s] == A.STEP_STOP and s not in named:
                named[s] = (CM.PHASE, int(rng.integers(A.PHASE_PENDING, A.PHASE_SKIPPED + 1)))
        out += [(r, s, k, c) for s, (k, c) in named.items()]
    return np.array(out, dtype=Frontier.COMMIT_DTYPE) if out else np.zeros(0, Frontier.COMMIT_DTYPE)


def _codes(c):
    return c if c < 14 else 1


@pytest.mark.parametrize("S,fields,n_par,n,seed", [(40, ALL | A.F_CHILD, 3, 500, 1), (120, A.F_OUT_FAIL, 0, 300, 2),
                                                   (300, A.F_ALL_OUT | A.F_CHILD, 6, 150, 3)])
def test_mirror_commit_sequences(fr, S, fields, n_par, n, seed):
    rng = np.random.default_rng(seed)
    stories = [M.random_story(rng, "s%d-" % k, S - 7 * k, n_par) for k in range(2)]
    packed = [M.story_from_steps(s) for s in stories]
    hs = [_host_story(s) for s in stories]
    slots = [h.upload(fr) for h in hs]
    b = H.HostBatch(fr, S, max(p.child_nibbles() for p in packed), fields, n)
    fr.batches.append(b)
    b.set_resident(True)
    of = rng.integers(0, 2, n)
    types = []
    for r in range(n):
        ps, kind = packed[of[r]], {s["name"]: s["type"] for s in stories[of[r]]}
        assert b.add_run(hs[of[r]], slots[of[r]]) == r
        st = M.random_state(rng, ps)
        # mostly unstarted, running or succeeded steps, a few of any code: most runs have steps to launch at every size
        st["codes"] = {k: (_codes(v[0]) if rng.random() < 2.0 / ps.S else int(rng.choice([0, 0, 0, 2, 3])), v[1], v[2])
                       for k, v in st["codes"].items()}
        st["par"] = {k: (on, [_codes(c) for c in kids]) for k, (on, kids) in st["par"].items()}
        _fill_fields(b, r, ps, st, fields)
        types.append([kind[nm] for nm in ps.names])
    wrote = pending_won = 0
    for rnd in range(5):
        b.eval()
        # sets after the eval: pending deltas, some on steps the commit writes (they win)
        for r in rng.choice(n, size=n // 5, replace=False):
            ready = [int(s) for s in b.ready(int(r))]
            pick = ready[:1] if ready and rng.random() < 0.7 else [int(rng.integers(0, packed[of[r]].S))]
            for s in pick:
                b.set_phase_code(int(r), s, int(rng.choice([0, 1, 3, 4, 13])))
                pending_won += 1
        ents = _entries(rng, b, n, types)
        if rnd == 2:   # a refusal: an entry on a step that is not ready changes neither side
            r0 = next(r for r in range(n) if len(b.ready(r)) < packed[of[r]].S)
            free = next(s for s in range(packed[of[r0]].S) if s not in set(b.ready(r0)))
            bad = np.concatenate([ents, np.array([(r0, free, CM.HOLD, 0)], dtype=Frontier.COMMIT_DTYPE)])
            mirror, dev = b.state().copy(), fr.resident_download(0, 0, n, b.L.state_stride)
            with pytest.raises(A.FrontierError) as e:
                b.commit(bad)
            assert e.value.bad_run <= r0
            assert np.array_equal(b.state(), mirror) and np.array_equal(fr.resident_download(0, 0, n, b.L.state_stride), dev)
        got = b.commit(ents)
        wrote += got["n_runs_written"]
        b.eval()
        mirror = b.state().copy()
        dev = fr.resident_download(0, 0, n, b.L.state_stride)
        diff = np.nonzero(np.any(mirror != dev, axis=1))[0]
        assert diff.size == 0, (rnd, diff[:10].tolist())
        assert fr.resident_resync(0, n, mirror, check=True, items_cap=1024)["n_drifted"] == 0
    assert wrote > 0 and pending_won > 0


def _fill_fields(b, r, ps, st, fields):
    """the run's state through the setters the layout takes"""
    if fields & A.F_COND and fields & A.F_DECISION and fields & A.F_CHILD:
        _fill(b, r, ps, st)
        return
    for i, nm in enumerate(ps.names):
        b.set_phase_code(r, i, st["codes"][nm][0])
    for q, stp in enumerate(ps.par_steps):
        b.register_children(r, q, st["par"][ps.names[stp]][0])


def test_mirror_commit_needs_resident_mode(fr):
    rng = np.random.default_rng(4)
    hs = _host_story(M.random_story(rng, "x-", 20, 1))
    slot = hs.upload(fr)
    b = H.HostBatch(fr, 32, 16, A.F_ALL_OUT, 4)
    fr.batches.append(b)
    b.add_run(hs, slot)
    b.eval()
    with pytest.raises(A.FrontierError) as e:
        b.commit()
    assert e.value.status == A.BF_EINVAL
