"""bfh_batch_commit_rewrites: the C++ host mirror commits a tick on the device through bf_resident_commit_rewrites and applies the
journal, rewrite items included, to its own records.  The sequences of tests/test_gpu_mirror_commit.py with the rewriting commit:
after each commit and the next eval the mirror's records equal the device's download, and bf_resident_resync with BF_RESYNC_CHECK
over the mirror's records reports no drift; pending deltas win, a refused commit changes neither side."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200 import host as H
from tests import commit as CM
from tests import migration as M
from tests.test_gpu_migrate import _host_story
from tests.test_gpu_mirror_commit import ALL, _entries, _codes, _fill_fields, fr  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("S,fields,n_par,n,seed", [(40, ALL | A.F_CHILD, 3, 500, 1), (120, A.F_OUT_FAIL, 0, 300, 2),
                                                   (300, A.F_ALL_OUT | A.F_CHILD, 6, 150, 3)])
def test_mirror_rewriting_commit_sequences(fr, S, fields, n_par, n, seed):
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
    wrote = pending_won = rewritten = 0
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
                b.commit(bad, rewrites=True)
            assert e.value.bad_run <= r0
            assert np.array_equal(b.state(), mirror) and np.array_equal(fr.resident_download(0, 0, n, b.L.state_stride), dev)
        got = b.commit(ents, rewrites=True)
        wrote += got["n_runs_written"]
        rewritten += got["n_rewritten"]
        b.eval()
        mirror = b.state().copy()
        dev = fr.resident_download(0, 0, n, b.L.state_stride)
        diff = np.nonzero(np.any(mirror != dev, axis=1))[0]
        assert diff.size == 0, (rnd, diff[:10].tolist())
        assert fr.resident_resync(0, n, mirror, check=True, items_cap=1024)["n_drifted"] == 0
    assert wrote > 0 and pending_won > 0 and rewritten > 0
