"""GPU parity of the limiters (rows a9 / f4): bf_eval -> bf_schedule through the C ABI vs tests/schedref.py (oracle.limiters.schedule_packed),
bit for bit, on adversarial random batches (all step types, parallel children, every phase code) and random
stories / queues / limits / priorities."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from oracle import limiters as LM
from tests import randgen
from tests import schedref as SR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fr():
    f = Frontier(0)
    yield f
    f.close()


@pytest.mark.parametrize("seed", range(8))
def test_schedule_matches_oracle(fr, seed):
    rng = np.random.default_rng(7000 + seed)
    smax = [40, 257, 1024, 96, 600, 33, 8, 130][seed]
    ts = randgen.random_topologies(rng, 40, 1, smax, parallel=(seed % 2 == 0))
    slots = fr.put_topologies(ts)
    n = [3000, 2999, 700, 3001, 1200, 3003, 2000, 2500][seed]
    L, state, topo = randgen.random_state(rng, ts, slots, n, A.F_COND | A.F_DECISION, phase_mix=("any" if seed % 2 else "progress"))
    result, _ = fr.eval(L, state)
    W = L.words
    ready = np.ascontiguousarray(result[:, L.off_ready:L.off_ready + 4 * W]).view("<u4").reshape(n, W)
    n_stories, n_queues = int(rng.integers(1, 30)), int(rng.integers(1, 6))
    sched = np.zeros(n, dtype=LM.SCHED_RUN_DTYPE)
    sched["story_key"] = rng.integers(0, n_stories, size=n)
    sched["queue_key"] = rng.integers(0, n_queues, size=n)
    sched["priority"] = rng.integers(-3, 8, size=n)
    el = rng.integers(0, 4000, size=n).astype(np.uint32)
    el[rng.random(n) < 0.5] = LM.NONE_U32
    sched["queued_elapsed_s"] = el
    sched["run_phase"] = rng.choice([0, 1, 2, 3, 4, 8, 11], size=n)
    # limits sized to the batch so that every branch (no limit / some slots / zero slots) occurs
    story_limit = rng.choice([0, 0, 1, 3, 40, 200, 1000], size=n_stories).astype(np.int32)
    queue_limit = rng.choice([0, 50, 2000, 20000], size=n_queues).astype(np.int32)
    queue_aging = rng.choice([0, 30, 60, 600], size=n_queues).astype(np.int32)
    global_limit = int(rng.choice([0, 100, 5000, 100000]))
    story_base = rng.integers(0, 5, size=n_stories).astype(np.uint32)
    queue_base = rng.integers(0, 50, size=n_queues).astype(np.uint32)
    global_base = int(queue_base.sum())
    tables = dict(story_limit=story_limit, queue_limit=queue_limit, queue_aging_s=queue_aging, global_limit=global_limit,
                  story_running_base=story_base, queue_running_base=queue_base, global_running_base=global_base)
    got = fr.schedule(L, n, sched, **tables)
    SR.assert_schedule(got, SR.expected(L, state, result, SR.from_topology_set(ts, slots), sched, tables, loop=True))
    rec = got["records"]
    masks = np.ascontiguousarray(rec[:, 16:16 + 12 * W]).view("<u4").reshape(n, 3, W)
    # the three masks partition the ready set (every ready step is launched or queued, dag.go:1709-1728)
    assert np.array_equal(masks[:, 0] | masks[:, 1] | masks[:, 2], ready)


def test_schedule_requires_preceding_eval(fr):
    ts = randgen.random_topologies(np.random.default_rng(1), 4, 5, 20, parallel=False)
    slots = fr.put_topologies(ts)
    L, state, _ = randgen.random_state(np.random.default_rng(2), ts, slots, 10, 0)
    fr.eval(L, state)
    sched = np.zeros(11, dtype=LM.SCHED_RUN_DTYPE)
    with pytest.raises(A.FrontierError):
        fr.schedule(L, 11, sched, [0], [0], [0])   # n_runs differs from the evaluated batch
