"""Device groups through the C ABI (bf_group_*): one process, G GPUs, runs sharded in contiguous blocks, one NCCL
all-gather of the per-shard counts per pass, and limiters whose totals are all-reduced across the shards.

On a 1-GPU box the group has one shard (the communicator has one rank); with 2+ GPUs every G up to the device count runs."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import FrontierGroup, synth
from bobrapet_b200.records import make_layout
from oracle import limiters as LM
from oracle import packed as PK
from tests import randgen
from tests import schedref as SR

pytestmark = pytest.mark.gpu


# Group sizes are fixed, not taken from the device count at collection: a test's id must not depend on the machine that
# collects it (a host without a visible GPU would otherwise collect an empty parameter set).  Sizes above the device
# count skip at run time.
@pytest.fixture(params=(1, 2, 3, 4, 8))
def group(request):
    import torch
    if request.param > torch.cuda.device_count():
        pytest.skip("a group of %d GPUs needs %d devices" % (request.param, request.param))
    g = FrontierGroup(list(range(request.param)))
    yield g
    g.close()


def test_group_eval_sharded_topologies(group):
    """unique-topology mode: every shard holds the topologies of its own block of runs (slot ids are per shard)"""
    n, S = 9001, 256
    ts_all = synth.topologies(4, 0, n, S)
    L = make_layout(S, 0, A.F_COND | A.F_DECISION | A.F_ALL_OUT)
    state = np.zeros((n, L.state_stride), dtype=np.uint8)
    want = np.zeros((n, L.result_stride), dtype=np.uint8)
    per_want = []
    covered = 0
    for k in range(group.size):
        first, count = group.shard_range(n, k)
        assert first == covered
        covered += count
        if count == 0:
            per_want.append({"ready": 0, "skip": 0, "expansion": 0, "evals": 0})
            continue
        ts = synth.topologies(4, first, count, S)
        slots = group.shards[k].put_topologies(ts)
        state[first:first + count] = synth.state(4, first, count, L, slots, ts)
        want[first:first + count], wc = PK.evaluate(PK.PackedTopologies(ts, slots), L, state[first:first + count], threads=8)
        per_want.append(wc)
    assert covered == n
    got, counts, per = group.eval(L, state)
    assert np.array_equal(got, want)
    assert per == per_want
    assert counts == {f: sum(p[f] for p in per_want) for f in ("ready", "skip", "expansion", "evals")}


@pytest.mark.parametrize("seed", range(3))
def test_group_schedule_holds_limits_across_shards(group, seed):
    """replicated topologies; limits, bases and priority ordering are enforced over the WHOLE batch, not per shard"""
    rng = np.random.default_rng(8100 + seed)
    ts = randgen.random_topologies(rng, 30, 1, [60, 257, 130][seed], parallel=(seed == 0))
    slots = group.put_topologies_replicated(ts)
    n = [3001, 2500, 4003][seed]
    L, state, topo = randgen.random_state(rng, ts, slots, n, A.F_COND | A.F_DECISION, phase_mix=("any" if seed % 2 else "progress"))
    want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=8)
    result, counts, _ = group.eval(L, state)
    assert np.array_equal(result, want) and counts == wcounts
    n_stories, n_queues = int(rng.integers(1, 20)), int(rng.integers(1, 5))
    sched = np.zeros(n, dtype=LM.SCHED_RUN_DTYPE)
    sched["story_key"] = rng.integers(0, n_stories, size=n)
    sched["queue_key"] = rng.integers(0, n_queues, size=n)
    sched["priority"] = rng.integers(-3, 8, size=n)
    el = rng.integers(0, 4000, size=n).astype(np.uint32)
    el[rng.random(n) < 0.5] = LM.NONE_U32
    sched["queued_elapsed_s"] = el
    sched["run_phase"] = rng.choice([0, 1, 2, 3, 4, 8, 11], size=n)
    story_limit = rng.choice([0, 0, 1, 3, 40, 200, 1000], size=n_stories).astype(np.int32)
    queue_limit = rng.choice([0, 50, 2000, 20000], size=n_queues).astype(np.int32)
    queue_aging = rng.choice([0, 30, 60, 600], size=n_queues).astype(np.int32)
    global_limit = int(rng.choice([0, 100, 5000, 100000]))
    story_base = rng.integers(0, 5, size=n_stories).astype(np.uint32)
    queue_base = rng.integers(0, 50, size=n_queues).astype(np.uint32)
    global_base = int(queue_base.sum())
    tables = dict(story_limit=story_limit, queue_limit=queue_limit, queue_aging_s=queue_aging, global_limit=global_limit,
                  story_running_base=story_base, queue_running_base=queue_base, global_running_base=global_base)
    got = group.schedule(L, n, sched, **tables)
    SR.assert_schedule(got, SR.expected(L, state, result, SR.from_topology_set(ts, slots), sched, tables, loop=True))


@pytest.mark.parametrize("seed", range(2))
def test_group_schedule_edges(group, seed):
    """the edge generator of test_gpu_schedule.py across shards: keys out of range, every run_phase, int32 priority extremes and
    the wrap, limits at their extremes, padding and reserved codes, thousands of story keys, and queue_max_priority_base set"""
    rng = np.random.default_rng(8200 + seed)
    ts = randgen.random_topologies(rng, 30, 1, [300, 1024][seed], parallel=True)
    slots = group.put_topologies_replicated(ts)
    n = [6001, 3001][seed]
    L, state, topo = randgen.random_state(rng, ts, slots, n, A.F_COND | A.F_DECISION, phase_mix="any", reserved=0.1, padding=True)
    result, _, _ = group.eval(L, state)
    descs = SR.from_topology_set(ts, slots)
    for ns, nq in ((3000, 300), (0, 0), (7, 3)):
        sched = SR.random_sched(rng, n, ns, nq, out_of_range=0.1)
        tables = SR.random_tables(rng, ns, nq, n, maxprio_base=True)
        SR.assert_schedule(group.schedule(L, n, sched, **tables), SR.expected(L, state, result, descs, sched, tables),
                           "tables %d/%d" % (ns, nq))


def test_group_rejects_bad_arguments(group):
    L = make_layout(32, 0, 0)
    with pytest.raises(A.FrontierError):
        group.schedule(L, 5, np.zeros(5, dtype=LM.SCHED_RUN_DTYPE), [0], [0], [0])   # no preceding bf_group_eval of 5 runs
    import ctypes as C
    lib = A.load()
    g = C.c_void_p()
    dup = (C.c_int32 * 2)(0, 0)
    assert lib.bf_group_create(C.byref(g), dup, 2, None) == A.BF_EINVAL          # the same device twice
    assert lib.bf_group_create(C.byref(g), dup, 0, None) == A.BF_EINVAL


def test_queue_max_priority_base_blocks_lower_priority_runs():
    """bf_sched_tables.queue_max_priority_base: a higher-priority run with demand OUTSIDE the batch queues the batch's
    lower-priority runs (enforcePriorityOrdering compares against every non-terminal StoryRun of the queue, dag.go:1917-1944;
    dag_test.go:528 TestEnforcePriorityOrderingBlocksLowerPriority)"""
    from bobrapet_b200 import Frontier
    f = Frontier(0)
    try:
        ts = synth.topologies(3, 0, 16, 64)
        slots = f.put_topologies(ts)
        L = make_layout(64, 0, 0)
        state = np.zeros((16, L.state_stride), dtype=np.uint8)
        state[:, 0:4] = np.ascontiguousarray(slots, dtype="<u4").view(np.uint8).reshape(16, 4)
        result, counts = f.eval(L, state)               # nothing started: the steps without needs are ready
        assert counts["ready"] >= 16
        sched = np.zeros(16, dtype=LM.SCHED_RUN_DTYPE)
        sched["priority"], sched["queued_elapsed_s"], sched["run_phase"] = 1, LM.NONE_U32, 2
        free = f.schedule(L, 16, sched, [0], [0], [0])
        blocked = f.schedule(L, 16, sched, [0], [0], [0], queue_max_priority_base=[5])
        equal = f.schedule(L, 16, sched, [0], [0], [0], queue_max_priority_base=[1])
        hdr = lambda r: np.ascontiguousarray(r["records"][:, 0:16]).view("<u4").reshape(16, 4)
        assert (hdr(free)[:, 0] > 0).all() and (hdr(free)[:, 2] == 0).all()
        assert (hdr(blocked)[:, 0] == 0).all() and (hdr(blocked)[:, 3] == A.QUEUED_PRIORITY).all() and int(blocked["queue_max_priority"][0]) == 5
        assert np.array_equal(hdr(equal), hdr(free))    # an equal priority outside does not outrank (strictly greater, :1933)
    finally:
        f.close()
