"""bf_schedule and bf_schedule_device bit for bit against tests/schedref.py (oracle.limiters.schedule_packed over the
reductions include/bobrafrontier.h states): records with their zeroed stride tail, story / queue / global totals and queue
maxima.  At the scale where the grid-stride loops take several trips and the tables span several sched_init blocks, at
every input edge the header pins, on word boundaries of a 1024-step mask, and after every kind of pass that may precede
a schedule."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import _pack_planes, make_layout, pack_state
from oracle import limiters as LM
from tests import randgen
from tests import schedref as SR

pytestmark = pytest.mark.gpu

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)


@pytest.fixture(scope="module")
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _sm_count():
    import torch
    return int(torch.cuda.get_device_properties(0).multi_processor_count)


def _check(fr, L, state, result, descs, sched, tables, what=""):
    n = state.shape[0]
    got = fr.schedule(L, n, sched, **tables)
    want = SR.expected(L, state, result, descs, sched, tables)
    SR.assert_schedule(got, want, what)
    return got


def _batch(rng, fr, n, smax, smin=1, parallel=True, count=40, fields=A.F_COND | A.F_DECISION, **kw):
    ts = randgen.random_topologies(rng, count, smin, smax, parallel=parallel)
    slots = fr.put_topologies(ts)
    L, state, topo = randgen.random_state(rng, ts, slots, n, fields, **kw)
    return ts, slots, L, state, topo


# ------------------------------------------------------------------------------------------ scale
@pytest.mark.parametrize("narrow", [False, True])
def test_scale(fr, narrow):
    """~30k runs of S up to 256: several grid-stride trips on a one-SM ctx (8 blocks), thousands of story keys and hundreds
    of queue keys (several sched_init blocks)"""
    rng = np.random.default_rng(31 + narrow)
    f = Frontier(0, reserve_sms=_sm_count() - 1) if narrow else fr
    try:
        ts, slots, L, state, topo = _batch(rng, f, 30000, 256, smin=200, phase_mix="progress")
        result, _ = f.eval(L, state)
        descs = SR.from_topology_set(ts, slots)
        for k, (ns, nq) in enumerate([(3000, 300), (9000, 700), (40, 5)]):
            sched = SR.random_sched(rng, 30000, ns, nq, out_of_range=0.05)
            tables = SR.random_tables(rng, ns, nq, 30000, maxprio_base=bool(k % 2))
            got = _check(f, L, state, result, descs, sched, tables, "scale %d" % k)
            hdr = np.ascontiguousarray(got["records"][:, :16]).view("<u4")
            assert hdr[:, 0].any() and (hdr[:, 1].any() or hdr[:, 2].any())   # something launched and something queued
    finally:
        if narrow:
            f.close()


# ------------------------------------------------------------------------------------------ keys, phases, priorities
@pytest.mark.parametrize("seed", range(4))
def test_keys_phases_priorities(fr, seed):
    rng = np.random.default_rng(500 + seed)
    ts, slots, L, state, topo = _batch(rng, fr, 4000, [300, 40, 1024, 97][seed], phase_mix=("any" if seed % 2 else "progress"))
    result, _ = fr.eval(L, state)
    descs = SR.from_topology_set(ts, slots)
    for ns, nq in [(5000, 600), (0, 0), (1, 1), (7, 3), (300, 2)]:
        sched = SR.random_sched(rng, 4000, ns, nq, out_of_range=0.2)
        tables = SR.random_tables(rng, ns, nq, 4000, maxprio_base=ns % 2 == 1)
        _check(fr, L, state, result, descs, sched, tables, "tables %d/%d" % (ns, nq))


def test_every_run_phase_and_priority_edge(fr):
    """every run_phase 0..15 and past 15 against every priority / elapsed / aging edge, one queue per aging value, with the
    queue maxima's base at both extremes"""
    rng = np.random.default_rng(77)
    phases = np.array(list(range(16)) + [16, 17, 0x12, 0x1F, 0xFFFFFFF2, 0xFFFFFFFF], np.uint32)
    combos = np.array(np.meshgrid(np.arange(len(phases)), np.arange(len(SR.PRIORITY_EDGES)), np.arange(len(SR.ELAPSED_EDGES) + 2),
                                  np.arange(len(SR.AGING_EDGES)), indexing="ij")).reshape(4, -1).T
    n = combos.shape[0]
    ts, slots, L, state, topo = _batch(rng, fr, n, 70, phase_mix="any")
    result, _ = fr.eval(L, state)
    elapsed = np.array(list(SR.ELAPSED_EDGES) + [59, 60], np.uint32)   # aging - 1 and aging for the 60 s queue
    aging = np.array(list(SR.AGING_EDGES) + [60], np.int32)
    sched = np.zeros(n, LM.SCHED_RUN_DTYPE)
    sched["run_phase"] = phases[combos[:, 0]]
    sched["priority"] = np.array(SR.PRIORITY_EDGES, np.int64)[combos[:, 1]]
    sched["queued_elapsed_s"] = elapsed[combos[:, 2]]
    sched["queue_key"] = combos[:, 3] + 5 * (rng.random(n) < 0.5)   # the 60 s queue (key 4) for half of the rest
    sched["queue_key"][sched["queue_key"] > 4] = 4
    sched["story_key"] = rng.integers(0, 3, size=n)
    for base in (None, [SR.INT32_MIN] * 5, [SR.INT32_MAX] * 5, [SR.INT32_MIN, -1, 0, SR.INT32_MAX - 1, SR.INT32_MAX]):
        tables = dict(story_limit=[0, 5, 100], queue_limit=[0, 0, 50, 0, 3000], queue_aging_s=aging, global_limit=0)
        if base is not None:
            tables["queue_max_priority_base"] = np.array(base, np.int32)
        _check(fr, L, state, result, SR.from_topology_set(ts, slots), sched, tables, "maxprio base %s" % base)


# ------------------------------------------------------------------------------------------ limits
def test_limits_around_the_counts(fr):
    """story / queue limits negative, 0, 1, exactly the running count, below the base and INT32_MAX; the global limit across
    the global base"""
    rng = np.random.default_rng(91)
    ts, slots, L, state, topo = _batch(rng, fr, 3000, 200, smin=60, phase_mix="progress")
    result, _ = fr.eval(L, state)
    descs = SR.from_topology_set(ts, slots)
    rr, _ = SR.running_and_demand(L, state, descs)
    ns, nq = 30, 6
    sched = SR.random_sched(rng, 3000, ns, nq, edges=False)
    sched["priority"] = 0
    sched["queued_elapsed_s"] = LM.NONE_U32
    sr = np.bincount(sched["story_key"], weights=rr, minlength=ns).astype(np.int64)
    qr = np.bincount(sched["queue_key"], weights=rr, minlength=nq).astype(np.int64)
    sb = rng.integers(0, 20, size=ns).astype(np.uint32)
    qb = rng.integers(0, 20, size=nq).astype(np.uint32)
    total = int(rr.sum()) + int(qb.sum())
    for case in range(8):
        pick = lambda run, base, m: np.array([rng.choice([SR.INT32_MIN, -1, 0, 1, int(run[i] + base[i]), int(run[i] + base[i]) + 1,
                                                          int(run[i] + base[i]) - 1, int(base[i]) - 1, int(base[i]), SR.INT32_MAX])
                                              for i in range(m)]).astype(np.int32)
        tables = dict(story_limit=pick(sr, sb, ns), queue_limit=pick(qr, qb, nq), queue_aging_s=np.zeros(nq, np.int32),
                      global_limit=int([0, -1, total - 1, total, total + 1, total + 40, int(qb.sum()) - 1, SR.INT32_MAX][case]),
                      story_running_base=sb, queue_running_base=qb, global_running_base=int(qb.sum()))
        _check(fr, L, state, result, descs, sched, tables, "limits case %d" % case)


def _all_ready_batch(fr, n, rng, running_share):
    """Stories with S = 1024 and no needs: every step not started (0) or concurrency-queued (14) is ready; a share of the
    steps Running instead"""
    k = 3
    ts = TopologySet([1024] * k, [0] * k, np.zeros(k * 1025, np.uint32), np.zeros(0, np.uint16), np.zeros(k * 1024, np.uint8),
                     [0] * k, None, None)
    slots = fr.put_topologies(ts)
    L = make_layout(1024, 0, 0)
    topo = rng.integers(0, k, size=n)
    phase = np.where(rng.random((n, 1024)) < 0.1, 14, 0).astype(np.uint8)
    phase[rng.random((n, 1024)) < running_share[:, None]] = 2
    state = pack_state(L, slots[topo], np.zeros(n, np.uint8), phase)
    return ts, slots, L, state


def test_truncation_on_word_boundaries(fr):
    """limits that leave exactly 0, 31, 32, 33, 63, 64, 65, 1023, 1024 or 1025 slots of (nearly) full 1024-step ready masks,
    through the story limit, the queue limit and the global limit"""
    rng = np.random.default_rng(1024)
    keeps = np.array([0, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025])
    n = 60
    share = np.where(np.arange(n) % 3 == 0, 0.0, np.where(np.arange(n) % 3 == 1, 0.02, 0.5))   # Running-heavy thirds
    ts, slots, L, state = _all_ready_batch(fr, n, rng, share)
    result, _ = fr.eval(L, state)
    descs = SR.from_topology_set(ts, slots)
    ready = SR.ready_of(L, result)
    full = share == 0.0
    assert (SR.popcount(ready[full]) == 1024).all()
    rr, _ = SR.running_and_demand(L, state, descs)
    sched = np.zeros(n, LM.SCHED_RUN_DTYPE)
    sched["story_key"] = np.arange(n)
    sched["queue_key"] = np.arange(n)
    sched["queued_elapsed_s"] = LM.NONE_U32
    sched["run_phase"] = 2
    base = np.full(n, 3, np.uint32)
    for through in ("story", "queue", "both"):
        ks = keeps[np.arange(n) % 10]
        kq = keeps[(np.arange(n) * 3 + 1) % 10]
        sl = (rr.astype(np.int64) + 3 + ks).astype(np.int32) if through != "queue" else np.zeros(n, np.int32)
        ql = (rr.astype(np.int64) + 3 + kq).astype(np.int32) if through != "story" else np.zeros(n, np.int32)
        tables = dict(story_limit=sl, queue_limit=ql, queue_aging_s=np.zeros(n, np.int32), story_running_base=base,
                      queue_running_base=base, global_running_base=3 * n)
        got = _check(fr, L, state, result, descs, sched, tables, "through %s" % through)
        if through == "story":
            hdr = np.ascontiguousarray(got["records"][:, :16]).view("<u4")
            assert np.array_equal(hdr[full, 0], np.minimum(ks[full], 1024))
    total = int(rr.sum()) + 3 * n
    for k in keeps:   # the global limit leaves k slots to every run
        tables = dict(story_limit=np.zeros(n, np.int32), queue_limit=np.zeros(n, np.int32), queue_aging_s=np.zeros(n, np.int32),
                      global_limit=total + int(k), story_running_base=base, queue_running_base=base, global_running_base=3 * n)
        _check(fr, L, state, result, descs, sched, tables, "global keep %d" % k)


# ------------------------------------------------------------------------------------------ edge inputs
@pytest.mark.parametrize("flags", [0, A.EVAL_FIXPOINT])
def test_edge_records(fr, flags):
    """padding and reserved codes, registered bits past each topology's parallel steps, runs on dropped and never-put
    slots, a layout child area shorter than some topologies', topologies wider than the layout; the fixpoint pass leaves
    the counts to the stored records"""
    rng = np.random.default_rng(4242 + flags)
    ts = randgen.random_topologies(rng, 30, 1, 300, parallel=True)
    slots = fr.put_topologies(ts)
    L, state, topo = randgen.random_state(rng, ts, slots, 3000, A.F_COND | A.F_DECISION, phase_mix="any", reserved=0.1,
                                          padding=True)
    descs = SR.from_topology_set(ts, slots)
    sid = np.ascontiguousarray(state[:, 0:4]).view("<u4")[:, 0].copy()
    dead = rng.random(3000) < 0.05
    sid[dead] = rng.choice([0xFFFFFF, 0x7FFFFFFF, 0xFFFFFFFF], size=int(dead.sum()))   # never put
    state[:, 0:4] = sid.astype("<u4").view(np.uint8).reshape(3000, 4)
    gone = int(slots[int(topo[0])])
    fr.drop_topology(gone)
    del descs[gone]
    result, _ = fr.eval(L, state, flags=flags)
    sched = SR.random_sched(rng, 3000, 40, 6, out_of_range=0.1)
    _check(fr, L, state, result, descs, sched, SR.random_tables(rng, 40, 6, 3000), "edge records")


def test_slots_dropped_and_put_after_the_pass():
    """drops and puts between the pass and the schedule: the schedule reads the slot table as it stands (a dropped slot counts
    nothing, a reused one its new topology), also when the puts grow the table past what the pass saw"""
    rng = np.random.default_rng(1313)
    f = Frontier(0)
    try:
        ts, slots, L, state, topo = _batch(rng, f, 3000, 120, smin=40, count=12, phase_mix="progress")
        result, _ = f.eval(L, state)
        sched = SR.random_sched(rng, 3000, 30, 4)
        tables = SR.random_tables(rng, 30, 4, 3000)
        descs = SR.from_topology_set(ts, slots)
        for k in range(3):
            gone = [int(s) for s in rng.choice(slots, size=3, replace=False) if int(s) in descs]
            for s in gone:
                f.drop_topology(s)
                del descs[s]
            more = randgen.random_topologies(rng, 600, 40, 120, parallel=True)   # reuses the dropped slots, then grows the table
            descs.update(SR.from_topology_set(more, f.put_topologies(more)))
            _check(f, L, state, result, descs, sched, tables, "after drops and puts %d" % k)
    finally:
        f.close()


def test_no_runs(fr):
    rng = np.random.default_rng(0)
    ts, slots, L, state, topo = _batch(rng, fr, 1, 40)
    result, _ = fr.eval(L, state[:0].copy())
    tables = SR.random_tables(rng, 9, 4, 0, maxprio_base=True)
    got = fr.schedule(L, 0, np.zeros(0, LM.SCHED_RUN_DTYPE), **tables)
    assert np.array_equal(got["story_running"], tables["story_running_base"])
    assert np.array_equal(got["queue_running"], tables["queue_running_base"])
    assert np.array_equal(got["queue_max_priority"], tables["queue_max_priority_base"])
    assert got["global_running"] == tables["global_running_base"]


# ------------------------------------------------------------------------------------------ each kind of preceding pass
def _deltas(rng, ts, topo, n, k):
    runs = rng.choice(n, size=k, replace=False)
    d = np.zeros(k, Frontier.DELTA_DTYPE)
    d["run"] = runs
    d["index"] = [int(rng.integers(0, int(ts.S[int(topo[r])]))) for r in runs]
    d["field"] = A.DELTA_PHASE
    d["code"] = rng.choice([0, 1, 2, 2, 3, 14], size=k)
    return d


def _apply_host(L, state, d):
    """the deltas' phase codes written into host records"""
    from bobrapet_b200.records import _unpack_planes
    out = state.copy()
    W = L.words
    codes = _unpack_planes(out[:, L.off_phase:L.off_phase + 16 * W], W, 4, 32 * W)
    codes[d["run"].astype(np.int64), d["index"].astype(np.int64)] = d["code"]
    out[:, L.off_phase:L.off_phase + 16 * W] = _pack_planes(codes, W, 4)
    return out


@pytest.mark.parametrize("kind", ["eval_compact", "eval", "eval_chunked", "tick", "tick_chunked", "compact", "compact_unfused", "changed",
                                  "touched"])
def test_after_each_pass(fr, monkeypatch, kind):
    """the schedule after every pass that may precede it equals the reference over the records the pass leaves: a first pass,
    then deltas on some runs and a second pass (for touched ticks an incremental one over the touched runs only).  The result
    records pass 2 MiB several times over, so the chunked kinds run 5 chunks and the others are held to one; compact ticks are
    one chunk and fuse their heads unless BF_NO_FUSED_HEADS (changed-only ticks never fuse)"""
    rng = np.random.default_rng(8000 + len(kind) * 31 + ord(kind[-1]))
    n = 20000
    ts, slots, L, state, topo = _batch(rng, fr, n, 180, phase_mix="progress", fields=A.F_COND | A.F_DECISION | A.F_ALL_OUT)
    assert n * L.result_stride >= 2 * (2 << 20)
    descs = SR.from_topology_set(ts, slots)
    d = _deltas(rng, ts, topo, n, 300)
    state2 = _apply_host(L, state, d)
    sched = SR.random_sched(rng, n, 50, 5, out_of_range=0.05)
    tables = SR.random_tables(rng, 50, 5, n, maxprio_base=True)
    want = []
    monkeypatch.setenv("BF_E2E_CHUNKS", "1")
    for st in (state, state2):   # the reference results, from one-chunk bf_eval passes
        res, _ = fr.eval(L, st)
        assert fr.stats()["last_eval_chunks"] == 1
        want.append(SR.expected(L, st, res, descs, sched, tables))
    chunks = 5 if kind.endswith("chunked") else 1
    monkeypatch.setenv("BF_E2E_CHUNKS", str(chunks))
    if kind.endswith("unfused"):
        monkeypatch.setenv("BF_NO_FUSED_HEADS", "1")
    if kind.startswith("eval"):
        for i, st in enumerate((state, state2)):
            if kind == "eval_compact":
                fr.eval_compact(L, st, 4_000_000)
            else:
                fr.eval(L, st)
                assert fr.stats()["last_eval_chunks"] == chunks
            SR.assert_schedule(fr.schedule(L, n, sched, **tables), want[i], "%s pass %d" % (kind, i))
        return
    h = fr.resident_create(L, n)
    try:
        fr.resident_upload(h, 0, state)
        for i, dd in enumerate((NONE, d)):
            if kind.startswith("tick"):
                fr.resident_tick(h, L, n, dd)
                assert fr.stats()["last_eval_chunks"] == chunks
            elif kind.startswith("compact"):
                fr.resident_tick_compact(h, n, dd, 4_000_000)
            elif kind == "changed":
                fr.resident_tick_compact(h, n, dd, 4_000_000, flags=A.EVAL_CHANGED_ONLY)
            else:
                out = fr.resident_tick_touched(h, n, dd, n, 4_000_000)
                assert bool(out["full"]) == (i == 0)
                if i:
                    assert out["n_evaluated"] < n
            SR.assert_schedule(fr.schedule(L, n, sched, **tables), want[i], "%s pass %d" % (kind, i))
    finally:
        fr.resident_destroy(h)


# ------------------------------------------------------------------------------------------ bf_schedule_device
def test_schedule_device(fr):
    """after eval_device on a non-default stream: equals the reference and bf_schedule, with and without bases"""
    import torch
    rng = np.random.default_rng(606)
    n, ns, nq = 6000, 700, 40
    ts, slots, L, state, topo = _batch(rng, fr, n, 400, phase_mix="progress")
    descs = SR.from_topology_set(ts, slots)
    sched = SR.random_sched(rng, n, ns, nq, out_of_range=0.05)
    dev = torch.device("cuda", 0)
    s = torch.cuda.Stream(device=dev)
    d_state = torch.from_numpy(state).to(dev)
    d_result = torch.full((n, L.result_stride), 0x5A, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    fr.eval_device(L, n, d_state.data_ptr(), d_result.data_ptr(), stream=s.cuda_stream, flags=A.EVAL_NO_COUNTS)
    for with_bases in (False, True):
        tables = SR.random_tables(rng, ns, nq, n, maxprio_base=with_bases)
        if not with_bases:
            tables = {k: v for k, v in tables.items() if k not in ("story_running_base", "queue_running_base")}
            tables["global_running_base"] = 0
        got = SR.schedule_device(fr, L, n, d_state, d_result, sched, tables, s)
        result = d_result.cpu().numpy()
        SR.assert_schedule(got, SR.expected(L, state, result, descs, sched, tables), "device bases %s" % with_bases)
        res_host, _ = fr.eval(L, state)   # the host path over the same batch gives the same schedule
        assert np.array_equal(res_host, result)
        SR.assert_schedule(fr.schedule(L, n, sched, **tables), got, "host vs device")
    # no runs: the totals are the bases
    tables = SR.random_tables(rng, ns, nq, 0, maxprio_base=True)
    got = SR.schedule_device(fr, L, 0, None, None, sched[:0], tables, s)
    assert np.array_equal(got["story_running"], tables["story_running_base"])
    assert np.array_equal(got["queue_running"], tables["queue_running_base"])
    assert np.array_equal(got["queue_max_priority"], tables["queue_max_priority_base"])
    assert got["global_running"] == tables["global_running_base"]
    # the totals are the device path's reduction scratch: leaving one out is refused
    t = {k: SR.to_device(v, dev) for k, v in tables.items() if isinstance(v, np.ndarray)}
    bufs = [torch.zeros(max(m, 1), dtype=torch.int32, device=dev) for m in (ns, nq, nq, 1)]
    for missing in range(4):
        ptrs = [b.data_ptr() for b in bufs]
        ptrs[missing] = 0
        with pytest.raises(A.FrontierError) as e:
            fr.schedule_device(L, 0, 0, 0, 0, 0, *ptrs, ns, nq, t["story_limit"].data_ptr(), t["queue_limit"].data_ptr(),
                               t["queue_aging_s"].data_ptr(), stream=s.cuda_stream)
        assert e.value.status == A.BF_EINVAL


def test_schedule_device_outside_the_layout(fr):
    """records at a layout with fewer words and a shorter child area than some of their topologies need: the steps, phase
    codes and children the layout does not hold count nothing.  bf_schedule_device reads any (state, result) pair, so the
    ready masks here are random"""
    import torch
    rng = np.random.default_rng(707)
    n = 4000
    ts = randgen.random_topologies(rng, 30, 1, 300, parallel=True)
    slots = fr.put_topologies(ts)
    L, state, topo = randgen.random_state(rng, ts, slots, n, A.F_CHILD, phase_mix="any")
    narrow = make_layout(128, max(L.child_nibbles // 2, 8), A.F_CHILD)
    assert narrow.words < L.words and narrow.child_nibbles < L.child_nibbles
    from bobrapet_b200.records import _unpack_planes
    short = np.zeros((n, narrow.state_stride), np.uint8)
    short[:, :16] = state[:, :16]
    codes = _unpack_planes(state[:, L.off_phase:L.off_phase + 16 * L.words], L.words, 4, 32 * L.words)[:, :32 * narrow.words]
    short[:, narrow.off_phase:narrow.off_phase + 16 * narrow.words] = _pack_planes(codes, narrow.words, 4)
    nb = (narrow.child_nibbles + 1) // 2
    short[:, narrow.off_child:narrow.off_child + nb] = state[:, L.off_child:L.off_child + nb]
    result = rng.integers(0, 256, size=(n, narrow.result_stride), dtype=np.uint8)
    dev = torch.device("cuda", 0)
    s = torch.cuda.Stream(device=dev)
    sched = SR.random_sched(rng, n, 40, 6, out_of_range=0.1)
    tables = SR.random_tables(rng, 40, 6, n, maxprio_base=True)
    got = SR.schedule_device(fr, narrow, n, SR.to_device(short, dev), SR.to_device(result, dev), sched, tables, s)
    SR.assert_schedule(got, SR.expected(narrow, short, result, SR.from_topology_set(ts, slots), sched, tables), "outside the layout")
