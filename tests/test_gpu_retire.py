"""bf_resident_retire: runs leave a live resident batch and the last live runs move into the indices they free.  The records and
moves are checked byte for byte against tests/retire.py, and the ticks that follow against a changed-only twin, a twin batch
uploaded in the new order with the same history, and the packed oracle."""
import ctypes as C

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200 import host as H
from oracle import packed as PK
from tests import migration as M
from tests import randgen
from tests import retire as RT
from tests.test_gpu_migrate import _sched
from tests.test_gpu_reshape import _deltas, _fill, _host_story
from tests.test_host_retire import _runs

pytestmark = pytest.mark.gpu

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
# shape: (steps lo, hi, layout fields, parallel steps, runs)
SHAPES = {"cfg3": (200, 257, 0, False, 1500),         # phase only
          "cfg4": (200, 257, ALL, True, 1500),        # cond + decision planes, registered bits and child nibbles
          "cfg5": (513, 700, ALL, True, 600)}         # S > 512 (the general kernel)
SHARES = ["none", "one", "tail", "head", "all", "0.1", "0.5"]
CAPS = ["keep", "m", "between"]
EXTRA = 16   # records above n_runs: not runs for the call


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _batch(fr, rng, shape):
    lo, hi, fields, parallel, n = SHAPES[shape]
    ts = randgen.random_topologies(rng, 10, lo, hi, max_deg=4, parallel=parallel, fill=0.5)
    slots = fr.put_topologies(ts)
    L, st, _ = randgen.random_state(rng, ts, slots, n + EXTRA, fields, phase_mix="progress")
    return PK.PackedTopologies(ts, slots), L, st, n


def _remap(d, idx):
    """deltas on old run indices -> the same deltas on the new ones, those of retired runs dropped"""
    new = idx[d["run"].astype(np.int64)]
    out = d[new >= 0].copy()
    out["run"] = new[new >= 0]
    return out


def _tick_twin(fr, L, rows, n_cap, d1):
    """a batch holding `rows` from the start, with the history of the retired one: a changed-only tick, then d1"""
    h = fr.resident_create(L, n_cap)
    fr.resident_upload(h, 0, rows)
    fr.resident_tick_compact(h, rows.shape[0], NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    if d1.shape[0]:
        fr.resident_apply(h, d1)
    return h


@pytest.mark.parametrize("cap_mode", CAPS)
@pytest.mark.parametrize("share", SHARES)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_retire_records_and_the_ticks_that_follow(fr, shape, share, cap_mode):
    rng = np.random.default_rng(list(SHAPES).index(shape) * 100 + SHARES.index(share) * 10 + CAPS.index(cap_mode))
    pt, L, st, n = _batch(fr, rng, shape)
    cap = n + EXTRA + 8
    hA, hB = fr.resident_create(L, cap), fr.resident_create(L, cap)   # A: touched ticks; B: its twin, changed-only ticks
    hs = [hA, hB]
    try:
        for h in (hA, hB):
            fr.resident_upload(h, 0, st)
        assert fr.resident_tick_touched(hA, n, NONE, n, BIG)["full"] == 1
        fr.resident_tick_compact(hB, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        prev, _ = PK.evaluate(pt, L, st[:n], 0, 0, threads=8)           # the current result records of both
        d1 = _deltas(rng, L, n, 120)                                     # touched before the call
        for h in (hA, hB):
            fr.resident_apply(h, d1)
        st1 = fr.resident_download(hA, 0, cap, L.state_stride)
        runs = _runs(rng, n, share)
        m, src, dst = RT.moves(n, runs)
        capacity = {"keep": 0, "m": m, "between": (m + cap + 1) // 2}[cap_mode]
        new_cap = capacity or cap
        for h in (hA, hB):
            got_m, mf, mt = fr.resident_retire(h, n, runs, capacity)
            assert got_m == m and np.array_equal(mf, src) and np.array_equal(mt, dst)
        want = RT.retire_records(st1, n, runs, new_cap)
        for h in (hA, hB):
            assert np.array_equal(fr.resident_download(h, 0, new_cap, L.state_stride), want)
        with pytest.raises(A.FrontierError):   # the capacity is what the call left
            fr.resident_download(hA, 0, new_cap + 1, L.state_stride)
        if m == 0:
            o = fr.resident_tick_touched(hA, 0, NONE, 1, BIG)
            assert o["full"] == 0 and o["n_evaluated"] == 0
            return
        idx, order = RT.new_index(n, runs), RT.order(n, runs)
        # a twin uploaded in the new order with the same history
        hC = _tick_twin(fr, L, np.ascontiguousarray(st[order]), m, _remap(d1, idx))
        hs.append(hC)
        assert np.array_equal(fr.resident_download(hC, 0, m, L.state_stride), want[:m])
        # the next ticks: A touched, B and C changed-only, all with the same deltas
        d2 = _deltas(rng, L, m, 90)
        oA = fr.resident_tick_touched(hA, m, d2, m, BIG)
        bhead, bev, _, _, _ = fr.resident_tick_compact(hB, m, d2, BIG, flags=A.EVAL_CHANGED_ONLY)
        chead, cev, _, _, _ = fr.resident_tick_compact(hC, m, d2, BIG, flags=A.EVAL_CHANGED_ONLY)
        assert np.array_equal(bhead, chead) and np.array_equal(bev, cev)
        st2 = fr.resident_download(hA, 0, m, L.state_stride)
        for h in (hB, hC):
            assert np.array_equal(fr.resident_download(h, 0, m, L.state_stride), st2)
        res, _ = PK.evaluate(pt, L, st2, 0, 0, threads=8)
        whead, wev, _ = PK.compact_events(L, res, prev[order])
        assert np.array_equal(bhead, whead) and np.array_equal(bev, wev)
        # A: not full; evaluates the moved runs and every run touched before or after the call; lists the moved runs and the
        # runs whose result changed, with the heads and events a compact tick gives them
        touched = set(dst.tolist()) | set(d2["run"].tolist()) | set(int(i) for i in idx[d1["run"].astype(np.int64)] if i >= 0)
        listed = np.array(sorted(set(np.nonzero(bhead & A.HEAD_LISTED)[0].tolist()) | set(dst.tolist())), np.uint32)
        assert oA["full"] == 0 and oA["n_evaluated"] == len(touched)
        assert np.array_equal(oA["runs"], listed)
        lhead, lev, _ = PK.compact_events(L, res[listed])
        assert np.array_equal(oA["head"], lhead) and np.array_equal(oA["events"], lev)
        # and the tick after it: A lists exactly what the changed-only twin lists
        d3 = _deltas(rng, L, m, 60)
        oA = fr.resident_tick_touched(hA, m, d3, m, BIG)
        bhead, bev, _, _, _ = fr.resident_tick_compact(hB, m, d3, BIG, flags=A.EVAL_CHANGED_ONLY)
        st3 = fr.resident_download(hA, 0, m, L.state_stride)
        res3, _ = PK.evaluate(pt, L, st3, 0, 0, threads=8)
        whead, wev, _ = PK.compact_events(L, res3, res)
        assert np.array_equal(bhead, whead) and np.array_equal(bev, wev)
        assert oA["full"] == 0 and np.array_equal(oA["runs"], np.nonzero(whead & A.HEAD_LISTED)[0])
        assert np.array_equal(oA["head"], whead[oA["runs"]]) and np.array_equal(oA["events"], wev)
        got, _ = fr.resident_tick(hA, L, m, NONE)
        assert np.array_equal(got, res3)
        # uploads into the vacated tail: covered ones keep the touched tick incremental, a run beyond them makes it full
        k = min(8, new_cap - m)
        if k:
            fr.resident_tick_touched(hA, m, NONE, m, BIG)
            fr.resident_upload(hA, m, np.ascontiguousarray(st[:k]))
            o = fr.resident_tick_touched(hA, m + k, NONE, m + k, BIG)
            assert o["full"] == 0 and np.array_equal(o["runs"], np.arange(m, m + k))
        if m + k < new_cap:
            o = fr.resident_tick_touched(hA, m + k + 1, NONE, m + k + 1, BIG)
            assert o["full"] == 1 and o["n_listed"] == m + k + 1
    finally:
        for h in hs:
            fr.resident_destroy(h)


def test_retire_ends_the_snapshot_and_keeps_migrate_and_redrive_working(fr):
    """bf_schedule is refused until a new pass; migrations and redrives address the moved runs at their new index"""
    rng = np.random.default_rng(61)
    old = M.random_story(rng, "a-", 40, 2)
    new = M.edit_story(rng, old, "a-e")
    other = M.random_story(rng, "b-", 30, 1)
    ps = [M.story_from_steps(s) for s in (old, new, other)]
    hs = [_host_story(s) for s in (old, new, other)]
    slots = [h.upload(fr) for h in hs]
    fields = A.F_COND | A.F_DECISION | A.F_CHILD | A.F_ALL_OUT
    child = max(p.child_nibbles() for p in ps)
    n = 400
    story = rng.choice([0, 2], n)
    mr = H.HostBatch(None, 64, child, fields, n)
    try:
        for r in range(n):
            mr.add_run(hs[story[r]], slots[story[r]])
            _fill(mr, r, ps[story[r]], M.random_state(rng, ps[story[r]]))
        L = A.Layout.from_buffer_copy(mr.L)
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, mr.state().copy())
        fr.resident_eval(h, L, n)
        sched = _sched(n)
        fr.schedule(L, n, *sched, global_limit=20000)
        runs = rng.choice(n, size=150, replace=False).astype(np.uint32)
        m, mf, mt = fr.resident_retire(h, n, runs)
        hf, ht = mr.retire(runs)
        assert np.array_equal(hf, mf) and np.array_equal(ht, mt) and mr.size() == m
        with pytest.raises(A.FrontierError):   # the snapshot of the last pass is gone, as after an upload
            fr.schedule(L, n, *sched, global_limit=20000)
        fr.resident_eval(h, L, m)
        fr.schedule(L, m, *_sched(m), global_limit=20000)
        assert np.array_equal(fr.resident_download(h, 0, m, L.state_stride), mr.state())
        # an edit of Story 0 migrates the moved runs too, at their new index
        smap = hs[0].migration_map(hs[1])
        on_old = int((np.ascontiguousarray(mr.state()[:, 0:4]).view("<u4").reshape(m) == slots[0]).sum())
        assert fr.resident_migrate(h, slots[0], slots[1], smap, m) == on_old
        assert mr.migrate(hs[0], hs[1], slots[0], slots[1]) == on_old
        assert np.array_equal(fr.resident_download(h, 0, m, L.state_stride), mr.state())
        # redrives of moved runs (and one that kept its index)
        kept = [r for r in range(m) if r not in set(mt.tolist())][:1]
        targets = np.array(list(mt[:6]) + kept, np.uint32)
        slot_of = np.ascontiguousarray(mr.state()[:, 0:4]).view("<u4").reshape(m)
        req = np.zeros(len(targets), dtype=Frontier.REDRIVE_DTYPE)
        req["run"], req["slot"], req["step"] = targets, slot_of[targets], A.REDRIVE_ALL
        _, applied = fr.resident_redrive(h, req)
        assert applied == len(targets)
        mr.redrive(targets, np.full(len(targets), -1, np.int32))
        assert np.array_equal(fr.resident_download(h, 0, m, L.state_stride), mr.state())
        fr.resident_destroy(h)
    finally:
        mr.close()


def test_retire_rejections_change_nothing(fr):
    rng = np.random.default_rng(67)
    pt, L, st, n = _batch(fr, rng, "cfg4")
    hA, hB = fr.resident_create(L, n + EXTRA), fr.resident_create(L, n + EXTRA)   # B never sees the rejected calls
    try:
        for h in (hA, hB):
            fr.resident_upload(h, 0, st)
            fr.resident_tick_touched(h, n, NONE, n, BIG)
        d = _deltas(rng, L, n, 60)
        for h in (hA, hB):
            fr.resident_apply(h, d)
        lib = A.load()
        for runs, n_runs, capacity in [([n], n, 0),                       # not a run
                                       ([3, 3], n, 0),                    # twice
                                       ([1, 2], n + EXTRA + 1, 0),        # n_runs above the capacity
                                       ([1, 2], n, n - 3),                # a capacity below the runs that stay
                                       ([1, 2], n, n + EXTRA + 1)]:       # a capacity above the current one
            with pytest.raises(A.FrontierError) as e:
                fr.resident_retire(hA, n_runs, np.array(runs, np.uint32), capacity)
            assert e.value.status == A.BF_EINVAL, (runs, n_runs, capacity)
        rt = A.Retire(struct_size=C.sizeof(A.Retire) - 4, n_runs=n, runs=None, n=0)
        assert lib.bf_resident_retire(fr._ctx, hA, C.byref(rt)) == A.BF_EINVAL     # struct_size
        rt = A.Retire(struct_size=C.sizeof(A.Retire), n_runs=n, runs=None, n=2)
        assert lib.bf_resident_retire(fr._ctx, hA, C.byref(rt)) == A.BF_EINVAL     # null runs
        assert lib.bf_resident_retire(fr._ctx, hA, None) == A.BF_EINVAL
        with pytest.raises(A.FrontierError) as e:
            fr.resident_retire(hA + 7, n, np.array([1], np.uint32))                 # an unknown handle
        assert e.value.status == A.BF_EINVAL
        assert np.array_equal(fr.resident_download(hA, 0, n + EXTRA, L.state_stride),
                              fr.resident_download(hB, 0, n + EXTRA, L.state_stride))
        # n == 0 without a capacity is a no-op, and keeps the next touched tick as it was
        for h in (hA, hB):
            got_m, mf, mt = fr.resident_retire(h, n, np.zeros(0, np.uint32))
            assert got_m == n and mf.size == 0 and mt.size == 0
        oA = fr.resident_tick_touched(hA, n, NONE, n, BIG)
        oB = fr.resident_tick_touched(hB, n, NONE, n, BIG)
        for k in ("full", "n_listed", "n_evaluated", "n_events"):
            assert oA[k] == oB[k], k
        for k in ("runs", "head", "events"):
            assert np.array_equal(oA[k], oB[k]), k
        assert oA["full"] == 0
        # n == 0 with a capacity only trims the capacity
        assert fr.resident_retire(hA, n, np.zeros(0, np.uint32), n)[0] == n
        assert np.array_equal(fr.resident_download(hA, 0, n, L.state_stride), fr.resident_download(hB, 0, n, L.state_stride))
        with pytest.raises(A.FrontierError):
            fr.resident_download(hA, 0, n + 1, L.state_stride)
        o = fr.resident_tick_touched(hA, n, NONE, n, BIG)
        assert o["full"] == 0 and o["n_evaluated"] == 0
    finally:
        for h in (hA, hB):
            fr.resident_destroy(h)


def test_mirror_retire_in_resident_mode_keeps_pending_deltas(fr):
    """pending deltas on retired, moved and unmoved runs, and runs not yet on the device: the mirror and the device agree after the
    next eval, and equal a resident mirror built from the survivors"""
    rng = np.random.default_rng(71)
    steps = M.random_story(rng, "m-", 28, 2)
    ps = M.story_from_steps(steps)
    hs = _host_story(steps)
    slot = hs.upload(fr)
    fields = A.F_COND | A.F_DECISION | A.F_CHILD | A.F_OUT_SKIP_DEP
    c = ps.child_nibbles()
    n, n_dev = 150, 120
    states = [M.random_state(rng, ps) for _ in range(n)]
    a = H.HostBatch(fr, 32, c, fields, n)
    b = H.HostBatch(fr, 32, c, fields, n)
    try:
        a.set_resident(True)
        for r in range(n_dev):
            a.add_run(hs, slot)
            _fill(a, r, ps, states[r])
        a.eval()   # [0, n_dev) on the device
        for r in range(n_dev, n):   # the rest only in the mirror
            a.add_run(hs, slot)
            _fill(a, r, ps, states[r])
        edited_runs = np.concatenate([rng.choice(110, 50, replace=False), np.arange(110, 120)])
        edits = [(int(r), int(rng.integers(0, ps.S)), int(rng.choice([2, 3, 4]))) for r in edited_runs]
        for r, i, code in edits:   # pending deltas
            a.set_phase_code(int(r), i, code)
            states[r]["codes"][ps.names[i]] = (code,) + tuple(states[r]["codes"][ps.names[i]][1:])
        assert a.traffic()[2] > 0
        # retired runs with and without pending deltas, and none of [110, 120): its edited runs move with their deltas
        edited = sorted({int(r) for r, _, _ in edits})
        pool = np.array([r for r in range(1, n) if not 110 <= r < 120 and r != edited[0]])
        runs = np.concatenate([[edited[0]], rng.choice(pool, size=49, replace=False)]).astype(np.uint32)
        mf, mt = a.retire(runs, n - 20)
        m = n - 50
        assert a.size() == m
        b.set_resident(True)
        for j, r in enumerate(RT.order(n, runs)):
            b.add_run(hs, slot)
            _fill(b, j, ps, states[r])
        assert np.array_equal(a.state(), b.state())
        a.eval()
        b.eval()
        assert a.traffic()[2] == 0
        assert np.array_equal(a.state(), b.state()) and np.array_equal(a.result(), b.result())
    finally:
        a.close()
        b.close()
