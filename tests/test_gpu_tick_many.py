"""bf_resident_tick_touched_many: the touched ticks of several resident batches in one call equal, byte for byte, one
bf_resident_tick_touched per part in array order.  Twin sets of batches (widths 64 / 512 / 1024, with and without cond and
decision planes and a child area) take the same deltas and the same lifecycle calls; set M ticks through the new call, set S
through the single one, and after every tick the lists, counts, state records and the following resident schedule must agree."""
import ctypes as C

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import randgen

pytestmark = pytest.mark.gpu

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
# name -> (steps min, steps max, parallel steps (a child area), fields)
SPECS = {
    "w64": (20, 64, False, 0),
    "w64p": (20, 64, True, A.F_ALL_OUT),
    "w512d": (300, 512, False, ALL),
    "w1024p": (600, 1000, True, A.F_ALL_OUT),
    "w1024d": (600, 1000, True, ALL),
}
TABLES = dict(story_limit=np.array([0, 2, 40, 5], np.int32), queue_limit=np.array([0, 30, 7], np.int32),
              queue_aging_s=np.array([60, 0, 30], np.int32), global_limit=500)


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


class Part:
    """One width class: batch m (ticked by the new call) and its twin s (single calls), same records and the same calls"""

    def __init__(self, fr, rng, spec, n, cap=None, sched=False):
        s_lo, s_hi, par, fields = SPECS[spec]
        self.fr = fr
        self.ts = randgen.random_topologies(rng, 12, s_lo, s_hi, max_deg=4, parallel=par, fill=0.5)
        self.slots = fr.put_topologies(self.ts)
        self.L, self.state, _ = randgen.random_state(rng, self.ts, self.slots, n, fields, phase_mix="progress")
        self.n, self.cap = n, cap or n + 64
        self.m, self.s = fr.resident_create(self.L, self.cap), fr.resident_create(self.L, self.cap)
        put = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
        put["run"] = np.arange(n)
        put["story_key"], put["queue_key"] = rng.integers(0, 4, n), rng.integers(0, 3, n)
        put["priority"], put["queued_since"], put["run_phase"] = rng.integers(0, 5, n), 0xFFFFFFFF, 2
        for h in (self.m, self.s):
            fr.resident_upload(h, 0, self.state)
            if sched:
                fr.resident_sched(h)
                fr.resident_sched_put(h, put)

    def both(self, fn):
        return fn(self.m), fn(self.s)

    def same_records(self):
        a, b = self.both(lambda h: self.fr.resident_download(h, 0, self.cap, self.L.state_stride))
        assert np.array_equal(a, b)


def deltas(rng, p, k, rejected=False):
    """k coalesced deltas over phase / run-flag / topology-slot fields of runs below p.n; with rejected, one delta whose step is
    past the layout (rejected by the scatter, which still touches its run)"""
    W32 = 32 * p.L.words
    recs = {}
    for _ in range(k):
        r, f = int(rng.integers(0, p.n)), int(rng.choice([A.DELTA_PHASE] * 6 + [A.DELTA_RUN_FLAGS, A.DELTA_TOPO_SLOT]))
        if f == A.DELTA_PHASE:
            idx, code = int(rng.integers(0, W32)), int(rng.choice([0, 1, 2, 3, 3, 4, 9, 13, 14]))
        elif f == A.DELTA_RUN_FLAGS:
            idx, code = 0, int(rng.choice([0, A.RF_FAIL_FAST, A.RF_TOPOLOGY_TERMINATED]))
        else:
            new = int(rng.choice(p.slots))
            idx, code = new & 0xFFFF, new >> 16
        recs[(r, f, idx if f != A.DELTA_TOPO_SLOT else 0)] = (idx, code)
    if rejected:
        recs[(int(rng.integers(0, p.n)), A.DELTA_PHASE, 0xFFFF)] = (0xFFFF, 3)
    d = np.zeros(len(recs), dtype=Frontier.DELTA_DTYPE)
    for i, ((r, f, _), (idx, code)) in enumerate(recs.items()):
        d[i] = (r, idx, f, code)
    return d


def spec_of(p, d, runs_cap, events_cap, pinned):
    q = dict(n_runs=p.n, deltas=d, runs_cap=runs_cap, events_cap=events_cap)
    if pinned:
        fr = p.fr
        q.update(runs=fr.alloc_pinned(max(runs_cap, 1) * 4).view(np.uint32), head=fr.alloc_pinned(max(runs_cap, 1) * 4).view(np.uint32),
                 events=fr.alloc_pinned(max(events_cap, 1) * 2).view(np.uint16))
    return q


def free_pinned(fr, q):
    for k in ("runs", "head", "events"):
        if k in q:
            fr.free_pinned(q[k])


def same_result(a, b):
    for k in ("full", "n_listed", "n_evaluated", "n_events", "counts"):
        assert a[k] == b[k], (k, a[k], b[k])
    for k in ("runs", "head", "events"):
        assert np.array_equal(a[k], b[k]), k


def tick_both(fr, parts, ds, flags=0, max_iter=0, caps=None, pinned=None):
    """one tick of every part: the new call on the m batches, one single call per part (in order) on the s batches.  ->
    (results, rejected): the parts whose deltas the single calls rejected"""
    n = len(parts)
    caps = caps or [(p.n, 4_000_000) for p in parts]
    pinned = pinned or [False] * n
    qm = [dict(spec_of(p, d, rc, ec, pn), handle=p.m) for p, d, (rc, ec), pn in zip(parts, ds, caps, pinned)]
    qs = [dict(spec_of(p, d, rc, ec, pn), handle=p.s) for p, d, (rc, ec), pn in zip(parts, ds, caps, pinned)]
    try:
        single, rejected = [], []
        for k, q in enumerate(qs):
            try:
                single.append(fr.resident_tick_touched(q["handle"], q["n_runs"], q["deltas"], q["runs_cap"], q["events_cap"], flags,
                                                       max_iter, runs=q.get("runs"), head=q.get("head"), events=q.get("events")))
            except A.FrontierError as e:
                assert e.status == A.BF_EINVAL and "delta" in str(e), e
                single.append(None)
                rejected.append(k)
        if rejected:
            with pytest.raises(A.FrontierError) as ei:
                fr.resident_tick_touched_many(qm, flags, max_iter)
            assert ei.value.status == A.BF_EINVAL and ei.value.bad_part == rejected[0], (ei.value, rejected)
            got = None
        else:
            got = fr.resident_tick_touched_many(qm, flags, max_iter)
            assert len(got) == n
            for a, b in zip(got, single):
                same_result({**a, "runs": a["runs"].copy(), "head": a["head"].copy(), "events": a["events"].copy()}, b)
        for p in parts:
            p.same_records()
        return got, rejected
    finally:
        for q in qm + qs:
            free_pinned(fr, q)


def schedule_both(fr, parts, now):
    got = [fr.resident_schedule([dict(handle=getattr(p, w), n_runs=p.n) for p in parts], TABLES, now) for w in ("m", "s")]
    for a, b in zip(got[0]["parts"], got[1]["parts"]):
        for k in a:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    for k in ("story_running", "queue_running", "queue_max_priority", "global_running"):
        assert np.array_equal(np.asarray(got[0][k]), np.asarray(got[1][k])), k


@pytest.mark.parametrize("names,seed", [(("w64",), 0), (("w64", "w512d"), 1), (("w64p", "w512d", "w1024p"), 2),
                                        (("w1024d", "w64", "w512d", "w64p"), 3)])
def test_sequences_equal_single_calls(fr, names, seed):
    rng = np.random.default_rng(seed)
    parts = [Part(fr, rng, nm, int(rng.integers(300, 2500)), sched=True) for nm in names]
    spare = fr.put_topologies(randgen.random_topologies(rng, 3, 10, 40, parallel=False))   # no run holds them: dropped later
    flags = 0
    for t in range(24):
        op = int(rng.integers(0, 8))
        if op == 0 and len(spare):   # a slot drop: every part's next touched tick is full
            fr.drop_topology(int(spare[0]))
            spare = spare[1:]
        elif op == 1:   # BF_EVAL_FIXPOINT flips: full ticks
            flags ^= A.EVAL_FIXPOINT
        elif op == 2:   # uploads past n: the next tick lists them without being full
            p = parts[int(rng.integers(0, len(parts)))]
            k = int(min(rng.integers(1, 40), p.cap - p.n))
            if k:
                recs = p.state[rng.integers(0, p.state.shape[0], k)].copy()
                p.both(lambda h: fr.resident_upload(h, p.n, recs))
                p.n += k
        elif op == 3:   # retire a few runs
            p = parts[int(rng.integers(0, len(parts)))]
            runs = rng.choice(p.n, size=int(rng.integers(1, 6)), replace=False)
            (nm, _, _), (ns, _, _) = p.both(lambda h: fr.resident_retire(h, p.n, runs))
            assert nm == ns
            p.n = nm
        elif op == 4:   # redrive whole runs
            p = parts[int(rng.integers(0, len(parts)))]
            st = fr.resident_download(p.m, 0, p.n, p.L.state_stride)
            rr = rng.choice(p.n, size=3, replace=False)
            rq = np.zeros(3, dtype=Frontier.REDRIVE_DTYPE)
            rq["run"], rq["step"] = rr, A.REDRIVE_ALL
            rq["slot"] = st[rr, 0:4].copy().view("<u4")[:, 0] & 0xFFFFFF
            a, b = p.both(lambda h: fr.resident_redrive(h, rq))
            assert np.array_equal(a[0], b[0]) and a[1] == b[1]
        ds = [deltas(rng, p, int(rng.choice([0, 1, 5, 60]))) if rng.random() < 0.85 else NONE for p in parts]
        caps = [(int(rng.choice([p.n, 3, 0])), int(rng.choice([4_000_000, 50, 0]))) for p in parts]
        pinned = [bool(rng.random() < 0.5) for _ in parts]
        got, _ = tick_both(fr, parts, ds, flags, 0, caps, pinned)
        schedule_both(fr, parts, 1000 + t)
        if rng.random() < 0.5 and not flags & A.EVAL_FIXPOINT:   # commit the tick's launches on every part
            for p in parts:
                a, b = p.both(lambda h: fr.resident_commit(h, p.n))
                assert a == b
                p.same_records()


def test_full_in_one_part_only_and_empty_parts(fr):
    rng = np.random.default_rng(11)
    parts = [Part(fr, rng, nm, 1500) for nm in ("w64", "w512d", "w1024p")]
    tick_both(fr, parts, [NONE] * 3)                       # first ticks: full everywhere
    got, _ = tick_both(fr, parts, [deltas(rng, p, 20) for p in parts])
    assert [g["full"] for g in got] == [0, 0, 0]
    recs = parts[1].state[:10].copy()                     # n_runs past the last full tick without uploads: part 1 alone is full
    parts[1].both(lambda h: fr.resident_upload(h, 1500, recs))
    parts[1].n = 1510
    d1 = deltas(rng, parts[1], 3)
    parts[1].both(lambda h: fr.resident_apply(h, d1))
    parts[1].n = 1520                                     # ... past the uploads too
    got, _ = tick_both(fr, parts, [deltas(rng, parts[0], 9), deltas(rng, parts[1], 9), NONE])
    assert [g["full"] for g in got] == [0, 1, 0]
    assert got[2]["n_evaluated"] == 0                     # no deltas and nothing pending: no touched runs
    got, _ = tick_both(fr, parts, [NONE, NONE, NONE])
    assert [g["n_evaluated"] for g in got] == [0, 0, 0]
    assert fr.resident_tick_touched_many([]) == []


def test_rejected_delta_in_each_part(fr):
    rng = np.random.default_rng(12)
    parts = [Part(fr, rng, nm, 900) for nm in ("w64p", "w512d", "w1024d")]
    tick_both(fr, parts, [NONE] * 3)
    for k in range(3):
        ds = [deltas(rng, p, 10, rejected=(j == k)) for j, p in enumerate(parts)]
        _, rejected = tick_both(fr, parts, ds)
        assert rejected == [k]
        got, _ = tick_both(fr, parts, [NONE] * 3)   # the rejected delta touched its run exactly as in the single call
        assert got is not None


def test_caps_below_counts_and_pinned_buffers(fr):
    rng = np.random.default_rng(13)
    parts = [Part(fr, rng, nm, 3000) for nm in ("w64", "w512d", "w1024p")]
    tick_both(fr, parts, [NONE] * 3)
    for pinned in ([True] * 3, [False] * 3, [True, False, True]):
        ds = [deltas(rng, p, 400) for p in parts]
        tick_both(fr, parts, ds, caps=[(7, 11), (0, 0), (100, 3)], pinned=pinned)


@pytest.mark.parametrize("n_big", [524_288 + 1000, 2_100_000])
def test_list_grids_across_1024_ctas(fr, n_big):
    """a touched tick over more than 1024 * 512 listed positions (the compaction grid) and, at 2.1 M runs, more than
    1024 * 2048 marks (the list build's grid), beside small parts"""
    rng = np.random.default_rng(14)
    parts = [Part(fr, rng, "w64", n_big), Part(fr, rng, "w512d", 700)]
    tick_both(fr, parts, [NONE] * 2)
    d = np.zeros(n_big, dtype=Frontier.DELTA_DTYPE)   # every run of the big part touched
    d["run"], d["index"], d["field"], d["code"] = np.arange(n_big), 0, A.DELTA_PHASE, rng.choice([0, 2, 3], n_big)
    got, _ = tick_both(fr, parts, [d, deltas(rng, parts[1], 30)], caps=[(n_big, 40_000_000), (700, 1_000_000)],
                       pinned=[True, False])
    assert got[0]["full"] == 0 and got[0]["n_evaluated"] == n_big


def _raw_call(fr, parts, specs, flags=0):
    """the C call with parts built field by field (a part may carry a NULL out or a bad struct_size)"""
    outs, cs, keep = [], (A.TickPart * len(specs))(), []
    for k, q in enumerate(specs):
        runs, head, ev = np.zeros(q["n_runs"] + 1, np.uint32), np.zeros(q["n_runs"] + 1, np.uint32), np.zeros(1 << 16, np.uint16)
        to = A.TouchedOut(struct_size=C.sizeof(A.TouchedOut), runs=runs.ctypes.data, head=head.ctypes.data, runs_cap=q["n_runs"],
                          events=ev.ctypes.data, events_cap=1 << 16)
        keep += [runs, head, ev, to, q["deltas"]]
        cs[k] = A.TickPart(struct_size=q.get("struct_size", C.sizeof(A.TickPart)), handle=q["handle"], deltas=q["deltas"].ctypes.data,
                           n_deltas=q["deltas"].shape[0], n_runs=q["n_runs"], out=None if q.get("null_out") else C.addressof(to))
    bad = C.c_uint32(7)
    rc = fr._lib.bf_resident_tick_touched_many(fr._ctx, flags, 0, cs, len(specs), C.byref(bad))
    return rc, bad.value


def test_refusals_change_nothing(fr):
    rng = np.random.default_rng(15)
    parts = [Part(fr, rng, nm, 800) for nm in ("w64", "w512d", "w1024p")]
    tick_both(fr, parts, [NONE] * 3)
    for pos in range(3):
        for kind in ("repeat", "n_runs", "null_out", "struct_size", "handle"):
            if kind == "repeat" and pos == 0:
                continue
            ds = [deltas(rng, p, 25) for p in parts]
            specs = [dict(handle=p.m, n_runs=p.n, deltas=d) for p, d in zip(parts, ds)]
            if kind == "repeat":
                specs[pos]["handle"] = parts[pos - 1].m
            elif kind == "n_runs":
                specs[pos]["n_runs"] = parts[pos].cap + 1
            elif kind == "null_out":
                specs[pos]["null_out"] = True
            elif kind == "struct_size":
                specs[pos]["struct_size"] = C.sizeof(A.TickPart) - 8
            else:
                specs[pos]["handle"] = 999
            before = [fr.resident_download(p.m, 0, p.cap, p.L.state_stride) for p in parts]
            rc, bad = _raw_call(fr, parts, specs)
            assert rc == A.BF_EINVAL and bad == pos, (kind, pos, rc, bad)
            for p, b in zip(parts, before):
                assert np.array_equal(fr.resident_download(p.m, 0, p.cap, p.L.state_stride), b)
            tick_both(fr, parts, ds)   # touch state unchanged: the next ticks of both twins list the same runs
    ds = [deltas(rng, p, 5) for p in parts]
    rc, bad = _raw_call(fr, parts, [dict(handle=p.m, n_runs=p.n, deltas=d) for p, d in zip(parts, ds)], flags=A.EVAL_EXPANSION)
    assert rc == A.BF_EINVAL and bad == A.COMMIT_NONE
    tick_both(fr, parts, ds)


def test_one_part_is_the_single_call(fr):
    rng = np.random.default_rng(16)
    p = Part(fr, rng, "w512d", 2000)
    for t in range(6):
        got, _ = tick_both(fr, [p], [deltas(rng, p, 50) if t else NONE], flags=A.EVAL_FIXPOINT if t == 4 else 0)
        assert got[0]["full"] == (1 if t in (0, 4, 5) else 0)
