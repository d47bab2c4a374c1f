"""bf_resident_extent / bf_resident_narrow: a live resident batch sheds the width, planes and child area its wide Stories needed.
The records are checked byte for byte against packing every code again at the narrow layout, the extent against a numpy
computation over the downloaded records and the topologies, and the ticks that follow against a twin created at the narrow
layout from the start, a twin taking changed-only ticks, and the packed oracle."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier, TopologySet
from bobrapet_b200 import host as H
from bobrapet_b200.records import PAR_DTYPE, make_layout, pack_state
from oracle import packed as PK
from tests import randgen
from tests import reshape as RS
from tests.narrowing import narrow_result, narrow_state, numpy_extent, topo_child_nibbles

pytestmark = pytest.mark.gpu

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _deltas(rng, L, n, k, fields=None):
    """k coalesced deltas on about k / 3 runs, inside the layout's steps_max and child area, over every field it has"""
    runs = rng.choice(n, size=k // 3 + 1, replace=False)
    has = lambda off: off != A.OFF_NONE  # noqa: E731
    fl = [A.DELTA_PHASE] * 4 + [A.DELTA_RUN_FLAGS, A.DELTA_REGISTERED]
    fl += [A.DELTA_COND] * has(L.off_cond) + [A.DELTA_DECISION] * has(L.off_decision)
    fl += [A.DELTA_CHILD] * (has(L.off_child) and L.child_nibbles > 0)
    recs = {}
    for _ in range(k):
        r, f = int(rng.choice(runs)), int(rng.choice(fl))
        if f == A.DELTA_PHASE:
            idx, code = int(rng.integers(0, L.steps_max)), int(rng.choice([0, 1, 2, 3, 3, 4, 9, 13, 14]))
        elif f in (A.DELTA_COND, A.DELTA_DECISION):
            idx, code = int(rng.integers(0, L.steps_max)), int(rng.integers(0, 4))
        elif f == A.DELTA_CHILD:
            idx, code = int(rng.integers(0, L.child_nibbles)), int(rng.choice([0, 2, 3, 4, 13]))
        elif f == A.DELTA_RUN_FLAGS:
            idx, code = 0, int(rng.choice([0, A.RF_FAIL_FAST, A.RF_FAIL_FAST | A.RF_REALTIME, A.RF_TOPOLOGY_TERMINATED]))
        else:
            idx, code = int(rng.integers(0, 64)), int(rng.integers(0, 2))
        recs[(r, f, idx)] = code
    d = np.zeros(len(recs), dtype=Frontier.DELTA_DTYPE)
    for i, ((r, f, idx), code) in enumerate(recs.items()):
        d[i] = (r, idx, f, code)
    return d


def _zero_planes(L, st, off, nbits):
    if off != A.OFF_NONE:
        st[:, off:off + nbits * L.words * 4] = 0


# wide steps_max, narrow steps_max (the Stories' largest), wide fields, fields dropped, spare child nibbles of the wide layout,
# parallel steps
CASES = {"256-32": (256, 32, COND | DEC | OUT, 0, 0, True),
         "224-32": (224, 32, COND | DEC, 0, 8, True),           # 7 words -> 1, and the child area shrinks
         "64-40": (64, 40, COND | OUT, 0, 0, False),
         "cond-dropped": (96, 96, COND | DEC | OUT, COND, 0, True),
         "decision-dropped": (64, 32, COND | DEC | OUT, DEC, 0, False),
         "child-dropped": (64, 64, CHILD | A.F_OUT_SKIP_DEP, CHILD, 16, False),
         "out-dropped": (128, 32, COND | OUT, A.F_OUT_PHASE | A.F_OUT_NEEDS_COND, 0, True)}


def _batch(fr, rng, case, n):
    """-> (pt, wide layout, narrow layout, records at the wide layout) for a case"""
    s_w, s_n, f_w, drop, spare, parallel = CASES[case]
    ts = randgen.random_topologies(rng, 12, max(2, s_n // 2), s_n, max_deg=4, parallel=parallel, fill=0.5)
    slots = fr.put_topologies(ts)
    L0, st0, _ = randgen.random_state(rng, ts, slots, n, f_w & ~CHILD, phase_mix="progress")
    if drop & COND:
        _zero_planes(L0, st0, L0.off_cond, 2)
    if drop & DEC:
        _zero_planes(L0, st0, L0.off_decision, 2)
    Lw = make_layout(s_w, L0.child_nibbles + spare, L0.fields | f_w)
    Ln = make_layout(s_n, L0.child_nibbles, Lw.fields & ~drop)
    return PK.PackedTopologies(ts, slots), Lw, Ln, RS.reshape_state(L0, Lw, st0, n)


@pytest.mark.parametrize("case", list(CASES))
def test_narrow_records_and_the_ticks_that_follow(fr, case):
    rng = np.random.default_rng(list(CASES).index(case) + 300)
    n = 1500
    pt, Lw, Ln, st = _batch(fr, rng, case, n)
    drop = CASES[case][3]
    hA, hB = fr.resident_create(Lw, n), fr.resident_create(Lw, n)   # A: touched ticks; B: its twin, changed-only ticks
    hC = fr.resident_create(Ln, n)                                  # C: created at the narrow layout, the same uploads and deltas
    for h in (hA, hB):
        fr.resident_upload(h, 0, st)
    fr.resident_upload(hC, 0, narrow_state(Lw, Ln, st))
    assert fr.resident_tick_touched(hA, n, NONE, n, BIG)["full"] == 1
    assert fr.resident_tick_touched(hC, n, NONE, n, BIG)["full"] == 1
    fr.resident_tick_compact(hB, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    prev, _ = PK.evaluate(pt, Lw, st, 0, 0, threads=8)              # the current result records of A and B
    d1 = _deltas(rng, Ln, n, 90)                                      # touched before the narrow
    for h in (hA, hB, hC):
        fr.resident_apply(h, d1)
    st1 = fr.resident_download(hA, 0, n, Lw.state_stride)
    for h in (hA, hB):
        e = fr.resident_narrow(h, Ln, n)
        assert e["steps_max"] <= Ln.steps_max and not (e["fields"] & drop)
    want = narrow_state(Lw, Ln, st1)
    for h in (hA, hB, hC):
        assert np.array_equal(fr.resident_download(h, 0, n, Ln.state_stride), want)
    d2 = _deltas(rng, Ln, n, 90)
    oA = fr.resident_tick_touched(hA, n, d2, n, BIG)
    oC = fr.resident_tick_touched(hC, n, d2, n, BIG)
    bhead, bev, _, _, _ = fr.resident_tick_compact(hB, n, d2, BIG, flags=A.EVAL_CHANGED_ONLY)
    st2 = fr.resident_download(hA, 0, n, Ln.state_stride)
    for h in (hB, hC):
        assert np.array_equal(fr.resident_download(h, 0, n, Ln.state_stride), st2)
    res, _ = PK.evaluate(pt, Ln, st2, 0, 0, threads=8)
    whead, wev, _ = PK.compact_events(Ln, res)
    # the changed-only twin compares with its result records as the narrow truncated them
    ohead, oev, _ = PK.compact_events(Ln, res, narrow_result(Lw, Ln, prev))
    assert np.array_equal(bhead, ohead) and np.array_equal(bev, oev)
    if drop & (DEC | CHILD | OUT):   # any result may change: the next touched tick is full
        assert oA["full"] == 1 and np.array_equal(oA["head"], whead) and np.array_equal(oA["events"], wev)
    else:                             # incremental, exactly as the batch created at the narrow layout
        assert oA["full"] == 0 and oC["full"] == 0
        assert oA["n_evaluated"] == len(set(d1["run"].tolist()) | set(d2["run"].tolist()))
        for k in ("n_listed", "n_evaluated", "n_events"):
            assert oA[k] == oC[k], k
        for k in ("runs", "head", "events"):
            assert np.array_equal(oA[k], oC[k]), k
    # dense and changed-only ticks: the narrowed batch, the narrow-born one and the oracle agree
    for h in (hA, hC):
        got, _ = fr.resident_tick(h, Ln, n, NONE)
        assert np.array_equal(got, res)
    d3 = _deltas(rng, Ln, n, 60)
    oA, oC = fr.resident_tick_touched(hA, n, d3, n, BIG), fr.resident_tick_touched(hC, n, d3, n, BIG)
    assert oA["full"] == oC["full"] == 0
    for k in ("runs", "head", "events"):
        assert np.array_equal(oA[k], oC[k]), k
    for h in (hA, hB, hC):
        fr.resident_destroy(h)


@pytest.mark.parametrize("case", list(CASES))
def test_which_narrows_make_the_next_touched_tick_full(fr, case):
    rng = np.random.default_rng(list(CASES).index(case) + 400)
    n = 700
    _, Lw, Ln, st = _batch(fr, rng, case, n)
    h = fr.resident_create(Lw, n + 50)
    fr.resident_upload(h, 0, st)
    fr.resident_tick_touched(h, n, NONE, n, BIG)
    fr.resident_narrow(h, Ln, n)
    o = fr.resident_tick_touched(h, n, NONE, n, BIG)
    if CASES[case][3] & (DEC | CHILD | OUT):
        assert o["full"] == 1 and o["n_listed"] == n
    else:   # nothing touched since the last tick: nothing evaluated, nothing listed
        assert o["full"] == 0 and o["n_evaluated"] == 0 and o["n_listed"] == 0
    # the records above n_runs were not checked: a touched tick over them is full
    assert fr.resident_tick_touched(h, n + 50, NONE, n + 50, BIG)["full"] == 1
    fr.resident_destroy(h)


def _wide_topology(S):
    """S independent engram steps: every step with phase 0 is ready"""
    return TopologySet([S], [0], np.zeros(S + 1, np.uint32), np.zeros(0, np.uint16), np.zeros(S, np.uint8))


def _parallel_topology(branches):
    """4 independent steps, step 0 a parallel step of `branches` branches"""
    par = np.zeros(1, dtype=PAR_DTYPE)
    par[0] = (0, branches, 0)
    flags = np.array([A.STEP_PARALLEL, 0, 0, 0], np.uint8)
    return TopologySet([4], [0], np.zeros(5, np.uint32), np.zeros(0, np.uint16), flags, [1], par,
                       np.zeros((branches + 7) // 8, np.uint8))


REJECTIONS = ["phase-above", "record-above-n-runs", "slot-too-wide", "slot-child-area", "cond-code", "decision-code",
              "child-nibble", "result-bit", "grows-steps", "grows-field", "grows-child"]


@pytest.mark.parametrize("cause", REJECTIONS)
def test_narrow_rejections_change_nothing(fr, cause):
    rng = np.random.default_rng(REJECTIONS.index(cause) + 500)
    n, extra = 600, 16
    ts = randgen.random_topologies(rng, 10, 8, 32, max_deg=4, parallel=True, fill=0.5, branch_choices=(1, 2, 3, 7, 8))
    slots = fr.put_topologies(ts)
    L0, st0, _ = randgen.random_state(rng, ts, slots, n, COND | DEC, phase_mix="progress")
    big = _parallel_topology(L0.child_nibbles + 17)
    big_child = int(topo_child_nibbles(big)[0])
    assert big_child > L0.child_nibbles
    wide_slot = int(fr.put_topologies(_wide_topology(48))[0])
    big_slot = int(fr.put_topologies(big)[0])
    Lw = make_layout(128, max(L0.child_nibbles, big_child) + 8, L0.fields | OUT)
    st = RS.reshape_state(L0, Lw, st0, n)
    hA, hB = fr.resident_create(Lw, n + extra), fr.resident_create(Lw, n + extra)   # B never sees the rejected call
    for h in (hA, hB):
        fr.resident_upload(h, 0, st)
        fr.resident_tick_touched(h, n, NONE, n, BIG)
    Ln = make_layout(32, L0.child_nibbles, Lw.fields)
    setup, want = [], {}
    if cause == "phase-above":
        setup = [(17, 40, A.DELTA_PHASE, 3)]
        want = {"steps_max": 41, "widest_run": 17}
    elif cause == "record-above-n-runs":
        rec = np.zeros((1, Lw.state_stride), np.uint8)
        rec[0, Lw.off_phase + 4 * 1 + 2] = 0x04   # phase plane 0, word 1, bit 18: step 50
        for h in (hA, hB):
            fr.resident_upload(h, n + 5, rec)
        want = {"steps_max": 51, "widest_run": n + 5}
    elif cause == "slot-too-wide":
        setup = [(9, wide_slot & 0xFFFF, A.DELTA_TOPO_SLOT, wide_slot >> 16)]
        want = {"steps_max": 48, "widest_run": 9}
    elif cause == "slot-child-area":
        setup = [(12, big_slot & 0xFFFF, A.DELTA_TOPO_SLOT, big_slot >> 16)]
        want = {"child_nibbles": big_child}
    elif cause == "cond-code":
        Ln = make_layout(32, L0.child_nibbles, Lw.fields & ~COND)
        want = {"fields": COND}
    elif cause == "decision-code":
        Ln = make_layout(32, L0.child_nibbles, Lw.fields & ~DEC)
        want = {"fields": DEC}
    elif cause == "child-nibble":
        Ln = make_layout(32, 0, Lw.fields & ~CHILD)
        want = {"fields": CHILD}
    elif cause == "result-bit":   # run 11 evaluated on the 48-step slot, then moved back: its result record keeps steps 32..47
        d = np.zeros(2, dtype=Frontier.DELTA_DTYPE)
        d[0] = (11, wide_slot & 0xFFFF, A.DELTA_TOPO_SLOT, wide_slot >> 16)
        d[1] = (11, 0, A.DELTA_RUN_FLAGS, 0)
        for h in (hA, hB):
            fr.resident_tick_touched(h, n, d, n, BIG)
        back = int(np.ascontiguousarray(st[11, 0:4]).view("<u4")[0])
        setup = [(11, back & 0xFFFF, A.DELTA_TOPO_SLOT, back >> 16)]
        want = {"steps_max": 48, "widest_run": 11}
    elif cause == "grows-steps":
        Ln = make_layout(160, L0.child_nibbles, Lw.fields)
    elif cause == "grows-field":
        Ln = make_layout(32, L0.child_nibbles, Lw.fields | A.F_OUT_SKIP_DEP)
        Lw2 = make_layout(128, Lw.child_nibbles, Lw.fields & ~A.F_OUT_SKIP_DEP)
        for h in (hA, hB):   # a batch without the field
            fr.resident_narrow(h, Lw2, n)
        Lw = Lw2
    elif cause == "grows-child":
        Ln = make_layout(32, Lw.child_nibbles + 8, Lw.fields)
    if setup:
        d = np.zeros(len(setup), dtype=Frontier.DELTA_DTYPE)
        for i, t in enumerate(setup):
            d[i] = t
        for h in (hA, hB):
            fr.resident_apply(h, d)
    before = fr.resident_download(hA, 0, n + extra, Lw.state_stride)
    with pytest.raises(A.FrontierError) as e:
        fr.resident_narrow(hA, Ln, n)
    assert e.value.status == A.BF_EINVAL
    got = e.value.extent
    for k, v in want.items():
        assert (got[k] & v if k == "fields" else got[k]) == v, (k, got)
    assert got == fr.resident_extent(hA, n)   # the rejected call reports the extent (over the planes the layout keeps)
    after = fr.resident_download(hA, 0, n + extra, Lw.state_stride)
    assert np.array_equal(after, before) and np.array_equal(after, fr.resident_download(hB, 0, n + extra, Lw.state_stride))
    d = _deltas(rng, Ln if not cause.startswith("grows") else Lw, n, 60)
    for flags in (0, A.EVAL_FIXPOINT):
        oA = fr.resident_tick_touched(hA, n, d, n, BIG, flags=flags)
        oB = fr.resident_tick_touched(hB, n, d, n, BIG, flags=flags)
        for k in ("full", "n_listed", "n_evaluated", "n_events"):
            assert oA[k] == oB[k], k
        for k in ("runs", "head", "events"):
            assert np.array_equal(oA[k], oB[k]), k
        d = NONE
    for h in (hA, hB):
        fr.resident_destroy(h)


@pytest.mark.parametrize("seed", range(4))
def test_extent_matches_numpy(fr, seed):
    rng = np.random.default_rng(600 + seed)
    ts = randgen.random_topologies(rng, 14, 4, [40, 100, 256, 700][seed], max_deg=4, parallel=True, fill=0.5)
    slots = fr.put_topologies(ts)
    n = 900
    L0, st0, topo = randgen.random_state(rng, ts, slots, n, [COND | DEC, COND, DEC | OUT, 0][seed] | A.F_OUT_SKIP_DEP,
                                         phase_mix=["any", "progress"][seed % 2], padding=seed == 2)
    L = make_layout(L0.steps_max + 40, L0.child_nibbles + 24 * (L0.child_nibbles > 0), L0.fields)
    cap = n + 100
    st = RS.reshape_state(L0, L, st0, cap)
    st[n:n + 100] = RS.reshape_state(L0, L, st0[rng.choice(n, 100)], 100)   # records above n_runs, uploaded ahead
    h = fr.resident_create(L, cap)
    fr.resident_upload(h, 0, st)
    fr.resident_tick(h, L, n, NONE)
    dead = [int(slots[k]) for k in rng.choice(ts.count, 3, replace=False)]
    for s in dead:
        fr.drop_topology(s)
    S = {int(s): int(ts.S[k]) for k, s in enumerate(slots) if int(s) not in dead}
    ch = topo_child_nibbles(ts)
    C = {int(s): int(ch[k]) for k, s in enumerate(slots) if int(s) not in dead}
    state = fr.resident_download(h, 0, cap, L.state_stride)
    # the current result records are those of the tick above (the drops do not rewrite them)
    result, _ = PK.evaluate(PK.PackedTopologies(ts, slots), L, state[:n], 0, 0, threads=8)
    for n_runs in (0, n // 3, n, cap):
        if n_runs > n:
            continue
        want = numpy_extent(L, state, result, n_runs, S, C)
        assert fr.resident_extent(h, n_runs) == want, n_runs
    fr.resident_destroy(h)


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


def test_mirror_narrow_in_resident_mode_keeps_pending_deltas(fr):
    from tests import migration as M
    rng = np.random.default_rng(71)
    steps = M.random_story(rng, "n-", 28, 2)
    ps = M.story_from_steps(steps)
    hs = _host_story(steps)
    slot = hs.upload(fr)
    fields = COND | DEC | CHILD | OUT
    c = ps.child_nibbles()
    n = 120
    a = H.HostBatch(fr, 200, c + 30, fields, n)
    b = H.HostBatch(fr, 32, c, fields, n)
    try:
        a.set_resident(True)
        for x in (a, b):
            for r in range(n):
                x.add_run(hs, slot)
                x.set_phase_code(r, r % ps.S, 3)
                x.set_decision(r, (r * 3) % ps.S, A.DEC_SUCCEED)
        a.eval()
        for x in (a, b):   # pending deltas at the time of the narrow
            for r in range(0, n, 7):
                x.set_phase_code(r, 3, 2)
                x.set_cond(r, 5, A.COND_SKIP)
        pending = a.traffic()[2]
        assert pending > 0
        with pytest.raises(A.FrontierError):
            a.narrow(32, c, fields & ~COND)   # cond codes are pending: nothing is dropped silently
        a.narrow(32, c, fields)
        assert a.L.as_dict() == b.L.as_dict()
        assert a.traffic()[2] == pending and np.array_equal(a.state(), b.state())
        a.eval()
        b.eval()
        assert np.array_equal(a.state(), b.state()) and np.array_equal(a.result(), b.result())
    finally:
        a.close()
        b.close()


def _records_on(L, slots):
    """records of runs with no step state yet on the given slots"""
    n = len(slots)
    return pack_state(L, np.asarray(slots, np.uint32), np.zeros(n, np.uint8), np.zeros((n, 1), np.uint8))


def test_extent_ignores_result_records_no_tick_compares_with(fr):
    """result records that hold no current evaluation never limit a narrow: those of a batch before its first tick (device memory a
    destroyed batch of wide runs used), of indices a retire vacated and an upload re-admitted, and of a run replaced by an upload"""
    rng = np.random.default_rng(77)
    ts = randgen.random_topologies(rng, 6, 8, 24, max_deg=3, parallel=False, fill=0.5)
    small = [int(s) for s in fr.put_topologies(ts)]
    wide = int(fr.put_topologies(_wide_topology(48))[0])   # 48 independent steps: every result has bits up to step 47
    L, T = make_layout(64, 0, COND | OUT), make_layout(24, 0, COND | OUT)
    n = 512
    narrow_recs = _records_on(L, rng.choice(small, n))
    for _ in range(2):   # result memory a destroyed batch of wide runs leaves behind
        g = fr.resident_create(L, n)
        fr.resident_upload(g, 0, _records_on(L, [wide] * n))
        got, _ = fr.resident_tick(g, L, n, NONE)
        assert RS._planes(got, L.off_ready, L.words, 1)[:, 40:].any()
        fr.resident_destroy(g)
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, narrow_recs)
    e = fr.resident_extent(h, n)
    assert e["steps_max"] == int(ts.S.max()) and e["steps_max"] <= 24, e
    fr.resident_narrow(h, T, n)
    o = fr.resident_tick_touched(h, n, NONE, n, BIG)
    pt = PK.PackedTopologies(ts, np.asarray(small, np.uint32))
    res, _ = PK.evaluate(pt, T, fr.resident_download(h, 0, n, T.state_stride), 0, 0, threads=8)
    assert o["full"] == 1 and np.array_equal(o["head"], PK.compact_events(T, res)[0])
    fr.resident_destroy(h)
    # a retire vacates the tail of wide runs, an upload re-admits narrow runs there, another replaces wide run 3 in place
    h = fr.resident_create(L, n)
    slots = rng.choice(small, n)
    slots[3], slots[n - 16:] = wide, wide
    fr.resident_upload(h, 0, _records_on(L, slots))
    fr.resident_tick_touched(h, n, NONE, n, BIG)
    assert fr.resident_extent(h, n)["steps_max"] == 48
    fr.resident_retire(h, n, np.arange(n - 16, n))
    fr.resident_upload(h, n - 16, narrow_recs[:16])
    fr.resident_upload(h, 3, narrow_recs[3:4])
    e = fr.resident_extent(h, n)
    assert e["steps_max"] <= 24, e
    fr.resident_narrow(h, T, n)
    o = fr.resident_tick_touched(h, n, NONE, n, BIG)   # incremental: the retire and the narrow keep the bookkeeping
    assert o["full"] == 0 and np.array_equal(o["runs"], np.r_[3, np.arange(n - 16, n)])
    st = fr.resident_download(h, 0, n, T.state_stride)
    res, _ = PK.evaluate(pt, T, st, 0, 0, threads=8)
    assert np.array_equal(o["head"], PK.compact_events(T, res)[0][o["runs"]])
    fr.resident_destroy(h)


def test_a_narrow_below_the_last_ticks_run_count_makes_later_ticks_over_them_full(fr):
    """the result records at or above the narrow's n_runs were truncated unchecked: a changed-only tick over them lists every run
    and a touched tick over them is full, although nothing changed"""
    rng = np.random.default_rng(79)
    n, k = 900, 100
    _, Lw, Ln, st = _batch(fr, rng, "256-32", n)
    # narrowed over all n runs, the same batches stay incremental: nothing changed, nothing listed
    hA, hB = fr.resident_create(Lw, n), fr.resident_create(Lw, n)
    for h in (hA, hB):
        fr.resident_upload(h, 0, st)
    fr.resident_tick_compact(hA, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    fr.resident_tick_touched(hB, n, NONE, n, BIG)
    for h in (hA, hB):
        fr.resident_narrow(h, Ln, n)
    assert fr.resident_tick_compact(hA, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)[4] == 0
    o = fr.resident_tick_touched(hB, n, NONE, n, BIG)
    assert o["full"] == 0 and o["n_evaluated"] == 0
    hA2, hB2 = fr.resident_create(Lw, n), fr.resident_create(Lw, n)   # narrowed over n - k runs, then ticked over all n
    for h in (hA2, hB2):
        fr.resident_upload(h, 0, st)
    fr.resident_tick_compact(hA2, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    fr.resident_tick_touched(hB2, n, NONE, n, BIG)
    for h in (hA2, hB2):
        fr.resident_narrow(h, Ln, n - k)
    _, _, _, _, listed = fr.resident_tick_compact(hA2, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    assert listed == n
    o = fr.resident_tick_touched(hB2, n, NONE, n, BIG)
    assert o["full"] == 1 and o["n_listed"] == n
    for h in (hA, hB, hA2, hB2):
        fr.resident_destroy(h)
