"""bf_resident_reshape: a live resident batch grows its capacity and layout in place.  The records are checked byte for byte
against packing every old code again at the new layout (tests/reshape.py), and the ticks that follow against a fresh batch
created at the new layout, a twin taking changed-only ticks, and the packed oracle."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200 import host as H
from bobrapet_b200.records import make_layout
from oracle import packed as PK
from tests import migration as M
from tests import randgen
from tests import reshape as RS

pytestmark = pytest.mark.gpu

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _deltas(rng, L, n, k):
    """k coalesced deltas on about k / 3 runs, over every field the layout has"""
    runs = rng.choice(n, size=k // 3 + 1, replace=False)
    fields = [A.DELTA_PHASE] * 4 + [A.DELTA_RUN_FLAGS, A.DELTA_REGISTERED]
    fields += [A.DELTA_COND] * (L.off_cond != A.OFF_NONE) + [A.DELTA_DECISION] * (L.off_decision != A.OFF_NONE)
    fields += [A.DELTA_CHILD] * (L.off_child != A.OFF_NONE and L.child_nibbles > 0)
    recs = {}
    for _ in range(k):
        r, f = int(rng.choice(runs)), int(rng.choice(fields))
        if f == A.DELTA_PHASE:
            idx, code = int(rng.integers(0, 32 * L.words)), int(rng.choice([0, 1, 2, 3, 3, 4, 9, 13, 14]))
        elif f in (A.DELTA_COND, A.DELTA_DECISION):
            idx, code = int(rng.integers(0, 32 * L.words)), int(rng.integers(0, 4))
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


def _batch(fr, rng, s_old, fields, parallel, n):
    """random topologies of at most s_old steps and n runs packed at a layout of exactly s_old steps -> (pt, Lo, records)"""
    ts = randgen.random_topologies(rng, 12, max(2, s_old // 2), s_old, max_deg=4, parallel=parallel, fill=0.5)
    slots = fr.put_topologies(ts)
    L0, st0, _ = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
    Lo = make_layout(s_old, L0.child_nibbles, L0.fields)
    return PK.PackedTopologies(ts, slots), Lo, RS.reshape_state(L0, Lo, st0, n)


def _listed(head, events):
    """runs, heads and events of the listed runs of a compact tick"""
    runs = np.nonzero(head & A.HEAD_LISTED)[0]
    return runs, head[runs], events


# (steps_max old -> new, fields old -> added, child nibbles added, capacity factor, parallel steps)
CASES = {"none-cond": (64, 64, 0, COND, 0, 1, False),
         "none-decision": (64, 64, 0, DEC, 0, 2, False),
         "none-child": (64, 64, 0, CHILD, 24, 1, False),
         "none-all-31-33": (31, 33, 0, COND | DEC | CHILD, 9, 2, False),
         "out-added": (256, 256, COND, A.F_OUT_NEEDS_COND | A.F_OUT_FAIL, 0, 1, False),
         "decision-added": (128, 160, COND | OUT, DEC, 0, 1, True),
         "64-256": (64, 256, OUT, 0, 0, 1, True),
         "256-288": (256, 288, COND | DEC | OUT, 0, 16, 2, True),
         "512-544": (512, 544, COND | DEC | OUT, 0, 5, 2, True)}


@pytest.mark.parametrize("flags", [0, A.EVAL_FIXPOINT], ids=["single", "fixpoint"])
@pytest.mark.parametrize("case", list(CASES))
def test_reshape_records_and_the_ticks_that_follow(fr, case, flags):
    s_old, s_new, f_old, f_add, grow, mult, parallel = CASES[case]
    rng = np.random.default_rng(list(CASES).index(case) * 10 + (flags != 0))
    n = 1500
    pt, Lo, st = _batch(fr, rng, s_old, f_old, parallel, n)
    Ln = make_layout(s_new, Lo.child_nibbles + grow, Lo.fields | f_add)
    cap = n * mult
    hA, hB = fr.resident_create(Lo, n), fr.resident_create(Lo, n)   # A: touched ticks; B: its twin, changed-only ticks
    fr.resident_upload(hA, 0, st)
    fr.resident_upload(hB, 0, st)
    assert fr.resident_tick_touched(hA, n, NONE, n, BIG, flags=flags)["full"] == 1
    fr.resident_tick_compact(hB, n, NONE, BIG, flags=flags | A.EVAL_CHANGED_ONLY)
    prev, _ = PK.evaluate(pt, Lo, st, flags, 0, threads=8)          # the current result records of both
    d1 = _deltas(rng, Lo, n, 90)                                      # touched before the reshape
    fr.resident_apply(hA, d1)
    fr.resident_apply(hB, d1)
    st1 = fr.resident_download(hA, 0, n, Lo.state_stride)
    for h in (hA, hB):
        fr.resident_reshape(h, Ln, cap)
    want = RS.reshape_state(Lo, Ln, st1, cap)
    for h in (hA, hB):
        assert np.array_equal(fr.resident_download(h, 0, cap, Ln.state_stride), want)
    # a fresh batch at the new layout, given the same codes
    hC = fr.resident_create(Ln, cap)
    fr.resident_upload(hC, 0, want)
    d2 = _deltas(rng, Ln, n, 90)
    oA = fr.resident_tick_touched(hA, n, d2, n, BIG, flags=flags)
    bhead, bev, _, _, _ = fr.resident_tick_compact(hB, n, d2, BIG, flags=flags | A.EVAL_CHANGED_ONLY)
    chead, cev, _, _, _ = fr.resident_tick_compact(hC, n, d2, BIG, flags=flags)
    st2 = fr.resident_download(hA, 0, cap, Ln.state_stride)
    assert np.array_equal(st2, fr.resident_download(hB, 0, cap, Ln.state_stride))
    assert np.array_equal(st2, fr.resident_download(hC, 0, cap, Ln.state_stride))
    res, _ = PK.evaluate(pt, Ln, st2[:n], flags, 0, threads=8)
    whead, wev, _ = PK.compact_events(Ln, res)
    assert np.array_equal(chead, whead) and np.array_equal(cev, wev)
    # the changed-only twin compares with its result records re-laid by the reshape
    ohead, oev, _ = PK.compact_events(Ln, res, RS.reshape_result(Lo, Ln, prev, n))
    assert np.array_equal(bhead, ohead) and np.array_equal(bev, oev)
    runs, heads, events = _listed(bhead, bev)
    if (Ln.fields & ~Lo.fields) & (OUT | DEC):   # any result may change (PENDING decisions, new masks): a full tick
        assert oA["full"] == 1 and np.array_equal(oA["head"], whead) and np.array_equal(oA["events"], wev)
    else:                                # exactly the runs touched before and after the reshape, listed as the twin lists them
        assert oA["full"] == 0
        assert oA["n_evaluated"] == len(set(d1["run"].tolist()) | set(d2["run"].tolist()))
        assert np.array_equal(oA["runs"], runs) and np.array_equal(oA["head"], heads) and np.array_equal(oA["events"], events)
    # dense ticks: the reshaped batch and the fresh one give the oracle's records
    for h in (hA, hC):
        got, _ = fr.resident_tick(h, Ln, n, NONE, flags=flags)
        assert np.array_equal(got, res)
    for h in (hA, hB, hC):
        fr.resident_destroy(h)


def test_reshape_keeps_the_touched_bookkeeping(fr):
    rng = np.random.default_rng(41)
    n = 1200
    pt, Lo, st = _batch(fr, rng, 96, COND | DEC | OUT, True, n)
    Ln = make_layout(160, Lo.child_nibbles + 8, Lo.fields)
    hA, hB = fr.resident_create(Lo, n), fr.resident_create(Lo, n)
    for h in (hA, hB):
        fr.resident_upload(h, 0, st)
    fr.resident_tick_touched(hA, n, NONE, n, BIG)
    fr.resident_tick_compact(hB, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    for h in (hA, hB):
        fr.resident_reshape(h, Ln, n + 100)
    # nothing touched since the last tick: nothing evaluated, nothing listed
    o = fr.resident_tick_touched(hA, n, NONE, n, BIG)
    assert o["full"] == 0 and o["n_evaluated"] == 0 and o["n_listed"] == 0
    _, _, _, _, n_listed = fr.resident_tick_compact(hB, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
    assert n_listed == 0
    # bf_schedule may follow the tick, and needs a new pass after a reshape, as after an upload
    from oracle import limiters as LM
    sched = np.zeros(n, dtype=LM.SCHED_RUN_DTYPE)
    sched["run_phase"], sched["queued_elapsed_s"] = 2, LM.NONE_U32
    limits = (np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32))
    fr.resident_eval(hA, Ln, n)
    fr.schedule(Ln, n, sched, *limits, global_limit=100)
    fr.resident_reshape(hA, Ln, n + 200)
    with pytest.raises(A.FrontierError):
        fr.schedule(Ln, n, sched, *limits, global_limit=100)
    # runs uploaded into the added capacity are listed by the next touched tick, which stays incremental
    more = RS.reshape_state(Lo, Ln, st[:100], 100)
    fr.resident_upload(hA, n, more)
    o = fr.resident_tick_touched(hA, n + 100, NONE, n + 100, BIG)
    assert o["full"] == 0 and np.array_equal(o["runs"], np.arange(n, n + 100))
    res, _ = PK.evaluate(pt, Ln, fr.resident_download(hA, 0, n + 100, Ln.state_stride), 0, 0, threads=8)
    whead, _, _ = PK.compact_events(Ln, res)
    assert np.array_equal(o["head"], whead[n:])
    for h in (hA, hB):
        fr.resident_destroy(h)


def test_reshape_rejections_change_nothing(fr):
    rng = np.random.default_rng(43)
    n = 800
    _, Lo, st = _batch(fr, rng, 100, COND | A.F_OUT_SKIP_DEP, True, n)
    hA, hB = fr.resident_create(Lo, n), fr.resident_create(Lo, n)   # B never sees the rejected calls
    for h in (hA, hB):
        fr.resident_upload(h, 0, st)
        fr.resident_tick_touched(h, n, NONE, n, BIG)
    d = _deltas(rng, Lo, n, 60)
    for h in (hA, hB):
        fr.resident_apply(h, d)
    c, f = Lo.child_nibbles, Lo.fields
    dropped = make_layout(128, c, f)
    dropped.off_skip_dep = A.OFF_NONE  # passes check_layout, but drops a field the batch has
    bad_words = make_layout(128, c, f)
    bad_words.words = 3
    for L, cap, status in [(make_layout(100, c, f), n - 1, A.BF_EINVAL),          # fewer runs
                           (make_layout(99, c, f), n, A.BF_EINVAL),               # fewer steps
                           (make_layout(100, c - 1, f), n, A.BF_EINVAL),          # a smaller child area
                           (make_layout(100, c, f & ~COND), n, A.BF_EINVAL),      # a dropped input field
                           (make_layout(100, c, f & ~A.F_OUT_SKIP_DEP), n, A.BF_EINVAL),   # a dropped output field
                           (dropped, n, A.BF_EINVAL), (bad_words, n, A.BF_EINVAL),
                           (make_layout(1024, c, f | DEC), 0xFFFFFFFF, A.BF_ENOMEM)]:      # more than the device holds
        with pytest.raises(A.FrontierError) as e:
            fr.resident_reshape(hA, L, cap)
        assert e.value.status == status, (L.as_dict(), cap)
        assert np.array_equal(fr.resident_download(hA, 0, n, Lo.state_stride), fr.resident_download(hB, 0, n, Lo.state_stride))
    with pytest.raises(A.FrontierError) as e:
        fr.resident_reshape(hA + 7, make_layout(128, c, f), n)   # an unknown handle
    assert e.value.status == A.BF_EINVAL
    oA = fr.resident_tick_touched(hA, n, NONE, n, BIG)
    oB = fr.resident_tick_touched(hB, n, NONE, n, BIG)
    for k in ("full", "n_listed", "n_evaluated", "n_events"):
        assert oA[k] == oB[k], k
    for k in ("runs", "head", "events"):
        assert np.array_equal(oA[k], oB[k]), k
    for h in (hA, hB):
        fr.resident_destroy(h)


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


def _fill(b, r, ps, st):
    for i, nm in enumerate(ps.names):
        ph, cd, dc = st["codes"][nm]
        b.set_phase_code(r, i, ph)
        b.set_cond(r, i, cd)
        b.set_decision(r, i, dc)
    for q, stp in enumerate(ps.par_steps):
        on, kids = st["par"][ps.names[stp]]
        b.register_children(r, q, on)
        for br, code in enumerate(kids):
            b.set_child_phase(r, q, br, A.PHASE_NAMES[min(code, 13)])


def test_migrate_and_redrive_after_a_reshape(fr):
    """the motivating flows: an edited Story outgrows steps_max (migrate is refused, then succeeds after a reshape), and runs in
    the added capacity take uploads and redrives; the C++ mirror reshaped alongside holds the same records"""
    rng = np.random.default_rng(47)
    old = M.random_story(rng, "a-", 30, 2)
    new = M.edit_story(rng, old, "a-e") + [dict(name="x%d" % k, group=0, type=A.STEP_ENGRAM, needs=[], branches=0) for k in range(12)]
    ps_old, ps_new = M.story_from_steps(old), M.story_from_steps(new)
    assert ps_old.S <= 32 < ps_new.S
    hs_old, hs_new = _host_story(old), _host_story(new)
    so, sn = hs_old.upload(fr), hs_new.upload(fr)
    fields = COND | DEC | CHILD | OUT
    c_old, c_new = ps_old.child_nibbles(), max(ps_old.child_nibbles(), ps_new.child_nibbles()) + 3
    n = 300
    mr = H.HostBatch(None, 32, c_old, fields, n)
    try:
        for r in range(n):
            mr.add_run(hs_old, so)
            _fill(mr, r, ps_old, M.random_state(rng, ps_old))
        Lo = A.Layout.from_buffer_copy(mr.L)
        h = fr.resident_create(Lo, n)
        fr.resident_upload(h, 0, mr.state().copy())
        fr.resident_tick_touched(h, n, NONE, n, BIG)
        smap = hs_old.migration_map(hs_new)
        with pytest.raises(A.FrontierError) as e:
            fr.resident_migrate(h, so, sn, smap, n)
        assert e.value.status == A.BF_ETOPO
        Ln = make_layout(64, c_new, fields)
        fr.resident_reshape(h, Ln, 2 * n)
        mr.reshape(64, c_new, fields, 2 * n)
        assert mr.L.as_dict() == Ln.as_dict()
        assert np.array_equal(fr.resident_download(h, 0, n, Ln.state_stride), mr.state())
        assert fr.resident_migrate(h, so, sn, smap, n) == n
        assert mr.migrate(hs_old, hs_new, so, sn) == n
        assert np.array_equal(fr.resident_download(h, 0, n, Ln.state_stride), mr.state())
        for r in range(n, 2 * n):   # runs of the larger Story in the added capacity
            mr.add_run(hs_new, sn)
            _fill(mr, r, ps_new, M.random_state(rng, ps_new))
        fr.resident_upload(h, n, mr.state()[n:].copy())
        runs = np.array([n, n + 1, n + 7, 2 * n - 1], np.uint32)
        steps = np.array([-1, 0, 5, ps_new.S - 1], np.int32)
        req = np.zeros(len(runs), dtype=Frontier.REDRIVE_DTYPE)
        req["run"], req["slot"] = runs, sn
        req["step"] = np.where(steps < 0, A.REDRIVE_ALL, steps).astype(np.uint32)
        status, applied = fr.resident_redrive(h, req)
        assert applied == len(runs)
        mr.redrive(runs, steps)
        assert np.array_equal(fr.resident_download(h, 0, 2 * n, Ln.state_stride), mr.state())
        # the reshaped batch ticks as a fresh batch holding the same records
        hF = fr.resident_create(Ln, 2 * n)
        fr.resident_upload(hF, 0, mr.state().copy())
        got, _ = fr.resident_tick(h, Ln, 2 * n, NONE)
        want, _ = fr.resident_tick(hF, Ln, 2 * n, NONE)
        assert np.array_equal(got, want)
        fr.resident_destroy(h)
        fr.resident_destroy(hF)
    finally:
        mr.close()


def test_mirror_reshape_in_resident_mode_keeps_pending_deltas(fr):
    rng = np.random.default_rng(53)
    steps = M.random_story(rng, "m-", 28, 2)
    ps = M.story_from_steps(steps)
    hs = _host_story(steps)
    slot = hs.upload(fr)
    fields = COND | DEC | CHILD | A.F_OUT_SKIP_DEP
    c = ps.child_nibbles()
    n = 120
    states = [M.random_state(rng, ps) for _ in range(n)]
    a = H.HostBatch(fr, 32, c, fields, n)
    b = H.HostBatch(fr, 96, c + 9, fields | OUT, 2 * n)
    try:
        a.set_resident(True)
        for x in (a, b):
            for r in range(n):
                x.add_run(hs, slot)
                _fill(x, r, ps, states[r])
        a.eval()   # every run on the device
        for x in (a, b):   # pending deltas at the time of the reshape
            for r in range(0, n, 7):
                x.set_phase_code(r, 3, 2)
                x.register_children(r, 1, True)
        pending = a.traffic()[2]
        assert pending > 0
        a.reshape(96, c + 9, fields | OUT, 2 * n)
        assert a.traffic()[2] == pending and np.array_equal(a.state(), b.state())
        a.eval()
        b.eval()
        assert np.array_equal(a.state(), b.state()) and np.array_equal(a.result(), b.result())
        assert a.traffic()[2] == 0
    finally:
        a.close()
        b.close()
