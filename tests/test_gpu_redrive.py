"""bf_resident_redrive: operator redrives of live runs, reset on the device.  Every case runs a resident batch whose runs of several
Stories are interleaved, redrives some of them (from main, compensation and finally steps, whole runs, duplicates and overlapping
sets on one run, stale slots, a run on a dropped slot), and checks the records byte for byte against packing the object-level
reset and against the delta path, then the ticks that follow: touched, changed-only, compact, and bf_schedule refused."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200 import host as H
from bobrapet_b200.records import make_layout
from oracle import packed as PK
from tests import migration as M
from tests import packing as P
from tests import redrive as RD
from tests.test_gpu_migrate import _sched
from tests.test_redrive_oracle import _host_story, child_codes, fill_mirror

pytestmark = pytest.mark.gpu

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
# shape: (steps lo, hi, parallel steps per story, runs, layout fields)
SHAPES = {"cfg3": (200, 257, 0, 3000, 0),                       # phase only
          "cfg4": (200, 257, 6, 3000, ALL),                     # cond + decision, registered bits without a child area
          "cfg5": (513, 700, 20, 1200, ALL | A.F_CHILD)}        # S > 512, child nibbles and registered bits


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _req(run, slot, step):
    q = np.zeros(1, Frontier.REDRIVE_DTYPE)
    q["run"], q["slot"], q["step"] = run, slot, step
    return q


def _requests(rng, packed, story, slots, n):
    """-> REDRIVE_DTYPE requests over runs [0, n): from a step of each group, whole runs, duplicates, two overlapping sets on one
    run, stale slots (the slot of another Story) and the run on the dropped slot (story 0)"""
    out = []
    groups = [(ps.flags.astype(np.int64) >> A.SF_GROUP_SHIFT) & 3 for ps in packed]
    live = np.nonzero(story[:n] != 0)[0]
    for r in rng.choice(live, size=len(live) // 8, replace=False):
        s = int(story[r])
        g = int(rng.choice([0, 0, 1, 2]))
        cand = np.nonzero(groups[s] == g)[0]
        step = A.REDRIVE_ALL if rng.random() < 0.1 or not cand.size else int(rng.choice(cand))
        out.append(_req(r, slots[s], step))
        if rng.random() < 0.1:
            out.append(out[-1].copy())                                              # a duplicate
        if rng.random() < 0.1:
            out.append(_req(r, slots[s], int(rng.integers(0, packed[s].S))))         # an overlapping set on the same run
        if rng.random() < 0.05:
            other = 1 + (s % (len(packed) - 1))                                     # a stale request: another Story's slot
            out.append(_req(r, slots[other], int(rng.integers(0, packed[other].S))))
    dead = np.nonzero(story[:n] == 0)[0]
    out.append(_req(int(dead[0]), slots[1], 0))                                     # its run holds the dropped slot
    req = np.concatenate(out)
    return req[rng.permutation(req.shape[0])]


@pytest.mark.parametrize("shape", list(SHAPES))
def test_redrive(fr, shape):
    rng = np.random.default_rng({"cfg3": 31, "cfg4": 32, "cfg5": 33}[shape])
    lo, hi, n_par, n, fields = SHAPES[shape]
    gens = [RD.random_story(rng, "t%d-" % k, int(rng.integers(lo, hi)), n_par) for k in range(7)]
    packed = [RD.packed_story(s) for s in gens]
    stories = [RD.oracle_story(s) for s in gens]
    slots = [int(s) for s in fr.put_topologies(P.topology_set(packed))]
    fr.drop_topology(slots[0])                                   # story 0's runs hold a dropped slot
    pt = PK.PackedTopologies(P.topology_set(packed[1:]), slots[1:])
    child = max(p.child_nibbles() for p in packed) if fields & A.F_CHILD else 0
    L = make_layout(max(p.S for p in packed), child, fields)
    cap = n + 64
    story = rng.integers(1, 7, cap)
    story[rng.random(cap) < 0.02] = 0                           # a few runs on the dropped slot
    story[5] = 0
    states = [M.random_state(rng, packed[s]) for s in story]
    tt = rng.random(cap) < 0.5
    rflags = np.array([f | (A.RF_TOPOLOGY_TERMINATED if t else 0) for f, t in
                       zip(rng.choice([0, A.RF_FAIL_FAST, A.RF_FAIL_FAST | A.RF_REALTIME], size=cap), tt)], np.uint8)
    rec0 = M.pack_by_name(L, packed, story, slots, states, rflags)
    hT, hD, hC = (fr.resident_create(L, cap) for _ in range(3))
    try:
        for h in (hT, hD, hC):
            fr.resident_upload(h, 0, rec0)
        assert fr.resident_tick_touched(hT, n, NONE, n, BIG)["full"] == 1
        fr.resident_tick_compact(hC, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        fr.resident_eval(hT, L, n)                               # the snapshot bf_schedule would limit
        req = _requests(rng, packed, story, slots, n)
        status, applied = fr.resident_redrive(hT, req)
        holds = np.array([slots[story[q["run"]]] == q["slot"] and story[q["run"]] != 0 for q in req])
        assert np.array_equal(status.astype(bool), holds) and applied == int(holds.sum()) and 0 < applied < req.shape[0]
        # the records: pack(object-level reset), byte for byte
        want_states, want_flags = list(states), rflags.copy()
        by_run = {}
        for q in req[holds]:
            s = int(story[q["run"]])
            by_run.setdefault(int(q["run"]), []).append(None if q["step"] == A.REDRIVE_ALL else packed[s].names[int(q["step"])])
        for r, names in by_run.items():
            want_states[r], t = RD.by_name_reset(states[r], bool(tt[r]), stories[story[r]], packed[story[r]], names)
            assert not t
            want_flags[r] = rflags[r] & ~np.uint8(A.RF_TOPOLOGY_TERMINATED)
        want = M.pack_by_name(L, packed, story, slots, want_states, want_flags)
        got = fr.resident_download(hT, 0, cap, L.state_stride)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert bad.size == 0, bad[:10]
        # the delta path leaves the same records
        fr.resident_apply(hD, RD.redrive_deltas(fr.closure, L, {slots[k]: packed[k] for k in range(1, 7)}, req[holds], rflags))
        assert np.array_equal(fr.resident_download(hD, 0, cap, L.state_stride), want)
        # bf_schedule needs a new pass after the redrive
        with pytest.raises(A.FrontierError):
            fr.schedule(L, n, *_sched(n), global_limit=20000)
        # the touched tick: exactly the reset runs are evaluated, and those whose result changed are listed, as a changed-only
        # tick over the same records lists them
        live = story[:n] != 0
        prev, res = _evaluate(pt, L, rec0[:n], live), _evaluate(pt, L, want[:n], live)
        whead, wev, wl = PK.compact_events(L, res, prev)
        wst = np.concatenate(([0], np.cumsum((whead >> A.HEAD_COUNT_SHIFT) * ((whead & A.HEAD_LISTED) != 0)))).astype(np.int64)
        listed = np.nonzero(whead & A.HEAD_LISTED)[0]
        out = fr.resident_tick_touched(hT, n, NONE, n, BIG)
        assert out["full"] == 0 and out["n_evaluated"] == len(by_run)
        assert out["runs"].tolist() == listed.tolist() and set(listed.tolist()) <= set(by_run)
        assert np.array_equal(out["head"], whead[listed])
        assert np.array_equal(out["events"], np.concatenate([wev[wst[r]:wst[r + 1]] for r in listed] + [np.zeros(0, np.uint16)]))
        for lo_, hi_ in _ranges(sorted(by_run)):
            fr.resident_upload(hC, lo_, np.ascontiguousarray(want[lo_:hi_]))
        chead, cev, _, _, _ = fr.resident_tick_compact(hC, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        cst = np.concatenate(([0], np.cumsum(chead >> A.HEAD_COUNT_SHIFT))).astype(np.int64)
        assert np.array_equal(out["head"], chead[listed])
        assert np.array_equal(out["events"], np.concatenate([cev[cst[r]:cst[r + 1]] for r in listed] + [np.zeros(0, np.uint16)]))
        # a compact tick of the reset batch equals the packed oracle
        head, ev, n_ev, _, _ = fr.resident_tick_compact(hT, n, NONE, BIG)
        ahead, aev, _ = PK.compact_events(L, res)
        assert np.array_equal(head, ahead) and n_ev == len(aev) and np.array_equal(ev, aev)
        out = fr.resident_tick_touched(hT, n, NONE, n, BIG)
        assert out["full"] == 0 and out["n_evaluated"] == 0
    finally:
        for h in (hT, hD, hC):
            fr.resident_destroy(h)


def _evaluate(pt, L, state, live):
    """the packed oracle's result records; a run on a dead slot gets the summary word 0xFFFFFFFF (BF_HEAD_DEAD in the lists)"""
    res = np.zeros((state.shape[0], L.result_stride), np.uint8)
    res[:, 0:4] = 0xFF
    res[live], _ = PK.evaluate(pt, L, np.ascontiguousarray(state[live]), threads=8)
    return res


def _ranges(runs):
    out = []
    for r in runs:
        if out and out[-1][1] == r:
            out[-1][1] = r + 1
        else:
            out.append([r, r + 1])
    return out


def test_redrive_rejects_bad_arguments(fr):
    E, PA = A.STEP_ENGRAM, A.STEP_PARALLEL
    mk = lambda spec: [dict(name=nm, group=0, type=t, needs=[], branches=b) for nm, t, b in spec]
    small = RD.packed_story(mk([("a", E, 0), ("p", PA, 3), ("b", E, 0)]))
    big = RD.packed_story(mk([("s%d" % k, E, 0) for k in range(70)]))                 # more steps than the layout
    kids = RD.packed_story(mk([("a", E, 0), ("p", PA, 3), ("q", PA, 9)]))             # more child nibbles
    spare = RD.packed_story(mk([("a", E, 0)]))
    packed = [small, big, kids, spare]
    slots = [int(s) for s in fr.put_topologies(P.topology_set(packed))]
    fr.drop_topology(slots[3])
    L = make_layout(64, small.child_nibbles(), ALL | A.F_CHILD)
    n = 100
    rng = np.random.default_rng(4)
    states = [M.random_state(rng, small) for _ in range(n)]
    rec = M.pack_by_name(L, packed, np.zeros(n, int), slots, states, np.full(n, A.RF_TOPOLOGY_TERMINATED, np.uint8))
    h = fr.resident_create(L, n)
    try:
        fr.resident_upload(h, 0, rec)
        good = _req(0, slots[0], 1)
        bad = []
        for run, slot, step, res in ((n, slots[0], 1, 0), (1, slots[3], 0, 0), (1, 9999, 0, 0), (1, slots[0], 3, 0),
                                     (1, slots[1], 0, 0), (1, slots[2], 0, 0), (1, slots[0], 0, 7)):
            q = _req(run, slot, step)
            q["reserved"] = res
            bad.append(q)
        want = [A.BF_EINVAL, A.BF_ETOPO, A.BF_ETOPO, A.BF_EINVAL, A.BF_ETOPO, A.BF_ETOPO, A.BF_EINVAL]
        for q, st in zip(bad, want):
            with pytest.raises(A.FrontierError) as e:
                fr.resident_redrive(h, np.concatenate([good, q]))
            assert e.value.status == st, (q, e.value)
            assert np.array_equal(fr.resident_download(h, 0, n, L.state_stride), rec)
        with pytest.raises(A.FrontierError) as e:
            fr.resident_redrive(h + 7, good)
        assert e.value.status == A.BF_EINVAL
        assert fr.resident_redrive(h, np.zeros(0, Frontier.REDRIVE_DTYPE))[1] == 0
        assert np.array_equal(fr.resident_download(h, 0, n, L.state_stride), rec)
        st, applied = fr.resident_redrive(h, good)
        assert st.tolist() == [1] and applied == 1
        RD.reset_packed(L, rec[0], small, 1)
        assert np.array_equal(fr.resident_download(h, 0, n, L.state_stride), rec)
    finally:
        fr.resident_destroy(h)


def test_host_mirror_redrives_with_the_device():
    """bfh_batch_redrive in resident mode with pending deltas: the pending deltas of reset fields are dropped, the others still go
    up after the reset, and after bfh_batch_eval the device records equal the mirror's and pack(object-level reset)"""
    fr = Frontier(0)   # a fresh ctx: the batch's resident handle is its first, 0
    try:
        rng = np.random.default_rng(15)
        gens = [RD.random_story(rng, "a-", 180, 8), RD.random_story(rng, "b-", 120, 4)]
        packed = [RD.packed_story(s) for s in gens]
        stories = [RD.oracle_story(s) for s in gens]
        hs = [_host_story(s) for s in gens]
        slots = [hs[k].upload(fr) for k in range(2)]
        n = 500
        b = H.HostBatch(fr, max(p.S for p in packed), max(p.child_nibbles() for p in packed), ALL | A.F_CHILD, n)
        b.set_resident(True)
        story = rng.integers(0, 2, n)
        states = [child_codes(M.random_state(rng, packed[s])) for s in story]
        tt = rng.random(n) < 0.5
        for r in range(n):
            assert b.add_run(hs[story[r]], slots[story[r]]) == r
            fill_mirror(b, r, packed[story[r]], states[r], tt[r])
        b.eval()
        # pending deltas on a third of each run's steps, and on the TopologyTerminated flag
        for r in range(n):
            ps = packed[story[r]]
            pick = set(rng.choice(ps.names, size=ps.S // 3, replace=False).tolist())
            fresh = child_codes(M.random_state(rng, ps))
            for nm in pick:
                states[r]["codes"][nm] = fresh["codes"][nm]
                if nm in states[r]["par"]:
                    states[r]["par"][nm] = fresh["par"][nm]
            fill_mirror(b, r, ps, {"codes": {k: states[r]["codes"][k] for k in ps.names},
                                   "par": {k: states[r]["par"][k] for k in states[r]["par"]}}, not tt[r])
            tt[r] = not tt[r]
        assert b.traffic()[2] > 0
        runs = rng.choice(n, size=n // 3, replace=False)
        steps = [-1 if rng.random() < 0.2 else int(rng.integers(0, packed[story[r]].S)) for r in runs]
        b.redrive(runs, steps)
        out_states, out_flags = list(states), np.zeros(n, np.uint8)
        by_run = {}
        for r, s in zip(runs, steps):
            by_run.setdefault(int(r), []).append(None if s < 0 else packed[story[r]].names[s])
        for r in range(n):
            t = bool(tt[r])
            if r in by_run:
                out_states[r], t = RD.by_name_reset(states[r], t, stories[story[r]], packed[story[r]], by_run[r])
            out_flags[r] = A.RF_FAIL_FAST | (A.RF_TOPOLOGY_TERMINATED if t else 0)
        want = M.pack_by_name(b.L, packed, story, slots, out_states, out_flags)
        assert np.array_equal(b.state(), want)
        b.eval()   # the surviving deltas go up after the reset
        assert np.array_equal(fr.resident_download(0, 0, n, b.L.state_stride), b.state())
        b.close()
    finally:
        fr.close()
