"""Side-area resyncs of resident batches on the device (bf_resident_resync_areas) against the host model tests/resync_areas.py.

Each batch starts with non-default entries in every area it has (tests/lifecycle.seed_requests) and its device copy and host model
agree byte for byte.  The caller's areas are the batch's own, perturbed: deadlines and codes moved, slots dropped or added (due
ones among them, on both sides of fired_now), limiter inputs and deadlines changed, stops added, removed or changed.  Items,
drifted runs, n_written, and after the call every state record and every area over the whole capacity must be the model's; the
next touched tick evaluates exactly the runs a repair stopped, and bf_resident_schedule lists what the model lists."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import make_layout, pack_state
from tests import resync_areas as M
from tests import timers as T
from tests.lifecycle import RUNCTL, SCHED, TIMERS, area_sets, seeded, subset_name
from tests.test_gpu_run_areas import NOW, Env, Twin, schedule
from tests.test_host_resync_areas import _refusals

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
SETS = area_sets(ks=(1, 2, 5, 64))
SET_IDS = [subset_name(s, k) for s, k in SETS]
FIRED_NOW = NOW + 110


@pytest.fixture(scope="module")
def env():
    f = Frontier(0)
    yield Env(f)
    f.close()


class Batch:
    """a device batch and its model, as tests/test_gpu_run_areas.Twin without the schedule of its set-up (any size)"""
    check = Twin.check
    snapshot = Twin.snapshot

    def __init__(self, env, subset, K, n, cap):
        fr, L = env.fr, env.L
        self.env, self.fr = env, fr
        recs = env.records(n)
        m, (p, arms, q) = seeded(L, cap, subset, K, recs, env.S[0] - 1, NOW)
        self.m = m
        self.h = fr.resident_create(L, cap)
        fr.resident_upload(self.h, 0, recs)
        if m.sched is not None:
            fr.resident_sched(self.h)
            fr.resident_sched_put(self.h, p)
        if m.K:
            fr.resident_timers(self.h, m.K)
            fr.resident_timers_arm(self.h, arms)
        if m.runctl is not None:
            fr.resident_runctl(self.h)
            fr.resident_runctl_put(self.h, q)
        self.check("set-up")

    @property
    def n(self):
        return self.m.n


def perturb(rng, b, runs, share=0.5, fired_now=FIRED_NOW, areas=None, step_hi=None):
    """the batch's own areas for `runs` (or `areas`, the caller's), with a share of the rows changed -> (timers, sched, runctl),
    None where it has no area.  Slots the caller adds lie below step_hi (default: the layout's steps_max)"""
    t, s, c = M.device_areas(b, runs=runs) if areas is None else areas
    L = b.L
    for i, r in enumerate(runs):
        if rng.random() > share:
            continue
        if t is not None:
            e = {st: (d, cd) for st, d, cd in T.armed(b.timers[r])}
            for _ in range(int(rng.integers(1, 4))):
                k = int(rng.integers(0, 5))
                if k == 0 and e:                       # a deadline moves
                    st = list(e)[int(rng.integers(0, len(e)))]
                    e[st] = (e[st][0] + int(rng.integers(1, 9)), e[st][1])
                elif k == 1 and e:                     # a code changes
                    st = list(e)[int(rng.integers(0, len(e)))]
                    e[st] = (e[st][0], (e[st][1] + 1) % 4)
                elif k == 2 and e:                     # the caller lost a slot
                    e.pop(list(e)[int(rng.integers(0, len(e)))])
                elif len(e) < b.K:                     # the device lost one, due or not at FIRED_NOW
                    st = int(rng.integers(0, L.steps_max if step_hi is None else step_hi))
                    e.setdefault(st, (fired_now + int(rng.integers(-3, 4)), int(rng.integers(0, 4))))
            t[i] = T.canonical(e, b.K).view(M.SLOT_DTYPE)
        if s is not None and rng.random() < 0.5:
            f = M.SCHED_FIELDS[int(rng.integers(0, 5))]
            v = int(s[f][i]) + int(rng.integers(1, 5))
            s[f][i] = v if f == "priority" else (v + 2) % 15 if f == "run_phase" else v & 0xFFFFFFFF
        if c is not None:
            k = int(rng.integers(0, 4))
            if k == 0:
                c["story_deadline"][i] = NOW + int(rng.integers(0, 400))
            elif k == 1:
                c["drain_deadline"][i] = fired_now - int(rng.integers(0, 3)) if rng.random() < 0.5 else NOW + 900
            else:
                c["stop"][i] = int(rng.integers(0, 4))
    return t, s, c


def _same(got, want):
    assert got["n_items"] == want["items"].size, (got["n_items"], want["items"].size, got["items"][:6], want["items"][:6])
    assert got["items"].tobytes() == want["items"].tobytes(), next(
        (i, got["items"][i], want["items"][i]) for i in range(want["items"].size) if got["items"][i].tobytes() != want["items"][i].tobytes())
    assert got["drifted"].tolist() == want["drifted"].tolist() and got["n_drifted"] == want["drifted"].size


def _call(b, runs, arrays, check, **kw):
    t, s, c = arrays
    return b.fr.resident_resync_areas(b.h, b.n, runs=runs, timers=t, sched=s, runctl=c, fired_now=FIRED_NOW, check=check, **kw)


def _model(b, runs, arrays, check):
    t, s, c = arrays
    return M.resync(b.m, b.n, runs=runs, timers=t, sched=s, runctl=c, fired_now=FIRED_NOW, check=check)


@pytest.mark.parametrize("subset,K", SETS, ids=SET_IDS)
def test_check_then_repair_match_the_model(env, subset, K):
    rng = np.random.default_rng(subset * 100 + K)
    b = Batch(env, subset, K, 16, 24)
    if subset & SCHED:
        schedule([b])
    for runs in (None, np.array([1, 2, 3, 5, 8, 13], np.uint32)):
        arrays = perturb(rng, b.m, np.arange(b.n) if runs is None else runs)
        before = b.snapshot()
        _same(_call(b, runs, arrays, True), _model(b, runs, arrays, True))
        assert b.snapshot() == before, "a check changed something"
        want = _model(b, runs, arrays, False)
        got = _call(b, runs, arrays, False)
        _same(got, want)
        assert got["n_written"] == want["n_written"]
        b.check("repair")
        _same(_call(b, runs, arrays, True), _model(b, runs, arrays, True))   # kept stops, and inputs a timeout stop rewrote
        t = b.fr.resident_tick_touched(b.h, b.n, NONE_D, b.n, 1 << 16)
        if not t["full"]:
            assert t["n_evaluated"] == len(want["stopped"])
        if subset & SCHED:
            schedule([b])   # lists what the model lists after the repaired inputs and stops


@pytest.mark.parametrize("ctas", [1023, 1024, 1025, 2049])
def test_list_offsets_across_scan_chunks(env, ctas):
    """8 listed runs per CTA: the lists cross the scan's 1024-CTA chunks; the outputs staged (pageable) and truncated"""
    rng = np.random.default_rng(ctas)
    n = 8 * ctas
    b = Batch(env, TIMERS | SCHED | RUNCTL, 2, n, n)
    arrays = perturb(rng, b.m, np.arange(n), share=0.05)
    want = _model(b, None, arrays, True)
    _same(_call(b, None, arrays, True, items_cap=want["items"].size + 5), want)
    cut = _call(b, None, arrays, True, items_cap=want["items"].size // 3, drifted_cap=want["drifted"].size // 2)
    assert cut["n_items"] == want["items"].size and cut["items"].tobytes() == want["items"][:want["items"].size // 3].tobytes()
    assert cut["drifted"].tolist() == want["drifted"][:want["drifted"].size // 2].tolist()
    want = _model(b, None, arrays, False)
    got = _call(b, None, arrays, False, items_cap=want["items"].size)
    _same(got, want)
    assert got["n_written"] == want["n_written"]
    b.check("repair")


def test_pinned_outputs(env):
    rng = np.random.default_rng(3)
    b = Batch(env, TIMERS | SCHED | RUNCTL, 5, 300, 300)
    arrays = perturb(rng, b.m, np.arange(b.n))
    want = _model(b, None, arrays, False)
    nw = want["items"].size
    p_items = b.fr.alloc_pinned(16 * max(nw, 1)).view(Frontier.DRIFT_DTYPE)
    p_drift = b.fr.alloc_pinned(4 * b.n).view(np.uint32)
    t, s, c = arrays
    q = A.ResyncAreas(struct_size=ctypes.sizeof(A.ResyncAreas), n_runs=b.n, n=b.n, areas=A.RESYNC_ALL_AREAS, fired_now=FIRED_NOW,
                      timers=t.ctypes.data, sched=s.ctypes.data, runctl=c.ctypes.data, drifted_cap=b.n,
                      drifted=p_drift.ctypes.data, items=p_items.ctypes.data, items_cap=nw)
    assert b.fr._lib.bf_resident_resync_areas(b.fr._ctx, b.h, ctypes.byref(q)) == A.BF_OK
    assert q.n_items == nw and p_items[:nw].tobytes() == want["items"].tobytes()
    assert p_drift[:q.n_drifted].tolist() == want["drifted"].tolist() and q.n_written == want["n_written"]
    b.check("pinned repair")
    b.fr.free_pinned(p_items)
    b.fr.free_pinned(p_drift)


def test_refusals_change_nothing(env):
    b = Batch(env, TIMERS | SCHED | RUNCTL, 4, 24, 28)
    before = b.snapshot()
    for name, kw, want in _refusals(b.m):
        kw = dict(kw)
        n_runs = kw.pop("n_runs", b.n)
        assert M.resync(b.m, n_runs, **kw)["bad_run"] == want, name
        with pytest.raises(A.FrontierError) as e:
            b.fr.resident_resync_areas(b.h, n_runs, **kw)
        assert e.value.bad_run == want, name
        assert b.snapshot() == before, name
    t, s, c = M.device_areas(b.m)
    with pytest.raises(ValueError):   # a timer row narrower than the batch's K: the library would read past it
        b.fr.resident_resync_areas(b.h, b.n, timers=np.ascontiguousarray(t[:, :2]))
    for struct in (dict(areas=0x8), dict(flags=0x2), dict(areas=A.RESYNC_AREA_TIMERS), dict(n=b.n - 1),
                   dict(items_cap=4), dict(drifted_cap=4)):
        q = A.ResyncAreas(struct_size=ctypes.sizeof(A.ResyncAreas), n_runs=b.n, n=b.n, fired_now=A.TIMER_NONE)
        for k, v in struct.items():
            setattr(q, k, v)
        assert b.fr._lib.bf_resident_resync_areas(b.fr._ctx, b.h, ctypes.byref(q)) == A.BF_EINVAL, struct
    q = A.ResyncAreas(struct_size=ctypes.sizeof(A.ResyncAreas) - 8, n_runs=b.n, n=b.n)
    assert b.fr._lib.bf_resident_resync_areas(b.fr._ctx, b.h, ctypes.byref(q)) == A.BF_EINVAL
    for subset in (SCHED | RUNCTL, TIMERS | RUNCTL, TIMERS | SCHED):   # a selected area the batch has no area for
        lack = Batch(env, subset, 4, 24, 28)
        with pytest.raises(A.FrontierError):
            lack.fr.resident_resync_areas(lack.h, lack.n, timers=t, sched=s, runctl=c)
        lack.check("refused")
    assert b.snapshot() == before


def test_stuck_sleep_end_to_end():
    """a sleep's arm lost (the device has no slot, the annotation has a due one): the run stays Paused and no fire or tick
    lists it; the resync re-arms it, the next fire writes SUCCEED and the next tick readies the sleep's dependent"""
    fr = Frontier(0)
    try:
        ts = TopologySet([2], [1], [0, 0, 1], [0], [A.STEP_SLEEP, A.STEP_ENGRAM])
        slot = int(fr.put_topologies(ts)[0])
        L = make_layout(32, 0, A.F_DECISION)
        n = 4
        ph = np.zeros((n, 32), np.uint8)
        ph[:, 0] = A.PHASE_PAUSED
        rec = pack_state(L, np.full(n, slot, np.uint32), np.zeros(n, np.uint8), ph, np.zeros_like(ph), np.zeros_like(ph))
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, rec)
        fr.resident_timers(h, 2)
        fr.resident_tick_touched(h, n, NONE_D, n, 1024)
        fired = fr.resident_fire(h, n, 100)
        assert fired["n_fired"] == 0
        assert fr.resident_tick_touched(h, n, NONE_D, n, 1024)["n_listed"] == 0   # stuck: nothing lists run 2
        annot = np.full((1, 2), T.EMPTY, np.uint64)
        annot[0] = T.canonical({0: (90, A.DEC_SUCCEED)}, 2)
        got = fr.resident_resync_areas(h, n, runs=[2], timers=annot.view(M.SLOT_DTYPE), fired_now=100)
        assert got["items"].tolist() == [(2, 0, A.DRIFT_TIMER, 0, A.TIMER_NONE, 90)] and got["n_written"] == 1
        fired = fr.resident_fire(h, n, 101)
        assert fired["fired"].tolist() == [(2, 0, A.DEC_SUCCEED, 1)]
        t = fr.resident_tick_touched(h, n, NONE_D, n, 1024)
        assert t["runs"].tolist() == [2]
        steps = {int(e) & 0x3FF: int(e) >> 10 for e in t["events"]}
        assert steps.get(1, 0) & A.EVT_READY
        assert fr.resident_resync_areas(h, n, runs=[2], timers=annot.view(M.SLOT_DTYPE), fired_now=101, check=True)["n_items"] == 0
    finally:
        fr.close()
