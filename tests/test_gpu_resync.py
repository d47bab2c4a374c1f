"""Resyncs of resident batches on the device (bf_resident_resync) against the host model tests/resync.py.

Random batches with gates, sleeps, waits, parallel steps, fail-fast runs, stopped runs and runs on a dropped slot go through the
per-tick loop (upload, fire, touched tick, schedule, commit).  The records a batcher packs from the cluster afterwards (the phases
after the pass's rewrites, no decision on a terminal step, the device's cond codes and child phases) list nothing; perturbed
records list, byte for byte, what the model lists; a repair leaves the records the model gives and touches only what it wrote."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import _pack_planes
from tests import randgen
from tests import resync as M
from tests.test_gpu_commit import BIG, TABLES
from tests.test_host_commit import no_stops

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
F = A.resync_field


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _looped(fr, rng, S, fields, n, ticks=4, parallel=True):
    """a batch of n runs of random topologies (one dropped after the upload), with timers, limiter inputs and run control, after
    `ticks` rounds of fire -> touched tick -> schedule -> commit; parallel=False: no parallel steps, so no child area.
    -> (topos of the live slots, L, handle)"""
    ts = no_stops(randgen.random_topologies(rng, 10, max(2, S // 2), S, max_deg=4, parallel=parallel, fill=0.5))
    slots = fr.put_topologies(ts)
    L, st, topo = randgen.random_state(rng, ts, slots, n, fields | A.F_ALL_OUT, phase_mix="progress")
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    keep = np.ones(ts.count, bool)
    keep[ts.count - 1] = False
    fr.drop_topology(int(slots[-1]))   # its runs hold a dropped slot
    fr.resident_timers(h, 2)
    fr.resident_sched(h)
    fr.resident_runctl(h)
    runs = np.sort(rng.choice(n, size=n // 3, replace=False))
    tq = np.zeros(runs.size, dtype=Frontier.TIMER_DTYPE)
    tq["run"], tq["step"] = runs, rng.integers(0, 2, runs.size)
    tq["code"] = rng.choice([A.DEC_SUCCEED, A.DEC_FAIL, A.DEC_TIMED_OUT], runs.size) if L.off_decision != A.OFF_NONE else A.DEC_PENDING
    tq["deadline"] = rng.integers(0, 12, runs.size)
    fr.resident_timers_arm(h, tq)
    q = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
    q["run"], q["story_key"], q["queue_key"] = np.arange(n), np.arange(n) % 4, np.arange(n) % 3
    q["priority"], q["queued_since"], q["run_phase"] = np.arange(n) % 5, A.SCHED_NONE, A.PHASE_RUNNING
    fr.resident_sched_put(h, q)
    c = np.zeros(runs.size, dtype=Frontier.RUNCTL_PUT_DTYPE)
    c["run"], c["story_deadline"], c["drain_deadline"] = runs, rng.integers(5, 40, runs.size), A.TIMER_NONE
    c["stop"] = np.where(np.arange(runs.size) % 7 == 0, A.STOP_HOST, A.STOP_NONE)
    fr.resident_runctl_put(h, c)
    for k in range(ticks):
        fr.resident_fire(h, n, 4 * k)
        d = np.zeros(30, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"] = rng.choice(n, size=30, replace=False), rng.integers(0, 2, 30)
        d["field"], d["code"] = A.DELTA_PHASE, rng.choice([A.PHASE_RUNNING, A.PHASE_SUCCEEDED, A.PHASE_FAILED], 30)
        fr.resident_tick_touched(h, n, d, n, n * 1024)
        fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], TABLES, 4 * k)
        fr.resident_commit(h, n)
    return M.Topos(_subset(ts, keep), slots[keep]), L, h


def _subset(ts, keep):
    """the TopologySet of the topologies `keep` selects"""
    from bobrapet_b200.frontier import TopologySet
    S, E, P = ts.S.astype(np.int64), ts.E.astype(np.int64), ts.P.astype(np.int64)
    rp0, ci0, sf0, pd0 = (np.concatenate(([0], np.cumsum(x)[:-1])) for x in (S + 1, E, S, P))
    idx = np.flatnonzero(keep)
    rp = np.concatenate([ts.row_ptr[rp0[i]:rp0[i] + S[i] + 1] for i in idx])
    ci = np.concatenate([ts.col_idx[ci0[i]:ci0[i] + E[i]] for i in idx]) if E[idx].sum() else np.zeros(0, np.uint16)
    sf = np.concatenate([ts.step_flags[sf0[i]:sf0[i] + S[i]] for i in idx])
    par = np.concatenate([ts.parallel[pd0[i]:pd0[i] + P[i]] for i in idx]) if P[idx].sum() else None
    return TopologySet(list(S[idx]), list(E[idx]), rp, ci, sf, list(P[idx]), par, ts.allow_bits)


def cluster_view(L, topos, state, runctl):
    """what a batcher packs from StoryRun.status and the StepRuns: the phases after the pass's rewrites (those bf_resident_status
    reports), no decision (PENDING) on a terminal step, the device's cond codes, child phases and registered bits, the run's own
    flags byte (a stopped run's saved one); a dead slot's record as the device holds it"""
    out = state.copy()
    post = M.post_phases(L, topos, list(state))
    W = L.words
    for r, ph in enumerate(post):
        if runctl["stop"][r]:
            out[r][4] = runctl["saved_flags"][r]
        if ph is None:
            continue
        codes = np.zeros((1, 32 * W), np.uint8)
        codes[0, :ph.size] = ph
        out[r][L.off_phase:L.off_phase + 16 * W] = _pack_planes(codes, W, 4)[0]
        if L.off_decision != A.OFF_NONE:
            dec = M._codes2(state[r], L.off_decision, W, 32 * W)[None, :].copy()
            dec[0, :ph.size][np.isin(ph, M.TERMINAL)] = 0
            out[r][L.off_decision:L.off_decision + 8 * W] = _pack_planes(dec, W, 2)[0]
    return out


def perturb(rng, L, view, slots, k):
    """k random runs of the view with one code of a random field changed (or another live slot)"""
    out = view.copy()
    W = L.words
    for r in rng.choice(view.shape[0], size=k, replace=False):
        f = int(rng.integers(0, 7))
        if f == A.DELTA_PHASE or (f == A.DELTA_COND and L.off_cond != A.OFF_NONE) or (f == A.DELTA_DECISION and L.off_decision != A.OFF_NONE):
            off, planes = {A.DELTA_PHASE: (L.off_phase, 4), A.DELTA_COND: (L.off_cond, 2), A.DELTA_DECISION: (L.off_decision, 2)}[f]
            b = int(rng.integers(0, 32 * W * planes))
            out[r][off + b // 8] ^= 1 << (b % 8)
        elif f == A.DELTA_CHILD and L.off_child != A.OFF_NONE:
            out[r][L.off_child + int(rng.integers(0, (L.child_nibbles + 1) // 2))] ^= int(rng.integers(1, 256))
        elif f == A.DELTA_RUN_FLAGS:
            out[r][4] ^= 1 << int(rng.integers(0, 3))
        elif f == A.DELTA_REGISTERED:
            out[r][8 + int(rng.integers(0, 8))] ^= 1 << int(rng.integers(0, 8))
        else:
            out[r][:4] = np.frombuffer(np.uint32(slots[int(rng.integers(0, len(slots)))]).tobytes(), np.uint8)
    return out


def _same_items(got, want):
    assert got["n_items"] == want.size, (got["n_items"], want.size, got["items"][:8], want[:8])
    assert got["items"].tobytes() == want.tobytes(), next(
        (i, got["items"][i], want[i]) for i in range(want.size) if got["items"][i].tobytes() != want[i].tobytes())


PLANES = [0, A.F_COND | A.F_DECISION]
# Runs whose cluster view drifts from the device, by (S, planes).  Every other run must list nothing.  "tt-then-ff": a realtime,
# fail-fast run with a terminated topology; the pass's stage I fails its live main steps (dag.go:436-464) after the fail-fast
# marking, so the Failed codes the cluster persists make the next pass skip the main steps that were still absent, which a pass
# over the device's record, where those Failed codes were never stored, does not (DESIGN.md, "Resyncs").
PINNED = {   # (S, planes, parallel)
    (32, 0, True): {284: "tt-then-ff", 393: "tt-then-ff"},
    (32, 0, False): {322: "tt-then-ff"},
    (32, A.F_COND | A.F_DECISION, False): {198: "tt-then-ff", 397: "tt-then-ff", 467: "tt-then-ff"},
    (256, 0, False): {35: "tt-then-ff"},
}


@pytest.mark.parametrize("parallel", [True, False])
@pytest.mark.parametrize("planes", PLANES)
@pytest.mark.parametrize("S", [32, 256, 1024])
def test_cluster_view_lists_nothing_and_perturbations_match(fr, S, planes, parallel):
    rng = np.random.default_rng(S * 7 + planes + (0 if parallel else 1000))
    n = 500 if S < 1024 else 160
    topos, L, h = _looped(fr, rng, S, planes, n, parallel=parallel)
    assert (L.off_child != A.OFF_NONE) == parallel
    state = fr.resident_download(h, 0, n, L.state_stride)
    area = fr.resident_runctl_download(h, 0, n)
    view = cluster_view(L, topos, state, area)
    got = fr.resident_resync(h, n, view, check=True)
    pinned = PINNED.get((S, planes, parallel), {})
    assert set(got["drifted"].tolist()) == set(pinned), (got["drifted"], got["items"][:10])   # equivalent encodings: no drift
    for r in pinned:
        own = area["saved_flags"][r] if area["stop"][r] else state[r][4]
        assert own & 7 == A.RF_FAIL_FAST | A.RF_REALTIME | A.RF_TOPOLOGY_TERMINATED
        assert set(got["items"]["field"][got["items"]["run"] == r].tolist()) == {A.DELTA_PHASE}
    _same_items(got, M.compare(L, topos, state, view, np.arange(n), A.RESYNC_ALL_FIELDS, area))
    bad = perturb(rng, L, view, topos.slots, n // 10)
    want = M.compare(L, topos, state, bad, np.arange(n), A.RESYNC_ALL_FIELDS, area)
    assert want.size
    _same_items(fr.resident_resync(h, n, bad, check=True), want)
    runs = np.sort(rng.choice(n, size=n // 3, replace=False)).astype(np.uint32)
    for fields in (F(A.DELTA_PHASE) | F(A.DELTA_RUN_FLAGS), F(A.DELTA_COND) | F(A.DELTA_DECISION) | F(A.DELTA_CHILD) | F(A.DELTA_REGISTERED)):
        want = M.compare(L, topos, state[runs], bad[runs], runs, fields, area)
        got = fr.resident_resync(h, n, bad[runs], runs=runs, fields=fields, check=True)
        _same_items(got, want)
        assert got["drifted"].tolist() == np.unique(want["run"]).tolist()
    assert fr.resident_download(h, 0, n, L.state_stride).tobytes() == state.tobytes()


@pytest.mark.parametrize("S", [64, 1024])
def test_repair(fr, S):
    """after a repair the records are the model's; the next touched tick evaluates exactly the written runs and lists those whose
    result changed and every slot-drifted one; the next schedule lists the slot-drifted runs; stops, timers and limiter inputs
    stay; a check changes nothing at all"""
    rng = np.random.default_rng(S + 1)
    n = 400 if S < 1024 else 160
    topos, L, h = _looped(fr, rng, S, A.F_COND | A.F_DECISION, n)
    dense0, _ = fr.resident_tick(h, L, n, NONE_D)   # every run evaluated: no touched run is left
    fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], TABLES, 100)
    state = fr.resident_download(h, 0, n, L.state_stride)
    area = fr.resident_runctl_download(h, 0, n)
    timers = fr.resident_timers_download(h, 0, n, 2)
    sched = fr.resident_sched_download(h, 0, n)
    bad = perturb(rng, L, cluster_view(L, topos, state, area), topos.slots, n // 8)

    # a check changes nothing: records, areas, touch marks (the touched tick evaluates nothing), the schedule baseline
    chk = fr.resident_resync(h, n, bad, check=True)
    assert chk["n_items"] > 0 and chk["n_written"] == 0
    assert fr.resident_download(h, 0, n, L.state_stride).tobytes() == state.tobytes()
    t = fr.resident_tick_touched(h, n, NONE_D, n, n * 1024)
    assert t["full"] == 0 and t["n_evaluated"] == 0 and t["n_listed"] == 0
    assert fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], TABLES, 100)["parts"][0]["n_listed"] == 0

    items, drifted, want_state, want_area = M.resync(L, topos, state, bad, n, runctl=area)
    got = fr.resident_resync(h, n, bad)
    _same_items(got, items)
    assert got["drifted"].tolist() == drifted.tolist() and got["n_written"] == drifted.size == got["n_drifted"]
    after = fr.resident_download(h, 0, n, L.state_stride)
    assert after.tobytes() == want_state.tobytes()
    assert fr.resident_runctl_download(h, 0, n).tobytes() == want_area.tobytes()
    assert fr.resident_timers_download(h, 0, n, 2).tobytes() == timers.tobytes()
    assert fr.resident_sched_download(h, 0, n).tobytes() == sched.tobytes()
    assert fr.resident_resync(h, n, bad, check=True)["n_items"] == 0   # repaired

    t = fr.resident_tick_touched(h, n, NONE_D, n, n * 1024)
    assert t["full"] == 0 and t["n_evaluated"] == drifted.size
    sch = fr.resident_schedule([dict(handle=h, n_runs=n, runs_cap=n, events_cap=BIG)], TABLES, 100)["parts"][0]
    dense1, _ = fr.resident_tick(h, L, n, NONE_D)
    changed = [int(r) for r in drifted if dense0[r].tobytes() != dense1[r].tobytes()]
    slot = M.slot_drifted(items)
    assert set(t["runs"].tolist()) == set(changed) | set(slot.tolist())
    assert set(slot.tolist()) <= set(sch["runs"].tolist()) <= set(drifted.tolist())

    # a full tick after the resync gives what a full tick after an upload of the caller's records gives: the same result records
    # for the repaired runs, and for the others the same but for BF_SUM_PHASE_CHANGED (a pass over the device's record rewrites the
    # codes the caller's record already holds); stopped runs are left out (the twin batch has no run control)
    h2 = fr.resident_create(L, n)
    fr.resident_upload(h2, 0, bad)
    dense2, _ = fr.resident_tick(h2, L, n, NONE_D)
    live = area["stop"] == 0
    rep = np.zeros(n, bool)
    rep[drifted] = True
    assert dense2[rep & live].tobytes() == dense1[rep & live].tobytes()
    flag = np.uint32(A.SUM_PHASE_CHANGED)
    s1, s2 = dense1[:, :4].copy().view("<u4") & ~flag, dense2[:, :4].copy().view("<u4") & ~flag
    assert np.array_equal(s1[live], s2[live]) and dense1[live][:, 4:].tobytes() == dense2[live][:, 4:].tobytes()


def test_refusals_and_truncation(fr):
    rng = np.random.default_rng(11)
    n = 300
    topos, L, h = _looped(fr, rng, 96, A.F_COND | A.F_DECISION, n, ticks=1)
    state = fr.resident_download(h, 0, n, L.state_stride)
    area = fr.resident_runctl_download(h, 0, n)
    bad = perturb(rng, L, cluster_view(L, topos, state, area), topos.slots, 60)
    want = M.compare(L, topos, state, bad, np.arange(n), A.RESYNC_ALL_FIELDS, area)
    got = fr.resident_resync(h, n, bad, check=True, drifted_cap=5, items_cap=7)
    assert got["n_items"] == want.size and got["items"].tobytes() == want[:7].tobytes()
    assert got["drifted"].tolist() == np.unique(want["run"])[:5].tolist() and got["n_drifted"] == np.unique(want["run"]).size

    def refused(**kw):
        args = dict(records=bad, check=False)
        args.update(kw)
        with pytest.raises(A.FrontierError) as e:
            fr.resident_resync(h, args.pop("n_runs", n), **args)
        assert fr.resident_download(h, 0, n, L.state_stride).tobytes() == state.tobytes()
        return e.value

    refused(n_runs=n + 1)
    refused(runs=np.array([3, 2], np.uint32), records=bad[:2])
    refused(runs=np.array([n], np.uint32), records=bad[:1])
    refused(fields=0x40)
    wrong = bad.copy()
    wrong[17][:4] = np.frombuffer(np.uint32(4000).tobytes(), np.uint8)
    assert refused(records=wrong).bad_run == 17
    q = A.Resync(struct_size=ctypes.sizeof(A.Resync), n_runs=n, n=n, records=bad.ctypes.data, flags=0x2)
    assert fr._lib.bf_resident_resync(fr._ctx, h, ctypes.byref(q)) == A.BF_EINVAL
    q = A.Resync(struct_size=ctypes.sizeof(A.Resync), n_runs=n, n=n - 1, records=bad.ctypes.data)
    assert fr._lib.bf_resident_resync(fr._ctx, h, ctypes.byref(q)) == A.BF_EINVAL   # runs == NULL needs n == n_runs
    q = A.Resync(struct_size=ctypes.sizeof(A.Resync), n_runs=n, n=n, records=None)
    assert fr._lib.bf_resident_resync(fr._ctx, h, ctypes.byref(q)) == A.BF_EINVAL
    q = A.Resync(struct_size=ctypes.sizeof(A.Resync), n_runs=n, n=n, records=bad.ctypes.data, items_cap=4)
    assert fr._lib.bf_resident_resync(fr._ctx, h, ctypes.byref(q)) == A.BF_EINVAL
    q = A.Resync(struct_size=ctypes.sizeof(A.Resync) - 4, n_runs=n, n=n, records=bad.ctypes.data)
    assert fr._lib.bf_resident_resync(fr._ctx, h, ctypes.byref(q)) == A.BF_EINVAL
    assert fr.resident_download(h, 0, n, L.state_stride).tobytes() == state.tobytes()


def test_pinned_outputs(fr):
    rng = np.random.default_rng(13)
    n = 300
    topos, L, h = _looped(fr, rng, 128, A.F_COND | A.F_DECISION, n, ticks=1)
    state = fr.resident_download(h, 0, n, L.state_stride)
    area = fr.resident_runctl_download(h, 0, n)
    bad = perturb(rng, L, cluster_view(L, topos, state, area), topos.slots, 40)
    want = M.compare(L, topos, state, bad, np.arange(n), A.RESYNC_ALL_FIELDS, area)
    p_items = fr.alloc_pinned(16 * max(want.size, 1)).view(Frontier.DRIFT_DTYPE)
    p_drift = fr.alloc_pinned(4 * n).view(np.uint32)
    q = A.Resync(struct_size=ctypes.sizeof(A.Resync), n_runs=n, n=n, records=bad.ctypes.data, fields=A.RESYNC_ALL_FIELDS,
                 flags=A.RESYNC_CHECK, drifted_cap=n, drifted=p_drift.ctypes.data, items=p_items.ctypes.data, items_cap=want.size)
    assert fr._lib.bf_resident_resync(fr._ctx, h, ctypes.byref(q)) == A.BF_OK
    assert q.n_items == want.size and p_items[:want.size].tobytes() == want.tobytes()
    assert p_drift[:q.n_drifted].tolist() == np.unique(want["run"]).tolist()
    fr.free_pinned(p_items)
    fr.free_pinned(p_drift)
