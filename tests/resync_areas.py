"""A host model of bf_resident_resync_areas (include/bobrafrontier.h, "resyncs"), written from the header.

The batch is a tests/lifecycle.AreaBatch: its state records, its step-timer slots (tests/timers.py), its limiter inputs
(tests/sched_resident.py) and its run-control records (tests/runctl.py), each present or absent.  The caller's areas are numpy
arrays in list order: timers SLOT_DTYPE of shape (n, K), sched SCHED_PUT_DTYPE[n], runctl RUNCTL_DTYPE[n]; None leaves an area out
of the call.  resync() changes the batch in place, as the device's repair does."""
import numpy as np

from bobrapet_b200 import _abi as A
from tests import runctl as R
from tests import timers as T

NONE = 0xFFFFFFFF
EINVAL = -1
DRIFT_DTYPE = np.dtype([("run", "<u4"), ("index", "<u2"), ("field", "u1"), ("reserved", "u1"), ("device", "<u4"),
                        ("record", "<u4")])
SLOT_DTYPE = np.dtype([("deadline", "<u4"), ("step", "<u2"), ("code", "u1"), ("reserved", "u1")])
SCHED_FIELDS = ("story_key", "queue_key", "priority", "queued_since", "run_phase")


def _u32(v):
    return int(v) & 0xFFFFFFFF


def refusal(b, n_runs, runs, n, areas, flags, timers=None, sched=None, runctl=None):
    """None when the call is accepted, else the bad_run it reports (NONE for a refusal that names no run)"""
    if n_runs > b.cap:
        return NONE
    if runs is None and n != n_runs:
        return NONE
    if runs is not None and (any(int(r) >= n_runs for r in runs) or any(int(runs[i]) <= int(runs[i - 1]) for i in range(1, n))):
        return NONE
    if flags & ~A.RESYNC_CHECK or areas & ~A.RESYNC_ALL_AREAS:
        return NONE
    sel_t, sel_s, sel_c = areas & A.RESYNC_AREA_TIMERS, areas & A.RESYNC_AREA_SCHED, areas & A.RESYNC_AREA_RUNCTL
    if (sel_t and not b.K) or (sel_s and b.sched is None) or (sel_c and b.runctl is None):
        return NONE
    if n and ((sel_t and timers is None) or (sel_s and sched is None) or (sel_c and runctl is None)):
        return NONE
    L = b.L
    for i in range(n):
        run = int(runs[i]) if runs is not None else i
        if sel_t:
            row, empty, prev = timers[i], False, -1
            for t in row:
                if int(t["deadline"]) == NONE:
                    if t["step"] or t["code"] or t["reserved"]:
                        return run
                    empty = True
                    continue
                s = int(t["step"])
                if empty or s <= prev or s >= L.steps_max or int(t["code"]) > 3 or t["reserved"]:
                    return run
                if int(t["code"]) != T.DEC_PENDING and L.off_decision == A.OFF_NONE:
                    return run
                prev = s
        if sel_s and (int(sched[i]["run"]) != run or sched[i]["reserved"].any()):
            return run
        if sel_c and (int(runctl[i]["stop"]) > R.STOP_HOST or runctl[i]["saved_flags"] or runctl[i]["reserved"].any()):
            return run
    return None


def _taken_as_fired(L, rec, s, deadline, code, fired_now):
    """a caller slot the device has no slot for, at step s: the last fire disarmed it"""
    return fired_now != NONE and deadline <= fired_now and (code == T.DEC_PENDING or T.decision(L, rec, s) != T.DEC_PENDING)


def run_items(b, r, i, areas, timers, sched, runctl, fired_now):
    """the items of listed run r (row i of the caller's arrays), in (field, index) order, as (index, field, device, record)"""
    L, out = b.L, []
    rec = b.state[r]
    dc = b.runctl[r] if b.runctl is not None else R.defaults(1)[0]
    rc = runctl[i] if areas & A.RESYNC_AREA_RUNCTL else dc
    stopped = bool(dc["stop"]) or bool(rc["stop"])
    if areas & A.RESYNC_AREA_TIMERS and not stopped:
        dev = {s: (d, c) for s, d, c in T.armed(b.timers[r])}
        cal = {int(t["step"]): (int(t["deadline"]), int(t["code"])) for t in timers[i] if int(t["deadline"]) != NONE}
        tim, code = [], []
        for s in sorted(set(dev) | set(cal)):
            if (T.LUT_TERMINAL >> T.phase(L, rec, s)) & 1:
                continue
            if s in dev and s in cal:
                if dev[s][0] != cal[s][0]:
                    tim.append((s, A.DRIFT_TIMER, dev[s][0], cal[s][0]))
                if dev[s][1] != cal[s][1]:
                    code.append((s, A.DRIFT_TIMER_CODE, dev[s][1], cal[s][1]))
            elif s in dev:
                tim.append((s, A.DRIFT_TIMER, dev[s][0], NONE))
            elif not _taken_as_fired(L, rec, s, cal[s][0], cal[s][1], fired_now):
                tim.append((s, A.DRIFT_TIMER, NONE, cal[s][0]))
        out += tim + code
    if areas & A.RESYNC_AREA_SCHED:
        for f, name in enumerate(SCHED_FIELDS):
            dv, rv = _u32(b.sched.inputs[r][name]), _u32(sched[i][name])
            if dv != rv:
                out.append((0, A.DRIFT_SCHED_STORY_KEY + f, dv, rv))
    if areas & A.RESYNC_AREA_RUNCTL:
        if int(dc["story_deadline"]) != int(rc["story_deadline"]):
            out.append((0, A.DRIFT_STORY_DEADLINE, int(dc["story_deadline"]), int(rc["story_deadline"])))
        dd, rd = int(dc["drain_deadline"]), int(rc["drain_deadline"])
        if dd != rd and not (dd == NONE and fired_now != NONE and rd <= fired_now):
            out.append((0, A.DRIFT_DRAIN_DEADLINE, dd, rd))
        if int(dc["stop"]) != int(rc["stop"]):
            out.append((0, A.DRIFT_STOP, int(dc["stop"]), int(rc["stop"])))
    return out


def resync(b, n_runs, runs=None, timers=None, sched=None, runctl=None, fired_now=NONE, check=False):
    """bf_resident_resync_areas on model batch b (changed in place unless check) -> dict(status, bad_run, items DRIFT_DTYPE,
    drifted, n_written, stopped: the runs the repair stopped, touched as by a delta)"""
    n = n_runs if runs is None else len(runs)
    areas = (A.RESYNC_AREA_TIMERS if timers is not None else 0) | (A.RESYNC_AREA_SCHED if sched is not None else 0) | \
            (A.RESYNC_AREA_RUNCTL if runctl is not None else 0)
    bad = refusal(b, n_runs, runs, n, areas, 0, timers, sched, runctl)
    if bad is not None:
        return {"status": EINVAL, "bad_run": bad}
    rows, drifted, written, stopped = [], [], 0, []
    L = b.L
    for i in range(n):
        r = int(runs[i]) if runs is not None else i
        its = run_items(b, r, i, areas, timers, sched, runctl, fired_now)
        if not its:
            continue
        drifted.append(r)
        rows += [(r, ix, f, 0, dv, rv) for ix, f, dv, rv in its]
        if check:
            continue
        fields = {f for _, f, _, _ in its}
        wrote = False
        dc_stop = b.runctl is not None and int(b.runctl["stop"][r])
        rc_stop = int(runctl[i]["stop"]) if runctl is not None else 0
        if fields & {A.DRIFT_TIMER, A.DRIFT_TIMER_CODE}:   # the caller's slots minus those taken as fired
            keep = {int(t["step"]): (int(t["deadline"]), int(t["code"])) for t in timers[i] if int(t["deadline"]) != NONE}
            dev = {s for s, _, _ in T.armed(b.timers[r])}
            keep = {s: dc for s, dc in keep.items() if s in dev or not _taken_as_fired(L, b.state[r], s, dc[0], dc[1], fired_now)}
            b.timers[r] = T.canonical(keep, b.K)
            wrote = True
        if fields & set(range(A.DRIFT_SCHED_STORY_KEY, A.DRIFT_SCHED_RUN_PHASE + 1)):
            q = sched[i].copy()
            q["run"] = 0
            b.sched.inputs[r] = q
            wrote = True
        if A.DRIFT_STORY_DEADLINE in fields:
            b.runctl["story_deadline"][r] = runctl[i]["story_deadline"]
            wrote = True
        if A.DRIFT_DRAIN_DEADLINE in fields:
            b.runctl["drain_deadline"][r] = runctl[i]["drain_deadline"]
            wrote = True
        if rc_stop and not dc_stop:
            R.stop(b.runctl, b.state, r, rc_stop, b.timers, b.inputs)
            stopped.append(r)
            wrote = True
        written += wrote
    items = np.array(rows, dtype=DRIFT_DTYPE) if rows else np.zeros(0, DRIFT_DTYPE)
    return {"status": 0, "bad_run": NONE, "items": items, "drifted": np.array(drifted, np.uint32), "n_written": written,
            "stopped": stopped}


def device_areas(b, runs=None, n_runs=None):
    """the caller's arrays that equal the model batch's own areas for the listed runs (what a batcher with no drift packs)
    -> (timers, sched, runctl), None for an area the batch lacks"""
    runs = np.arange(n_runs if n_runs is not None else b.n) if runs is None else np.asarray(runs)
    timers = b.timers[runs].copy().view(SLOT_DTYPE) if b.K else None
    sched = None
    if b.sched is not None:
        sched = b.sched.inputs[runs].copy()
        sched["run"] = runs
    runctl = None
    if b.runctl is not None:
        runctl = b.runctl[runs].copy()
        runctl["saved_flags"] = 0
    return timers, sched, runctl

