"""A host model of a resident batch's run-control area (bf_resident_runctl*, the run-level part of bf_resident_fire and what the
other resident calls do to the area), written from the contract in include/bobrafrontier.h.

An area is a numpy array of RUNCTL_DTYPE (bf_run_ctl), one record per run of the capacity.  State records are the uint8 arrays of
tests/packing.py (one row per run, run_flags at byte 4); timer areas are those of tests/timers.py (or None: no timer area); limiter
inputs those of tests/sched_resident.py (or None).  Every function changes its arguments in place unless it says otherwise and
returns the runs it touched (a stop touches its run as a delta does)."""
import numpy as np

from tests import timers as T

NONE = 0xFFFFFFFF
EINVAL = -1
STOP_NONE, STOP_TIMEOUT, STOP_CANCEL, STOP_HOST = 0, 1, 2, 3
FIRED_DRAIN, FIRED_STORY = 0xFFFE, 0xFFFF
DEC_PENDING, DEC_TIMED_OUT = 0, 3
RF_TOPOLOGY_TERMINATED = 0x04
STOPPED_FLAGS = 0x08 | 3 << 4          # BF_RF_HOST_GROUP | BF_GROUP_DONE << BF_RF_HOST_GROUP_SHIFT
PHASE_TIMEOUT = 11
REDRIVE_ALL = 0xFFFFFFFF

RUNCTL_DTYPE = np.dtype([("story_deadline", "<u4"), ("drain_deadline", "<u4"), ("stop", "u1"), ("saved_flags", "u1"),
                         ("reserved", "u1", (6,))])
PUT_DTYPE = np.dtype([("run", "<u4"), ("story_deadline", "<u4"), ("drain_deadline", "<u4"), ("stop", "u1"),
                      ("reserved", "u1", (3,))])


def defaults(n):
    a = np.zeros(n, dtype=RUNCTL_DTYPE)
    a["story_deadline"] = NONE
    a["drain_deadline"] = NONE
    return a


def due(deadline, now):
    return int(deadline) != NONE and int(deadline) <= now


def stop(area, state, r, reason, timers=None, sched=None):
    """stops run r for `reason` unless it is stopped -> True when it was stopped now (and so touched)"""
    if area["stop"][r]:
        return False
    area["saved_flags"][r] = state[r][4]
    area["stop"][r] = reason
    state[r][4] = STOPPED_FLAGS
    if timers is not None:
        timers[r] = T.EMPTY
    if reason == STOP_TIMEOUT and sched is not None:
        sched["run_phase"][r] = PHASE_TIMEOUT
    return True


def check_put(area, reqs):
    """the status bf_resident_runctl_put returns (0 or EINVAL)"""
    if area is None:
        return EINVAL
    seen = set()
    for q in reqs:
        r = int(q["run"])
        if r >= area.shape[0] or int(q["stop"]) > STOP_HOST or any(int(x) for x in q["reserved"]) or r in seen:
            return EINVAL
        seen.add(r)
    return 0


def put(area, state, reqs, timers=None, sched=None):
    """bf_resident_runctl_put -> (status, touched runs); nothing changes unless the status is 0"""
    rc = check_put(area, reqs)
    if rc:
        return rc, set()
    touched = set()
    for q in reqs:
        r = int(q["run"])
        area["story_deadline"][r] = q["story_deadline"]
        area["drain_deadline"][r] = q["drain_deadline"]
        if int(q["stop"]) and stop(area, state, r, int(q["stop"]), timers, sched):
            touched.add(r)
    return 0, touched


def fire(area, L, state, timers, n_runs, now, sched=None):
    """bf_resident_fire over runs [0, n_runs) of a batch with a run-control area (`area` may be None: the timers alone) and a timer
    area or none (`timers` None) -> dict as timers.fire gives it (touched included)"""
    out = {"n_fired": 0, "n_written": 0, "n_pruned": 0, "next_deadline": NONE, "fired": [], "touched": set()}
    for r in range(n_runs):
        entries = []
        if area is not None and not area["stop"][r] and due(area["story_deadline"][r], now):
            if timers is not None:
                out["n_pruned"] += len(T.armed(timers[r]))
            stop(area, state, r, STOP_TIMEOUT, timers, sched)
            out["touched"].add(r)
            out["n_written"] += 1
            entries.append((r, FIRED_STORY, DEC_TIMED_OUT, 1))
        elif timers is not None:
            o = T.fire(timers[r:r + 1], L, state[r:r + 1], 1, now)
            for k in ("n_written", "n_pruned"):
                out[k] += o[k]
            out["next_deadline"] = min(out["next_deadline"], o["next_deadline"])
            entries += [(r, s, c, w) for _, s, c, w in o["fired"]]
            if o["touched"]:
                out["touched"].add(r)
        if area is not None:
            if due(area["drain_deadline"][r], now):
                area["drain_deadline"][r] = NONE
                entries.append((r, FIRED_DRAIN, DEC_PENDING, 0))
            else:
                out["next_deadline"] = min(out["next_deadline"], int(area["drain_deadline"][r]))
            if not area["stop"][r]:
                out["next_deadline"] = min(out["next_deadline"], int(area["story_deadline"][r]))
        entries.sort(key=lambda e: e[1])
        out["fired"] += entries
        out["n_fired"] += len(entries)
    return out


def deltas(area, state, ds):
    """the run-control part of the delta scatter: the RUN_FLAGS deltas of stopped runs go to saved_flags.  -> the deltas the
    record scatter still applies as usual (the others)"""
    if area is None:
        return ds
    keep = np.ones(len(ds), dtype=bool)
    for i, d in enumerate(ds):
        r = int(d["run"])
        if int(d["field"]) == 4 and r < area.shape[0] and area["stop"][r]:
            area["saved_flags"][r] = d["code"]
            keep[i] = False
    return ds[keep]


def upload(area, state, first, records):
    """bf_resident_upload of `records` at first: the stopped runs keep their stop, with the uploaded byte saved"""
    state[first:first + len(records)] = records
    if area is None:
        return
    for r in range(first, first + len(records)):
        if area["stop"][r]:
            area["saved_flags"][r] = state[r][4]
            state[r][4] = STOPPED_FLAGS


def redrive(area, state, requests, status):
    """the run-control part of bf_resident_redrive, applied after the record reset (which clears TOPOLOGY_TERMINATED)"""
    if area is None:
        return
    for q, st in zip(requests, status):
        if not st:
            continue
        r = int(q["run"])
        if area["stop"][r]:
            state[r][4] = int(area["saved_flags"][r]) & ~RF_TOPOLOGY_TERMINATED & 0xFF
            area["stop"][r] = 0
            area["saved_flags"][r] = 0
        area["drain_deadline"][r] = NONE
        if int(q["step"]) == REDRIVE_ALL:
            area["story_deadline"][r] = NONE


def retire(area, N, runs, capacity=0):
    """bf_resident_retire -> the new area"""
    m, mv = T.retire_moves(N, runs)
    out = area.copy()
    for src, dst in mv.items():
        out[dst] = area[src]
    out[m:N] = defaults(N - m)
    return out[:capacity].copy() if capacity else out


def fits(src_area, dst_area, run):
    """a moved run has somewhere to keep its record"""
    return src_area is None or dst_area is not None or src_area[run].tobytes() == defaults(1)[0].tobytes()


def transfer(src_area, dst_area, src_N, dst_first, runs):
    """bf_resident_transfer after the fit check -> (source area, destination area); either may be None"""
    if dst_area is not None:
        dst_area = dst_area.copy()
        for i, r in enumerate(runs):
            dst_area[dst_first + i] = defaults(1)[0] if src_area is None else src_area[r]
    if src_area is not None:
        src_area = retire(src_area, src_N, runs)
    return src_area, dst_area


def reshape(area, capacity):
    out = defaults(max(capacity, area.shape[0]))
    out[:area.shape[0]] = area
    return out
