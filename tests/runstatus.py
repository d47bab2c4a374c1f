"""A host model of bf_resident_status, written from the contract in include/bobrafrontier.h ("run status").

State records are the uint8 arrays of tests/packing.py (one row per run).  The phases after stages G, H and I and the pass's
summary come from the packed oracle (oracle/packed.py: one single pass with BF_F_OUT_PHASE | BF_F_OUT_FAIL); its phase_out also
carries stage D's cond-FAIL writes, which reach a record only through a commit, so the steps of its fail mask get their input
codes back.  runctl is a run-control area (tests/runctl.py) or None.  Nothing here changes its arguments."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from oracle import packed as PK

STATUS_DTYPE = Frontier.STATUS_DTYPE
IN_FIELDS = A.F_COND | A.F_DECISION | A.F_CHILD
NO_STEP = A.STATUS_NO_STEP
_STORY_PHASE = {A.OUTCOME_SUCCEEDED: A.PHASE_SUCCEEDED, A.OUTCOME_DEPENDENCY_FAILED: A.PHASE_FAILED,
                A.OUTCOME_COMPENSATION_FAILED: A.PHASE_FAILED, A.OUTCOME_CLEANUP_FAILED: A.PHASE_FAILED,
                A.OUTCOME_COMPENSATED: A.PHASE_COMPENSATED, A.OUTCOME_TIMED_OUT: A.PHASE_TIMEOUT,
                A.OUTCOME_CANCELED: A.PHASE_FINISHED}
_STOP_OUTCOME = {A.STOP_TIMEOUT: A.OUTCOME_TIMED_OUT, A.STOP_CANCEL: A.OUTCOME_CANCELED, A.STOP_HOST: A.OUTCOME_STOPPED}


def _codes(row, off, words, S):
    """the 4-bit codes of steps [0, S) in the planes at `off`, code 15 read as 0"""
    w = np.frombuffer(row[off:off + 16 * words].tobytes(), "<u4").reshape(4, words)
    bits = np.unpackbits(w.view(np.uint8).reshape(4, words * 4), axis=1, bitorder="little")[:, :S]
    c = (bits * np.array([1, 2, 4, 8], np.uint8)[:, None]).sum(axis=0).astype(np.uint8)
    c[c == 15] = 0
    return c


def _mask(row, off, words, S):
    w = np.frombuffer(row[off:off + 4 * words].tobytes(), np.uint8)
    return np.unpackbits(w, bitorder="little")[:S].astype(bool)


def status(L, ts, slots, state, n_runs, runs=None, runctl=None, events_cap=None):
    """-> (records STATUS_DTYPE[len(runs)], events u16[min(n_events, events_cap)], n_events) for the listed runs (None: every
    run of [0, n_runs)), as bf_resident_status reports them"""
    runs = np.arange(n_runs, dtype=np.uint32) if runs is None else np.asarray(runs, dtype=np.uint32)
    # the width of the layout, not its steps_max: a slot whose S passes steps_max but not 32 * words is live on the device
    L2 = make_layout(32 * L.words, L.child_nibbles, (L.fields & IN_FIELDS) | A.F_OUT_PHASE | A.F_OUT_FAIL)
    assert L2.state_stride == L.state_stride
    info = {}   # slot -> (S, allowFailure, group per step, n_comp)
    s0 = 0
    for i in range(ts.count):
        S = int(ts.S[i])
        fl = ts.step_flags[s0:s0 + S].astype(np.int64)
        g = (fl >> A.SF_GROUP_SHIFT) & 3
        info[int(slots[i])] = (S, (fl & A.SF_ALLOW_FAILURE) != 0, g, int((g == 1).sum()))
        s0 += S
    # dead: a slot no topology holds, or one of more words than the layout (the oracle refuses both; the device reports them DEAD)
    slot_of = [int(state[r][:4].view("<u4")[0]) for r in runs]
    alive = [k for k, sl in enumerate(slot_of) if sl in info and (info[sl][0] + 31) // 32 <= L.words]
    res = np.zeros((runs.size, L2.result_stride), np.uint8)
    if alive:
        res[alive] = PK.evaluate(PK.PackedTopologies(ts, slots), L2, np.ascontiguousarray(state[runs[alive]]))[0]
    alive = set(alive)
    recs = np.zeros(runs.size, dtype=STATUS_DTYPE)
    events = []
    for k, r in enumerate(runs):
        rec = recs[k]
        rec["run"], rec["first_event"], rec["first_failed"] = r, len(events), NO_STEP
        summary = int(res[k][:4].view("<u4")[0])
        if k not in alive or summary == 0xFFFFFFFF:
            rec["outcome"] = A.OUTCOME_DEAD
            continue
        S, af, grp, n_comp = info[slot_of[k]]
        ph = _codes(res[k], L2.off_phase_out, L.words, S)
        fail = _mask(res[k], L2.off_fail, L.words, S)
        ph[fail] = _codes(state[r], L.off_phase, L.words, S)[fail]
        term = np.isin(ph, (4, 5, 6, 7, 11, 12))   # terminal and neither Succeeded nor Skipped
        failed, allowed = term & ~af, term & af
        stop = int(runctl[r]["stop"]) if runctl is not None else A.STOP_NONE
        group = summary & 3
        listed = np.zeros(S, bool)
        if stop != A.STOP_NONE:
            outcome = _STOP_OUTCOME[stop]
        elif group != A.GROUP_DONE:
            outcome = A.OUTCOME_NONE
        elif (failed & (grp == 2)).any():
            outcome, listed = A.OUTCOME_CLEANUP_FAILED, failed & (grp == 2)
        elif (failed & (grp == 1)).any():
            outcome, listed = A.OUTCOME_COMPENSATION_FAILED, failed & (grp == 1)
        elif (failed & (grp == 0)).any():
            outcome = A.OUTCOME_COMPENSATED if n_comp else A.OUTCOME_DEPENDENCY_FAILED
            listed = failed & (grp == 0)
        else:
            outcome = A.OUTCOME_SUCCEEDED
        rec["group"], rec["summary"], rec["outcome"] = group, summary & 0xFF, outcome
        rec["story_phase"] = _STORY_PHASE.get(outcome, 0)
        if listed.any():
            rec["first_failed"] = int(np.flatnonzero(listed)[0])
        rec["active"] = int(np.isin(ph, (A.PHASE_RUNNING, A.PHASE_PAUSED)).sum())
        rec["completed"] = int((ph == A.PHASE_SUCCEEDED).sum())
        rec["failed"] = int((ph == A.PHASE_FAILED).sum())
        rec["skipped"] = int((ph == A.PHASE_SKIPPED).sum())
        for s in np.flatnonzero(listed | allowed):
            kind = A.STATUS_EVT_FAILED if listed[s] else A.STATUS_EVT_ALLOWED
            events.append(int(s) | int(ph[s]) << 10 | kind << 14)
        rec["n_events"] = len(events) - int(rec["first_event"])
    n_events = len(events)
    cap = n_events if events_cap is None else min(int(events_cap), n_events)
    return recs, np.asarray(events[:cap], dtype=np.uint16), n_events
