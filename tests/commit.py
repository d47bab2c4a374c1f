"""A host model of bf_resident_commit, written from the contract in include/bobrafrontier.h ("tick commits").

State records are the uint8 arrays of tests/packing.py (one row per run), result records those of a pass (one row per run at the
layout's result_stride).  A schedule is None (the batch has no limiter area: launched = ready, nothing queued) or a dict run ->
(launch, queued) of step bit masks as Python ints (queued = queued_story | queued_sched).  Masks are Python ints, bit i = step i.
Every function changes its arguments in place unless it says otherwise."""
import numpy as np

from bobrapet_b200 import _abi as A

EINVAL = -1
HOLD, ERROR, PHASE = A.COMMIT_HOLD, A.COMMIT_ERROR, A.COMMIT_PHASE
NONE = A.COMMIT_NONE
NOT_LAUNCHED, NOT_STOP, NO_PHASE = 1, 2, 3
SKIPPED, FAILED, SUCCEEDED, PAUSED, RUNNING, QUEUED = 13, 4, 3, 8, 2, 14
COUNT_KEYS = ("n_runs_written", "n_skipped", "n_launched", "n_queued", "n_failed")


class Topologies:
    """per slot: S, the step-type masks and the parallel descs' steps (desc order), from a TopologySet and its slots"""

    def __init__(self, ts, slots):
        self.by_slot = {}
        s0 = p0 = 0
        for i in range(ts.count):
            S, P = int(ts.S[i]), int(ts.P[i])
            types = (ts.step_flags[s0:s0 + S] & A.SF_TYPE_MASK).astype(np.int64)
            mask = lambda *ks: sum(1 << j for j in range(S) if int(types[j]) in ks)  # noqa: E731
            par = [int(x) for x in ts.parallel["step"][p0:p0 + P]] if P else []
            self.by_slot[int(slots[i])] = dict(S=S, cond=mask(A.STEP_CONDITION), sync=mask(A.STEP_SLEEP, A.STEP_WAIT, A.STEP_GATE),
                                               par=mask(A.STEP_PARALLEL), stop=mask(A.STEP_STOP), par_steps=par)
            s0 += S
            p0 += P

    def drop(self, slot):
        self.by_slot.pop(int(slot), None)


def _word_int(row, off, words):
    return int.from_bytes(row[off:off + 4 * words].tobytes(), "little")


def _planes(row, L):
    return [_word_int(row, L.off_phase + b * 4 * L.words, L.words) for b in range(4)]


def _store_planes(row, L, p):
    n = 4 * L.words
    for b in range(4):
        row[L.off_phase + b * n:L.off_phase + (b + 1) * n] = np.frombuffer(p[b].to_bytes(n, "little"), np.uint8)


def _pset(code, m, p):
    return [(p[b] | m) if (code >> b) & 1 else (p[b] & ~m) for b in range(4)]


def masks(L, topo, state, result, sched, r):
    """-> (topology info or None, launched, queued, skip, fail) of run r"""
    slot = int(state[r][:4].view("<u4")[0])
    t = topo.by_slot.get(slot)
    if t is None or (t["S"] + 31) // 32 > L.words:
        return None, 0, 0, 0, 0
    res = result[r]
    ready = _word_int(res, L.off_ready, L.words)
    skip = _word_int(res, L.off_skip, L.words)
    fail = _word_int(res, L.off_fail, L.words) if L.off_fail != A.OFF_NONE else 0
    launched, queued = ready, 0
    if sched is not None:
        launched, queued = sched.get(r, (0, 0))
    return t, launched, queued, skip, fail


def check(L, topo, state, result, sched, n_runs, entries):
    """the entry checks, in the contract's order -> (0, None, None) or (EINVAL, bad_run, bad_step)"""
    seen = {}
    for e in entries:
        run, step, kind, code = (int(x) for x in e)
        if run >= n_runs or step >= L.steps_max or kind not in (HOLD, ERROR, PHASE) or \
                (not (A.PHASE_PENDING <= code <= A.PHASE_SKIPPED) if kind == PHASE else code != 0):
            return EINVAL, run, step
        seen.setdefault((run, step), []).append(kind)
    dups = sorted(k for k, v in seen.items() if len(v) > 1)
    if dups:
        return EINVAL, dups[0][0], dups[0][1]
    by_run = {}
    for (run, step), kinds in seen.items():
        by_run.setdefault(run, {})[step] = kinds[0]
    offences = []
    runs = set(by_run)
    for r in range(n_runs):
        t, launched, _q, _s, _f = masks(L, topo, state, result, sched, r)
        if t is None and r not in runs:
            continue
        ents = by_run.get(r, {})
        stop = t["stop"] if t else 0
        for step in sorted(ents):
            if not (launched >> step) & 1:
                offences.append((r, step, NOT_LAUNCHED))
                break
            if ents[step] == PHASE and not (stop >> step) & 1:
                offences.append((r, step, NOT_STOP))
                break
        if ERROR not in ents.values():
            covered = sum(1 << s for s in ents)
            miss = launched & stop & ~covered
            if miss:
                offences.append((r, (miss & -miss).bit_length() - 1, NO_PHASE))
    if offences:
        r, s, _ = min(offences)
        return EINVAL, r, s
    return 0, None, None


def commit(L, topo, state, result, sched, n_runs, entries=()):
    """bf_resident_commit's entry checks and writes -> (status, bad_run, bad_step, counts, touched runs); nothing changes unless
    the status is 0.  The call-level refusals (ticks, schedules, layout) are the caller's to model."""
    entries = [tuple(int(x) for x in e) for e in entries]
    rc, br, bs = check(L, topo, state, result, sched, n_runs, entries)
    counts = dict.fromkeys(COUNT_KEYS, 0)
    if rc:
        return rc, br, bs, counts, set()
    by_run = {}
    for run, step, kind, code in entries:
        by_run.setdefault(run, []).append((step, kind, code))
    touched = set()
    for r in range(n_runs):
        t, launched, queued, skip, fail = masks(L, topo, state, result, sched, r)
        if t is None:
            continue
        ents = by_run.get(r, [])
        if any(k == ERROR for _, k, _ in ents):
            continue
        hold = sum(1 << s for s, k, _ in ents if k == HOLD)
        valid = (1 << t["S"]) - 1
        row = state[r]
        p = _planes(row, L)
        keep = valid & ~(p[0] & p[1] & p[2] & p[3])
        m = [x & keep for x in p]
        SK = skip
        FA = fail & ~SK
        LA = launched & ~SK & ~FA & ~hold
        QU = queued & ~SK & ~FA & ~launched
        n = _pset(FAILED, FA, m)
        n = _pset(SKIPPED, SK, n)
        none_or_q = valid & (~(n[0] | n[1] | n[2] | n[3]) | (~n[0] & n[1] & n[2] & n[3]))
        n = _pset(SUCCEEDED, LA & t["cond"], n)
        n = _pset(PAUSED, LA & t["sync"], n)
        n = _pset(RUNNING, LA & t["par"], n)
        n = _pset(RUNNING, LA & ~t["cond"] & ~t["sync"] & ~t["par"] & ~t["stop"] & none_or_q, n)
        n = _pset(QUEUED, QU, n)
        for s, k, code in ents:
            if k == PHASE and (LA >> s) & 1:
                n = _pset(code, 1 << s, n)
        dirty = (n[0] ^ m[0]) | (n[1] ^ m[1]) | (n[2] ^ m[2]) | (n[3] ^ m[3])
        if dirty:
            _store_planes(row, L, [(p[b] & ~dirty) | (n[b] & dirty) for b in range(4)])
        reg = int(row[8:16].view("<u8")[0])
        newly, reg_only = 0, 0
        for q, s in enumerate(t["par_steps"]):
            if (LA >> s) & 1 and not (reg >> q) & 1:
                newly |= 1 << q
                reg_only += 0 if (dirty >> s) & 1 else 1
        if newly:
            row[8:16] = np.frombuffer(np.uint64(reg | newly).tobytes(), np.uint8)
        if dirty or newly:
            touched.add(r)
            counts["n_runs_written"] += 1
            counts["n_skipped"] += bin(dirty & SK).count("1")
            counts["n_launched"] += bin(dirty & LA).count("1") + reg_only
            counts["n_queued"] += bin(dirty & QU).count("1")
            counts["n_failed"] += bin(dirty & FA).count("1")
    return 0, None, None, counts, touched


def sched_rows(L, parts_out, rows=None):
    """the batcher's row of each run after a bf_resident_schedule (dict run -> (launch, queued)), updated from one part's listed
    runs and events"""
    rows = {} if rows is None else rows
    ev = parts_out["events"]
    pos = 0
    for r, hd in zip(parts_out["runs"], parts_out["heads"]):
        k = int(hd["n_launch"]) + int(hd["n_queued_story"]) + int(hd["n_queued_sched"])
        launch = queued = 0
        for e in ev[pos:pos + k]:
            step, kind = int(e) & 0x3FF, int(e) >> 10
            if kind & A.SEVT_LAUNCH:
                launch |= 1 << step
            if kind & (A.SEVT_QUEUED_STORY | A.SEVT_QUEUED_SCHED):
                queued |= 1 << step
        rows[int(r)] = (launch, queued)
        pos += k
    return rows
