"""A host model of bf_resident_commit_timed, written from the contract in include/bobrafrontier.h ("tick commits"), on top of the
commit model (tests/commit.py) and the timer-area model (tests/timers.py).

Timings are a dict slot -> {step: (code, delay)} (bf_topology_timings).  The area is the (capacity, K) uint64 array of
tests/timers.py; `decision` says whether the layout has decision planes."""
from tests import commit as M
from tests import timers as T

ENOMEM = -2
NO_DECISION, OVERFLOW = 4, 5   # the reasons after the entry offences (1..3)


def _host_refusal(L, n_runs, entries):
    """does one of the entry checks the host makes before the device's (each entry, then duplicates) refuse?"""
    seen = set()
    for run, step, kind, code in entries:
        if run >= n_runs or step >= L.steps_max or kind not in (M.HOLD, M.ERROR, M.PHASE) or \
                (not (1 <= code <= 13) if kind == M.PHASE else code != 0) or (run, step) in seen:
            return True
        seen.add((run, step))
    return False


def new_arms(L, topo, timings, state, result, sched, n_runs, entries, area):
    """-> {run: [(step, code, delay)] ascending by step}: what each written run would newly arm"""
    by_run = {}
    for run, step, kind, _code in entries:
        by_run.setdefault(run, {})[step] = kind
    out = {}
    for r in range(n_runs):
        t, launched, _q, skip, fail = M.masks(L, topo, state, result, sched, r)
        ents = by_run.get(r, {})
        if t is None or M.ERROR in ents.values():
            continue
        hold = sum(1 << s for s, k in ents.items() if k == M.HOLD)
        arm = launched & ~skip & ~fail & ~hold & t["sync"]
        slot = int(state[r][:4].view("<u4")[0])
        stored = {s for s, _d, _c in T.armed(area[r])}
        new = [(s, c, d) for s, (c, d) in sorted(timings.get(slot, {}).items()) if (arm >> s) & 1 and s not in stored]
        if new:
            out[r] = new
    return out


def commit_timed(L, topo, timings, state, result, sched, n_runs, entries, area, now, decision):
    """bf_resident_commit_timed's entry and arming checks and writes -> (status, bad_run, bad_step, counts, touched runs, n_armed,
    next_deadline); nothing changes unless the status is 0.  The call-level refusals are the caller's to model."""
    entries = [tuple(int(x) for x in e) for e in entries]
    counts = dict.fromkeys(M.COUNT_KEYS, 0)
    if _host_refusal(L, n_runs, entries):
        rc, br, bs = M.check(L, topo, state, result, sched, n_runs, entries)
        return rc, br, bs, counts, set(), 0, T.NONE
    rc, br, bs = M.check(L, topo, state, result, sched, n_runs, entries)
    offences = [(br, bs, 0, M.EINVAL)] if rc else []   # an entry offence wins a tie at the same (run, step)
    arms = new_arms(L, topo, timings, state, result, sched, n_runs, entries, area)
    K = area.shape[1]
    for r, new in arms.items():
        over = len(T.armed(area[r])) + len(new) > K
        dec = next((s for s, c, _d in new if c != T.DEC_PENDING), None) if not decision else None
        if dec is not None:
            offences.append((r, dec, NO_DECISION, M.EINVAL))
        if over:
            offences.append((r, new[0][0], OVERFLOW, ENOMEM))
    if offences:
        r, s, _why, code = min(offences)
        return code, r, s, counts, set(), 0, T.NONE
    rc, _br, _bs, counts, touched = M.commit(L, topo, state, result, sched, n_runs, entries)
    assert rc == 0
    n_armed, nxt = 0, T.NONE
    for r, new in arms.items():
        e = {s: (d, c) for s, d, c in T.armed(area[r])}
        for s, c, delay in new:
            e[s] = (min(now + delay, T.NONE - 1), c)
            nxt = min(nxt, e[s][0])
        area[r] = T.canonical(e, K)
        n_armed += len(new)
    return 0, None, None, counts, touched, n_armed, nxt


def arm_requests(L, topo, timings, state, result, sched, n_runs, entries, area, now, dtype):
    """what a batcher without the timed commit sends to bf_resident_timers_arm after a bf_resident_commit: a request for each
    launched sleep / gate / wait step with a timing that the run holds no armed slot for (TIMER_DTYPE rows)"""
    import numpy as np
    arms = new_arms(L, topo, timings, state, result, sched, n_runs, [tuple(int(x) for x in e) for e in entries], area)
    rows = [(r, s, c, 0, min(now + d, T.NONE - 1), 0) for r, new in sorted(arms.items()) for s, c, d in new]
    return np.array(rows, dtype=dtype) if rows else np.zeros(0, dtype=dtype)
