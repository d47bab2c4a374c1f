"""A host model of bf_resident_commit_rewrites, written from the contract in include/bobrafrontier.h ("tick commits").

The base codes of a run are tests/resync.py:post_phases (the packed oracle's single pass with stage D's cond-FAIL writes set back),
for every run that has masks (tests/commit.py:masks), no BF_COMMIT_ERROR entry and no stop; the writes of tests/commit.py go on
top of them.  The journal is the byte difference of the records (tests/commit_journal.py), a PHASE item of a step without a mask
bit marked BF_COMMIT_WRITE_REWRITE.  States, results, schedules and entries are those of tests/commit.py; runctl is a run-control
area (tests/runctl.py) or None.  commit() changes `state` in place, as tests/commit.py:commit."""
import numpy as np

from bobrapet_b200 import _abi as A
from tests import commit as M
from tests import commit_journal as J
from tests import resync as RS

REWRITE = A.COMMIT_WRITE_REWRITE


def _code_planes(codes):
    """codes of steps [0, S) -> the 4 phase planes as Python ints"""
    return [sum(1 << int(s) for s in np.flatnonzero((codes >> b) & 1)) for b in range(4)]


def commit(L, topo, topos, state, result, sched, n_runs, entries=(), runctl=None, post=None):
    """-> (status, bad_run, bad_step, counts, touched runs, n_rewritten, {run: the steps with a mask bit}); nothing changes
    unless the status is 0.  topo: tests/commit.py:Topologies, topos: tests/resync.py:Topos of the same slots (or post: the
    post_phases of runs [0, n_runs), already taken)."""
    entries = [tuple(int(x) for x in e) for e in entries]
    rc, br, bs = M.check(L, topo, state, result, sched, n_runs, entries)
    counts = dict.fromkeys(M.COUNT_KEYS, 0)
    if rc:
        return rc, br, bs, counts, set(), 0, {}
    if post is None:
        post = RS.post_phases(L, topos, [state[r] for r in range(n_runs)]) if n_runs else []
    by_run = {}
    for run, step, kind, code in entries:
        by_run.setdefault(run, []).append((step, kind, code))
    touched, masked, n_rw = set(), {}, 0
    for r in range(n_runs):
        t, launched, queued, skip, fail = M.masks(L, topo, state, result, sched, r)
        if t is None:
            continue
        ents = by_run.get(r, [])
        if any(k == M.ERROR for _, k, _ in ents):
            continue
        hold = sum(1 << s for s, k, _ in ents if k == M.HOLD)
        valid = (1 << t["S"]) - 1
        row = state[r]
        p = M._planes(row, L)
        keep = valid & ~(p[0] & p[1] & p[2] & p[3])
        m = [x & keep for x in p]
        stopped = runctl is not None and int(runctl[r]["stop"]) != 0
        n = m if stopped or post[r] is None else _code_planes(post[r])
        SK = skip
        FA = fail & ~SK
        LA = launched & ~SK & ~FA & ~hold
        QU = queued & ~SK & ~FA & ~launched
        n = M._pset(M.FAILED, FA, n)
        n = M._pset(M.SKIPPED, SK, n)
        none_or_q = valid & (~(n[0] | n[1] | n[2] | n[3]) | (~n[0] & n[1] & n[2] & n[3]))
        n = M._pset(M.SUCCEEDED, LA & t["cond"], n)
        n = M._pset(M.PAUSED, LA & t["sync"], n)
        n = M._pset(M.RUNNING, LA & t["par"], n)
        n = M._pset(M.RUNNING, LA & ~t["cond"] & ~t["sync"] & ~t["par"] & ~t["stop"] & none_or_q, n)
        n = M._pset(M.QUEUED, QU, n)
        for s, k, code in ents:
            if k == M.PHASE and (LA >> s) & 1:
                n = M._pset(code, 1 << s, n)
        dirty = (n[0] ^ m[0]) | (n[1] ^ m[1]) | (n[2] ^ m[2]) | (n[3] ^ m[3])
        masked[r] = SK | FA | LA | QU
        if dirty:
            _store = [(p[b] & ~dirty) | (n[b] & dirty) for b in range(4)]
            M._store_planes(row, L, _store)
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
            n_rw += bin(dirty & ~masked[r]).count("1")
            counts["n_runs_written"] += 1
            counts["n_skipped"] += bin(dirty & SK).count("1")
            counts["n_launched"] += bin(dirty & LA).count("1") + reg_only
            counts["n_queued"] += bin(dirty & QU).count("1")
            counts["n_failed"] += bin(dirty & FA).count("1")
    return 0, None, None, counts, touched, n_rw, masked


def journal(L, before, after, n_runs, masked, area_before=None, area_after=None):
    """-> (items, runs) of tests/commit_journal.py:journal, each PHASE item of a step outside masked[run] marked REWRITE"""
    items, runs = J.journal(L, before, after, n_runs, area_before, area_after)
    out = []
    for (r, idx, f, code, b, a) in items:
        if f == J.PHASE and not (masked.get(r, 0) >> idx) & 1:
            code = REWRITE
        out.append((r, idx, f, code, b, a))
    return out, runs


def post_differs(L, topos, state, n_runs):
    """the runs of [0, n_runs) whose post_phases differ from their stored codes (15 read as 0)"""
    from tests.runstatus import _codes
    post = RS.post_phases(L, topos, [state[r] for r in range(n_runs)]) if n_runs else []
    out = []
    for r in range(n_runs):
        if post[r] is None:
            continue
        if not np.array_equal(post[r], _codes(state[r], L.off_phase, L.words, post[r].size)):
            out.append(r)
    return out
