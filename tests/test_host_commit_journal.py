"""The journal of a tick commit (tests/commit_journal.py) read off the host models of the commit (tests/commit.py,
tests/commit_timers.py) over random batches at S = 32, 64, 256 and 1024: its order, its relation to the counts and the touched
runs, and that BF_COMMIT_ERROR runs, HOLD steps, runs without masks (a stopped run's tick) and dead slots list nothing, nor does a
second commit of the same tick.  No GPU."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from tests import commit as M
from tests import commit_journal as J
from tests import commit_timers as CT
from tests import randgen
from tests import timers as T
from tests.test_gpu_commit import entries_for

SYNC_CODES = {A.STEP_SLEEP: A.DEC_SUCCEED, A.STEP_GATE: A.DEC_TIMED_OUT, A.STEP_WAIT: A.DEC_PENDING}


def random_batch(rng, S, n, dead=True):
    ts = randgen.random_topologies(rng, 8, max(2, S // 2), S, max_deg=3, parallel=True, fill=0.5)
    slots = np.arange(ts.count, dtype=np.uint32)
    L, st, _ = randgen.random_state(rng, ts, slots, n, A.F_COND | A.F_DECISION | A.F_ALL_OUT, phase_mix="progress")
    topo = M.Topologies(ts, slots)
    if dead:
        topo.drop(0)   # slot 0 is dead: its runs have no masks
    timings, s0 = {}, 0
    for i in range(ts.count):
        types = ts.step_flags[s0:s0 + int(ts.S[i])] & A.SF_TYPE_MASK
        sync = [s for s, t in enumerate(types) if int(t) in SYNC_CODES][:A.TIMER_MAX_SLOTS // 2]   # no run overflows its slots
        timings[i] = {s: (SYNC_CODES[int(types[s])], int(rng.integers(0, 9))) for s in sync}
        s0 += int(ts.S[i])
    return topo, L, st, timings


def random_results(rng, L, topo, st, n, empty=()):
    """random ready / skip / fail masks over each run's steps; the runs in `empty` have none, as a stopped run's tick leaves"""
    res = np.zeros((n, L.result_stride), np.uint8)
    for r in range(n):
        t = topo.by_slot.get(int(st[r][:4].view("<u4")[0]))
        if t is None or r in empty:
            continue
        valid = (1 << t["S"]) - 1
        bits = [int.from_bytes(rng.bytes(4 * L.words), "little") & valid for _ in range(4)]
        ready = bits[0] & bits[1]
        skip, fail = bits[2] & bits[3] & ~ready, bits[1] & bits[2] & ~bits[3] & ~ready   # a launched step is neither
        for off, v in ((L.off_ready, ready), (L.off_skip, skip), (L.off_fail, fail)):
            res[r, off:off + 4 * L.words] = np.frombuffer(v.to_bytes(4 * L.words, "little"), np.uint8)
    return res


@pytest.mark.parametrize("S,n,timed", [(32, 400, False), (32, 300, True), (64, 300, True), (256, 120, False), (256, 100, True),
                                       (1024, 30, True)])
def test_journal_of_random_commits(S, n, timed):
    rng = np.random.default_rng(S * 31 + n + timed)
    topo, L, st, timings = random_batch(rng, S, n)
    empty = set(rng.choice(n, size=n // 10, replace=False).tolist())
    res = random_results(rng, L, topo, st, n, empty)
    ents = entries_for(rng, L, topo, st, res, None, n, p_hold=0.2, p_error=0.1)
    area = T.empty_area(n, A.TIMER_MAX_SLOTS) if timed else None
    before, area0 = st.copy(), None if area is None else area.copy()
    if timed:
        rc, _, _, counts, touched, n_armed, _ = CT.commit_timed(L, topo, timings, st, res, None, n, ents, area, 50, True)
    else:
        (rc, _, _, counts, touched), n_armed = M.commit(L, topo, st, res, None, n, ents), 0
    assert rc == 0
    items, runs = J.journal(L, before, st, n, area0, area)
    assert items == sorted(items, key=lambda x: (x[0], x[2], x[1])) and len(set((x[0], x[2], x[1]) for x in items)) == len(items)
    assert runs == sorted(touched) and len(runs) == counts["n_runs_written"]
    by_field = {f: [x for x in items if x[2] == f] for f in (J.PHASE, J.REGISTERED, J.TIMER)}
    assert len(by_field[J.TIMER]) == n_armed and (n_armed > 0) == timed
    n_steps = sum(counts[k] for k in ("n_skipped", "n_launched", "n_queued", "n_failed"))
    assert len(by_field[J.PHASE]) <= n_steps <= len(by_field[J.PHASE]) + len(by_field[J.REGISTERED])
    assert all(x[4] != x[5] and x[5] <= A.PHASE_PENDING_QUEUED for x in by_field[J.PHASE])
    assert {x[0] for x in by_field[J.PHASE] + by_field[J.REGISTERED]} == set(runs)
    # nothing of an ERROR run, a HOLD step, a run without masks or a dead slot
    errors = {int(e["run"]) for e in ents if e["kind"] == M.ERROR}
    holds = {(int(e["run"]), int(e["step"])) for e in ents if e["kind"] == M.HOLD}
    dead = {r for r in range(n) if int(st[r][:4].view("<u4")[0]) not in topo.by_slot}
    assert errors and holds and dead and empty
    assert not {x[0] for x in items} & (errors | dead | empty)
    assert not {(x[0], x[1]) for x in items if x[2] != J.REGISTERED} & holds
    # a second commit of the same tick lists nothing
    again = st.copy()
    if timed:
        area1 = area.copy()
        assert CT.commit_timed(L, topo, timings, st, res, None, n, ents, area, 50, True)[0] == 0
        assert J.journal(L, again, st, n, area1, area) == ([], [])
    else:
        assert M.commit(L, topo, st, res, None, n, ents)[0] == 0
        assert J.journal(L, again, st, n) == ([], [])


def test_journal_items_on_a_hand_case():
    """a skip, a cond FAIL, a launched parallel step (phase and registered bit), a queued step and a sleep arm, in that field
    order per run"""
    from tests.test_host_commit import COND, E, PAR, SLEEP, batch, result
    t, L, st = batch([E, PAR, SLEEP, COND, E], [[0, 0, 0, 0, A.PHASE_RUNNING]], fields=A.F_ALL_OUT | A.F_DECISION)
    area = T.empty_area(1, 2)
    before, area0 = st.copy(), area.copy()
    res = result(L, 1, ready=[1, 2, 4], skip=[0], fail=[3])
    rc, _, _, counts, touched, n_armed, nxt = CT.commit_timed(L, t, {0: {2: (A.DEC_SUCCEED, 4)}}, st, res, {0: (0b00110, 0b10000)}, 1,
                                                             (), area, 10, True)
    assert rc == 0 and n_armed == 1 and nxt == 14
    items, runs = J.journal(L, before, st, 1, area0, area)
    assert runs == [0]
    assert items == [(0, 0, J.PHASE, 0, 0, A.PHASE_SKIPPED), (0, 1, J.PHASE, 0, 0, A.PHASE_RUNNING),
                     (0, 2, J.PHASE, 0, 0, A.PHASE_PAUSED), (0, 3, J.PHASE, 0, 0, A.PHASE_FAILED),
                     (0, 4, J.PHASE, 0, A.PHASE_RUNNING, A.PHASE_PENDING_QUEUED),
                     (0, 0, J.REGISTERED, 0, 0, 1), (0, 2, J.TIMER, A.DEC_SUCCEED, T.NONE, 14)]
    assert counts == dict(n_runs_written=1, n_skipped=1, n_launched=2, n_queued=1, n_failed=1)
