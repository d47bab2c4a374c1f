"""The due rule of touched commits (bf_resident_commit_touched) on the host model, CPU only: random loops of deltas, touched and
full ticks, schedules and commits with random HOLD / ERROR / PHASE entries over tests/resident_model.py, with the commit of
tests/commit.py.  The model keeps the commit-due set as the contract states it: the runs a touched tick evaluated, the runs whose
schedule row changed, the runs an entry named; a full tick, a form change or the start makes the next commit consider every run;
a commit clears the runs it considered that no entry named.  At every commit two things are checked:
  - the commit restricted to the due runs (and the runs the entries name) gives the full commit's status, offender, counts,
    written runs and records: no run outside that set has a write or an offence;
  - the due set is tight: every due run below n_runs was evaluated, rescheduled or named by an entry since the last commit that
    cleared it, so a rule that marked every run would not satisfy the bookkeeping either.
The restricted commit is the full model commit over result records and schedule rows zeroed outside the set, which is what the
list-mode kernels see: a run they do not take has no masks."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import commit as M
from tests import resident_model as RM
from tests.seqrig import layout_for, random_records, story_pool

FIELDS = A.F_COND | A.F_DECISION | A.F_ALL_OUT


def _ready(L, row):
    return int.from_bytes(row[L.off_ready:L.off_ready + 4 * L.words].tobytes(), "little")


def _entries(rng, L, topo, state, cur, sched, n):
    out = []
    for r in range(n):
        t, launched, _q, _s, _f = M.masks(L, topo, state, cur, sched, r)
        if not launched:
            continue
        steps = [s for s in range(launched.bit_length()) if (launched >> s) & 1]
        named = {}
        if rng.random() < 0.04:
            named[int(rng.choice(steps))] = (M.ERROR, 0)
        elif rng.random() < 0.08:
            named[int(rng.choice(steps))] = (M.HOLD, 0)
        for s in steps:
            if (t["stop"] >> s) & 1 and s not in named:
                named[s] = (M.PHASE, int(rng.integers(A.PHASE_PENDING, A.PHASE_SKIPPED + 1)))
        out += [(r, s, k, c) for s, (k, c) in named.items()]
    if out and rng.random() < 0.1:   # an entry on a step that is not launched: the commit is refused
        r, s, _, _ = out[int(rng.integers(0, len(out)))]
        t = M.masks(L, topo, state, cur, sched, r)[0]
        free = [x for x in range(t["S"]) if not any((r, x) == (e[0], e[1]) for e in out)
                and not (M.masks(L, topo, state, cur, sched, r)[1] >> x) & 1]
        if free:
            out.append((r, int(rng.choice(free)), M.HOLD, 0))
    return out


class DueModel:
    """the commit-due set of one batch and why each run is in it"""

    def __init__(self, cap):
        self.cap = cap
        self.all = True
        self.form = None
        self.why = {r: "enabled" for r in range(cap)}

    def mark(self, runs, why):
        for r in runs:
            self.why.setdefault(r, why)

    def considered(self, n, form, entries):
        full = self.all or form != self.form
        named = {int(e[0]) for e in entries}
        return full, (set(range(n)) if full else ({r for r in self.why if r < n} | named))

    def committed(self, n, form, full, considered, entries):
        named = {int(e[0]) for e in entries}
        if full:
            self.mark(range(n, self.cap), "past n_runs")
        for r in considered - named:
            self.why.pop(r, None)
        self.mark(named, "entry")
        self.all, self.form = False, form


@pytest.mark.parametrize("seed", range(6))
def test_due_runs_carry_every_write_of_the_full_commit(seed):
    rng = np.random.default_rng(8800 + seed)
    pool = story_pool(rng, 20, 70, 2, 3)
    reg = RM.Registry(pool)
    slots = [reg.put(k) for k in range(len(pool))]
    L = layout_for(pool, FIELDS)
    topo = M.Topologies(reg.ts, slots)
    n = int(rng.integers(80, 200))
    cap = n + 10
    b = RM.Batch(reg, L, cap)
    kinds = rng.integers(0, 3, n)
    b.upload(0, random_records(rng, L, [pool[k] for k in kinds], [slots[k] for k in kinds]))
    due = DueModel(cap)
    sched = {}
    use_sched = seed % 2 == 1
    form = 0
    stats = {"listed": 0, "full": 0, "refused": 0, "outside": 0}
    for step in range(60):
        # deltas, then a tick (touched mostly, full now and then)
        k = int(rng.integers(0, max(n // 20, 2)))
        d = np.zeros(k, Frontier.DELTA_DTYPE)
        d["run"], d["index"], d["field"] = rng.integers(0, n, k), rng.integers(0, 8, k), A.DELTA_PHASE
        d["code"] = rng.integers(0, 9, k)
        if rng.random() < 0.1:
            b.tick_compact(d, n)
            due.all = True
        else:
            if b.full_due(n, 0, 0):
                due.all = True
                b.tick_touched(d, n)
            else:
                b.apply(d)
                evaluated = {r for r in b.touched if r < n}
                out = b.tick_touched(np.zeros(0, Frontier.DELTA_DTYPE), n)
                assert out["n_evaluated"] == len(evaluated)
                due.mark(evaluated, "evaluated")
        if use_sched:   # a schedule: each run launches a random part of its ready steps; a changed row makes the run due
            changed = set()
            for r in range(n):
                ready = _ready(L, b.cur[r])
                drop = int(rng.integers(0, 1 << 16)) if rng.random() < 0.2 else 0
                row = (ready & ~drop, 0)
                if sched.get(r) != row:
                    changed.add(r)
                sched[r] = row
            due.mark(changed, "rescheduled")
        if rng.random() < 0.1:
            form ^= 1   # another commit form: the next touched commit considers every run
        # the commit
        ents = _entries(rng, L, topo, b.state, b.cur, sched if use_sched else None, n)
        full, considered = due.considered(n, form, ents)
        # tight: every due run below n has a reason
        for r in considered:
            assert full or r in due.why or r in {int(e[0]) for e in ents}
        assert all(why in ("enabled", "evaluated", "rescheduled", "entry", "past n_runs") for why in due.why.values())
        want_state = b.state.copy()
        rc, br, bs, counts, touched = M.commit(L, topo, want_state, b.cur, sched if use_sched else None, n, ents)
        cur_r = np.zeros_like(b.cur)
        ix = sorted(considered)
        cur_r[ix] = b.cur[ix]
        sched_r = {r: v for r, v in sched.items() if r in considered} if use_sched else None
        got_state = b.state.copy()
        rc2, br2, bs2, counts2, touched2 = M.commit(L, topo, got_state, cur_r, sched_r, n, ents)
        assert (rc2, br2, bs2) == (rc, br, bs), ((rc2, br2, bs2), (rc, br, bs))
        if rc:
            stats["refused"] += 1
            continue
        assert counts2 == counts and touched2 == touched and np.array_equal(got_state, want_state)
        stats["full" if full else "listed"] += 1
        stats["outside"] += n - len(considered)
        due.committed(n, form, full, considered, ents)
        if touched:   # a commit that wrote touches its runs as a delta does
            b._end_snapshot()
            b.state[:] = want_state
            b.touched |= touched
    assert stats["listed"] > 0 and stats["full"] > 0 and stats["outside"] > 0, stats
