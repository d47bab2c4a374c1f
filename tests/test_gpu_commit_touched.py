"""Touched commits (bf_resident_commit_touched) against the full forms on the device: twin batches on one ctx, A committed with
bf_resident_commit / _timed / _journal / _rewrites and B with the touched call of the same form, driven by one random sequence
of deltas, uploads, touched ticks (single and _many), full ticks, schedules, commits with HOLD / ERROR / PHASE entries, refused
commits, form changes, retirements and reshapes.  After every call both batches must agree byte for byte: return codes and
refusals, outs, arms, journals, state records, timer slots, and the lists of every touched tick.  The commit-due set is also
modelled on the host (the runs a touched tick evaluated, the runs a schedule changed, the runs entries named, the calls that
make the next touched commit full), and `full` and `n_considered` must be the model's, so a call that always went full fails.
Also: the edges of the list build (no due run, n_runs = 0, entries on runs that are not due, list lengths around the 8-warp
blocks and the 1024-CTA scan chunk) and the launch counts."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import commit as M
from bobrapet_b200.records import make_layout
from tests.test_gpu_commit import ALL, TABLES, _batch

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
FORMS = ("plain", "timed", "journal", "rewrites")


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _events_by_run(runs, head, events):
    """run -> its ready steps as a bit set, from a compact or touched tick's listed runs"""
    out, pos = {}, 0
    for r, hd in zip(runs, head):
        k = int(hd) >> 16
        ready = 0
        for e in events[pos:pos + k]:
            if (int(e) >> 10) & A.EVT_READY:
                ready |= 1 << (int(e) & 0x3FF)
        out[int(r)] = ready
        pos += k
    return out


class Twins:
    """batch A (full forms) and batch B (touched commits) with the same records and areas, and the host model of B's due set"""

    def __init__(self, fr, rng, S, fields, parallel, n, sched=False, timers=False, extra=5, stops=True):
        self.fr, self.rng = fr, rng
        self.ts, self.slots, self.L, self.st = _batch(fr, rng, S, fields, parallel, n, stops)
        self.fields = fields | (A.F_CHILD if self.L.off_child != A.OFF_NONE else 0)
        self.n, self.cap = n, n + extra
        self.topo = M.Topologies(self.ts, self.slots)
        self.h = [fr.resident_create(self.L, self.cap) for _ in range(2)]
        self.sched = {} if sched else None
        self.timers = timers
        for h in self.h:
            if n:
                fr.resident_upload(h, 0, self.st)
            if sched:
                fr.resident_sched(h)
                q = np.zeros(n, dtype=Frontier.SCHED_PUT_DTYPE)
                q["run"] = np.arange(n)
                q["story_key"] = np.arange(n) % 4
                q["queue_key"] = np.arange(n) % 3
                q["priority"] = np.arange(n) % 5
                q["queued_since"] = A.SCHED_NONE
                q["run_phase"] = A.PHASE_RUNNING
                if n:
                    fr.resident_sched_put(h, q)
            if timers:
                fr.resident_timers(h, 8)
        if timers:
            for i, slot in enumerate(self.slots[:4]):
                t = self.topo.by_slot[int(slot)]
                steps = [s for s in range(t["S"]) if (t["sync"] >> s) & 1][:3]
                if steps:
                    fr.put_timings(int(slot), [(s, A.DEC_FAIL, 10 + s) for s in steps])
        fr.resident_commit_marks(self.h[1])
        self.ready = {}
        self.touched = set(range(n))      # runs marked since they were last evaluated
        self.due, self.all, self.form = set(range(self.cap)), True, None
        self.now = 100
        self.commits = {"full": 0, "listed": 0, "refused": 0}
        self.snap = None   # earlier records (and timer slots) of A: what a resync from a stale cluster view sends back

    # -- the calls, on both batches
    def both(self, fn):
        return [fn(h) for h in self.h]

    def check_records(self):
        a, b = self.both(lambda h: self.fr.resident_download(h, 0, self.cap, self.L.state_stride))
        assert np.array_equal(a, b), np.nonzero(np.any(a != b, axis=1))[0][:10]
        if self.timers:
            ta, tb = self.both(lambda h: self.fr.resident_timers_download(h, 0, self.cap, 8))
            assert np.array_equal(ta, tb)
        return a

    def deltas(self, k):
        d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
        if self.n == 0 or k == 0:
            return d[:0]
        d["run"] = self.rng.integers(0, self.n, k)
        d["index"] = self.rng.integers(0, min(self.L.steps_max, 32), k)
        d["field"] = A.DELTA_PHASE
        d["code"] = self.rng.integers(0, 9, k)
        return d

    def touched_tick(self, d=NONE_D):
        a, b = self.both(lambda h: self.fr.resident_tick_touched(h, self.n, d, max(self.n, 1), BIG))
        for k in ("full", "n_listed", "n_evaluated", "n_events", "counts"):
            assert a[k] == b[k], (k, a[k], b[k])
        for k in ("runs", "head", "events"):
            assert np.array_equal(a[k], b[k]), k
        self._ticked(a, d)
        return a

    def touched_many(self, d=NONE_D):
        outs = self.fr.resident_tick_touched_many([dict(handle=h, n_runs=self.n, deltas=d, runs_cap=max(self.n, 1), events_cap=BIG)
                                                  for h in self.h])
        a, b = outs
        for k in ("full", "n_listed", "n_evaluated", "n_events"):
            assert a[k] == b[k], (k, a[k], b[k])
        for k in ("runs", "head", "events"):
            assert np.array_equal(a[k], b[k]), k
        self._ticked(a, d)

    def _ticked(self, out, d):
        self.touched |= {int(r) for r in d["run"]}
        if out["full"]:
            self.all, self.touched = True, set()
        else:
            ev = {r for r in self.touched if r < self.n}
            assert out["n_evaluated"] == len(ev), (out["n_evaluated"], len(ev))
            self.due |= ev
            self.touched -= ev
        self.ready.update(_events_by_run(out["runs"], out["head"], out["events"]))

    def full_tick(self, d=NONE_D):
        a, b = self.both(lambda h: self.fr.resident_tick_compact(h, self.n, d, BIG))
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2:] == b[2:]
        self.all, self.touched = True, set()
        self.ready.update(_events_by_run(range(self.n), a[0], a[1]))

    def schedule(self):
        if self.sched is None:
            return
        self.now += 1
        outs = [self.fr.resident_schedule([dict(handle=h, n_runs=self.n, runs_cap=self.n, events_cap=BIG)], TABLES, self.now)
                for h in self.h]
        pa, pb = outs[0]["parts"][0], outs[1]["parts"][0]
        for k in ("runs", "heads", "events"):
            assert np.array_equal(pa[k], pb[k]), k
        self.due |= {int(r) for r in pa["runs"]}
        M.sched_rows(self.L, pa, self.sched)

    def entries(self, state, p_hold=0.05, p_error=0.03, bogus=False):
        """random HOLD / ERROR entries on launched steps and a PHASE entry on every other launched stop step; with bogus one
        entry on a step that is not launched"""
        out = []
        for r in range(self.n):
            slot = int(state[r][:4].view("<u4")[0])
            t = self.topo.by_slot.get(slot)
            launched = (self.sched.get(r, (0, 0))[0] if self.sched is not None else self.ready.get(r, 0))
            if t is None or not launched:
                continue
            steps = [s for s in range(launched.bit_length()) if (launched >> s) & 1]
            named = {}
            if self.rng.random() < p_error:
                named[int(self.rng.choice(steps))] = (M.ERROR, 0)
            elif self.rng.random() < p_hold:
                named[int(self.rng.choice(steps))] = (M.HOLD, 0)
            for s in steps:
                if (t["stop"] >> s) & 1 and s not in named:
                    named[s] = (M.PHASE, int(self.rng.integers(A.PHASE_PENDING, A.PHASE_SKIPPED + 1)))
            out += [(r, s, k, c) for s, (k, c) in named.items()]
        if bogus and self.n:
            r = int(self.rng.integers(0, self.n))
            launched = self.sched.get(r, (0, 0))[0] if self.sched is not None else self.ready.get(r, 0)
            free = [s for s in range(self.L.steps_max) if not (launched >> s) & 1 and all((r, s) != (e[0], e[1]) for e in out)]
            if free:
                out.append((r, int(self.rng.choice(free)), M.HOLD, 0))
        self.rng.shuffle(out)
        return np.array(out, dtype=Frontier.COMMIT_DTYPE) if out else np.zeros(0, Frontier.COMMIT_DTYPE)

    def commit(self, form, ents=None, bogus=False, n=None):
        n = self.n if n is None else n
        before = self.check_records()
        if ents is None:
            ents = self.entries(before, bogus=bogus)
        kw = {}
        if form in ("timed", "journal", "rewrites") and self.timers:
            kw["now"] = self.now
        if form in ("journal", "rewrites"):
            kw["journal_cap"] = n * (32 * self.L.words + 64) + 1
        if form == "rewrites":
            kw["rewrites"] = True
        if form == "timed" and not self.timers:
            form = "plain"
        fkey = (kw.get("now") is not None, "journal_cap" in kw, kw.get("rewrites", False))
        got = []
        for h, touched in zip(self.h, (False, True)):
            try:
                got.append(self.fr.resident_commit(h, n, ents, touched=touched, **kw))
            except A.FrontierError as e:
                got.append((e.status, e.bad_run, e.bad_step))
        a, b = got
        after = self.check_records()
        if isinstance(a, tuple):
            assert a == b, (a, b)
            self.commits["refused"] += 1
            return None
        full, n_considered = b["full"], b["n_considered"]
        for k in a:
            if isinstance(a[k], np.ndarray):
                assert np.array_equal(a[k], b[k]), k
            else:
                assert a[k] == b[k], (k, a[k], b[k])
        if n == 0:
            assert (full, n_considered) == (0, 0)
            return b
        want_full = self.all or self.form != fkey
        named = {int(e["run"]) for e in ents}
        considered = set(range(n)) if want_full else ({r for r in self.due if r < n} | named)
        assert (full, n_considered) == (int(want_full), len(considered)), ((full, n_considered), (want_full, len(considered)))
        if want_full:
            self.due = set(range(self.cap))
        self.due = (self.due - considered) | named
        self.all, self.form = False, fkey
        self.commits["full" if want_full else "listed"] += 1
        written = set(np.nonzero(np.any(before != after, axis=1))[0].tolist())
        assert len(written) == a["n_runs_written"]
        self.touched |= written
        return b

    def upload(self, k):
        if self.n == 0 or self.st.shape[1] != self.L.state_stride:
            return
        first = int(self.rng.integers(0, self.n))
        k = min(k, self.n - first)
        for h in self.h:
            self.fr.resident_upload(h, first, self.st[first:first + k])
        self.touched |= set(range(first, first + k))

    def retire(self, k, capacity=0):
        if self.n <= k:
            return
        gone = np.sort(self.rng.choice(self.n, size=k, replace=False)).astype(np.uint32)
        (m, mf, mt), (mb, mfb, mtb) = [self.fr.resident_retire(h, self.n, gone, capacity) for h in self.h]
        if capacity:   # whole due words below the new capacity carry over, the rest of the new area is due
            self.due = {r for r in self.due if r < 32 * (capacity // 32)} | set(range(32 * (capacity // 32), capacity))
            self.cap = capacity
        assert m == mb and np.array_equal(mf, mfb) and np.array_equal(mt, mtb)
        moved = set(mt.tolist())
        self.touched = {r for r in self.touched if r < m} | moved
        self.n = m
        self.ready = {r: v for r, v in self.ready.items() if r < m and r not in moved}
        if self.sched is not None:
            self.sched.clear()

    def reshape(self, extra):
        self.cap += extra
        for h in self.h:
            self.fr.resident_reshape(h, self.L, self.cap)
        self.due |= set(range(32 * ((self.cap - extra) // 32), self.cap))

    def take_snapshot(self):
        st = self.fr.resident_download(self.h[0], 0, self.cap, self.L.state_stride)
        tm = self.fr.resident_timers_download(self.h[0], 0, self.cap, 8) if self.timers else None
        self.snap = (self.L.state_stride, st, tm)

    def fire(self):
        """bf_resident_fire at the next now: fired timers, decisions written, story timeouts; a written run is touched"""
        if not self.timers:
            return
        self.now += 7
        a, b = self.both(lambda h: self.fr.resident_fire(h, self.n, self.now))
        assert {k: a[k] for k in a if k != "fired"} == {k: b[k] for k in b if k != "fired"} and np.array_equal(a["fired"], b["fired"])
        f = a["fired"]
        self.touched |= {int(r) for r in f["run"][f["written"] != 0]}

    def redrive(self, k):
        """redrive k random runs from their first step (BF_REDRIVE_ALL) or one step: the redriven runs are touched"""
        if self.n == 0:
            return
        runs = np.sort(self.rng.choice(self.n, size=min(k, self.n), replace=False))
        state = self.check_records()
        q = np.zeros(runs.shape[0], dtype=Frontier.REDRIVE_DTYPE)
        q["run"] = runs
        q["slot"] = [int(state[r][:4].view("<u4")[0]) for r in runs]
        q["step"] = A.REDRIVE_ALL
        a, b = self.both(lambda h: self.fr.resident_redrive(h, q))
        assert np.array_equal(a[0], b[0]) and a[1] == b[1]
        self.touched |= {int(r) for r, ok in zip(q["run"], a[0]) if ok == 1}

    def resync(self, k):
        """resync k random runs to the earlier snapshot of their records: the drifted runs are repaired and touched"""
        if self.snap is None or self.snap[0] != self.L.state_stride or self.n == 0:
            return
        runs = np.sort(self.rng.choice(self.n, size=min(k, self.n), replace=False)).astype(np.uint32)
        recs = np.ascontiguousarray(self.snap[1][runs])
        a, b = self.both(lambda h: self.fr.resident_resync(h, self.n, recs, runs=runs))
        assert np.array_equal(a["drifted"], b["drifted"]) and a["n_written"] == b["n_written"]
        self.touched |= {int(r) for r in a["drifted"]}

    def resync_timers(self, k):
        """resync k random runs' timer slots to the earlier snapshot: timers come back or go, and no run is touched"""
        if not self.timers or self.snap is None or self.n == 0:
            return
        runs = np.sort(self.rng.choice(self.n, size=min(k, self.n), replace=False)).astype(np.uint32)
        tm = np.ascontiguousarray(self.snap[2][runs])
        a, b = self.both(lambda h: self.fr.resident_resync_areas(h, self.n, runs=runs, timers=tm))
        assert np.array_equal(a["drifted"], b["drifted"]) and np.array_equal(a["items"], b["items"])

    def retire_to(self, k):
        """retire k runs and shrink the capacity to the live runs plus a few: the due bits of whole words below it carry over"""
        if self.n <= k:
            return
        self.retire(k, capacity=self.n - k + 3)

    def reshape_layout(self):
        """reshape to a layout with every output field (a no-op layout change keeps the capacity path only)"""
        fields = self.fields | A.F_ALL_OUT
        L2 = make_layout(self.L.steps_max, self.L.child_nibbles, fields)
        for h in self.h:
            self.fr.resident_reshape(h, L2, self.cap + 2)
        self.due |= set(range(32 * (self.cap // 32), self.cap + 2))
        self.cap += 2
        self.L, self.fields = L2, fields

    def destroy(self):
        for h in self.h:
            self.fr.resident_destroy(h)


def _tick_and_schedule(tw, kind):
    d = tw.deltas(int(tw.rng.integers(0, 1 + max(tw.n // 50, 2))))
    if kind == "many":
        tw.touched_many(d)
    elif kind == "full":
        tw.full_tick(d)
    else:
        tw.touched_tick(d)
    tw.schedule()


# (S, fields, parallel, runs, limiter area, timers)
CASES = [(64, ALL, False, 700, False, True), (64, A.F_OUT_FAIL, True, 1500, True, False), (256, ALL, True, 3000, True, True),
         (256, A.F_DECISION | A.F_ALL_OUT, False, 2000, False, False), (1024, ALL, True, 300, True, True),
         (1024, A.F_ALL_OUT, False, 200, False, False)]


@pytest.mark.parametrize("S,fields,parallel,n,sched,timers", CASES)
def test_touched_commits_match_the_full_forms(fr, S, fields, parallel, n, sched, timers):
    rng = np.random.default_rng(9100 + S + n + fields)
    tw = Twins(fr, rng, S, fields, parallel, n, sched, timers)
    try:
        _tick_and_schedule(tw, "touched")
        form = FORMS[int(rng.integers(0, 4))]
        for step in range(40):
            if step % 10 == 3:
                tw.take_snapshot()
            op = rng.random()
            if op < 0.06:
                tw.upload(int(rng.integers(1, 20)))
            elif op < 0.09:
                tw.retire(int(rng.integers(1, 10)))
            elif op < 0.11:
                tw.retire_to(int(rng.integers(1, 10)))
            elif op < 0.13:
                tw.reshape(int(rng.integers(1, 40)))
            elif op < 0.14:
                tw.reshape_layout()
            elif op < 0.2:
                tw.redrive(int(rng.integers(1, 8)))
            elif op < 0.26:
                tw.resync(int(rng.integers(1, 30)))
            elif op < 0.32:
                tw.resync_timers(int(rng.integers(1, 30)))
            elif op < 0.37:
                form = FORMS[int(rng.integers(0, 4))]   # a form change makes the next touched commit full
            tw.fire()
            kind = "full" if rng.random() < 0.1 else "many" if rng.random() < 0.3 else "touched"
            _tick_and_schedule(tw, kind)
            tw.commit(form, bogus=rng.random() < 0.1)
        assert tw.commits["listed"] > 0 and tw.commits["full"] > 0, tw.commits
    finally:
        tw.destroy()


def test_touched_commit_edges(fr):
    rng = np.random.default_rng(77)
    tw = Twins(fr, rng, 64, ALL, False, 9000, stops=False)
    none = np.zeros(0, Frontier.COMMIT_DTYPE)
    try:
        _tick_and_schedule(tw, "touched")
        assert tw.commit("journal", ents=none)["full"] == 1   # the area was just enabled
        for _ in range(100):                                  # tick and commit until no run is due: no list, no write
            tw.touched_tick()
            got = tw.commit("journal", ents=none)
            assert got["full"] == 0
            if got["n_considered"] == 0:
                break
        assert got["n_considered"] == 0 and got["n_runs_written"] == 0 and got["n_items"] == 0
        tw.commit("journal", ents=none, n=0)                 # n_runs = 0: nothing considered (checked in commit)
        # entries on runs that are not due: a run that is not due has no launched step (its writes are in place), so such an
        # entry is refused by the full form; the touched form must list the named run and refuse with the same offender
        tw.touched_tick()
        quiet = sorted(r for r in range(tw.n) if r not in tw.due)
        assert len(quiet) > 10
        named = quiet[:: max(len(quiet) // 10, 1)][:10]
        ents = np.array([(r, 0, M.HOLD, 0) for r in named], dtype=Frontier.COMMIT_DTYPE)
        refused = tw.commits["refused"]
        assert tw.commit("journal", ents=ents) is None and tw.commits["refused"] == refused + 1
        # list lengths around the blocks of 8 and the 1024-CTA scan chunk: deltas on that many distinct runs
        for k in (1, 7, 8, 9, 8 * 1024 - 1, 8 * 1024, 8 * 1024 + 1):
            d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
            d["run"] = np.sort(rng.choice(tw.n, size=k, replace=False))
            d["index"] = 0
            d["field"] = A.DELTA_PHASE
            d["code"] = rng.integers(0, 9, k)
            tw.touched_tick(d)
            tw.commit("journal")
    finally:
        tw.destroy()


def test_launch_counts(fr):
    """a batch without the area launches what it did in every call; with it, each call launches what the header documents"""
    rng = np.random.default_rng(5)
    ts, slots, L, st = _batch(fr, rng, 64, ALL, False, 500, stops=False)
    h = fr.resident_create(L, 500)
    fr.resident_upload(h, 0, st)
    fr.resident_timers(h, 4)
    fr.resident_sched(h)
    q = np.zeros(500, dtype=Frontier.SCHED_PUT_DTYPE)
    q["run"] = np.arange(500)
    q["queued_since"] = A.SCHED_NONE
    q["run_phase"] = A.PHASE_RUNNING
    fr.resident_sched_put(h, q)
    part = [dict(handle=h, n_runs=500, runs_cap=500, events_cap=BIG)]
    d = np.zeros(3, dtype=Frontier.DELTA_DTYPE)
    d["run"] = [1, 2, 3]
    d["field"] = A.DELTA_PHASE

    def launches(fn):
        k = fr.stats()["kernel_launches"]
        fn()
        return fr.stats()["kernel_launches"] - k

    def tick(code, with_area):
        d["code"] = code
        assert launches(lambda: fr.resident_tick_touched(h, 500, d, 500, BIG)) == 6 + with_area   # scatter, list pair, pass, compaction pair
        assert launches(lambda: fr.resident_schedule(part, TABLES, 100)) == 5 + with_area          # init, count, limit, scan, list

    forms = [dict(), dict(now=100), dict(journal_cap=1000), dict(journal_cap=1000, rewrites=True)]
    try:
        fr.resident_tick_touched(h, 500, NONE_D, 500, BIG)
        code = 0
        for kw, n in zip(forms, (2, 2, 3, 4)):   # the full forms without the area, as tests/test_gpu_commit*.py count them
            code += 1
            tick(code, 0)
            assert launches(lambda: fr.resident_commit(h, 500, **kw)) == n
        fr.resident_commit_marks(h)
        for kw, n in zip(forms, (2, 2, 3, 4)):   # with it: the form's launches when full (the area was just enabled, then a
            for full in (True, False):           # form change), 3 more (count, scan, list) when the call lists its due runs
                code += 1
                tick(code, 1)
                assert launches(lambda: fr.resident_commit(h, 500, touched=True, **kw)) == n + (0 if full else 3), (kw, full)
    finally:
        fr.resident_destroy(h)
