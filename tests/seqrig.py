"""A ctx, its batches and the host model of tests/resident_model.py side by side: every call goes to both, and every output and
the device state are compared after it.  Used by the random sequences and the directed cases of test_gpu_resident_sequences.py."""
from __future__ import annotations

import zlib
from collections import Counter

import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout, pack_state
from tests import migration as M
from tests import redrive as RD
from tests import resident_model as RM
from tests import schedref as SR
from tests.packing import topology_set

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
TICK_KINDS = ("dense", "eval", "compact", "changed", "touched")


def story_pool(rng, s_lo, s_hi, n_par, n_base, n_spare=2):
    """n_base Stories, one edit of each (pool index n_base + k edits Story k), and n_spare small Stories for slot churn"""
    base = [RD.random_story(rng, "t%d-" % k, int(rng.integers(s_lo, s_hi + 1)), n_par) for k in range(n_base)]
    edits = [M.edit_story(rng, s, "t%d-e" % k, parallel=n_par > 0) for k, s in enumerate(base)]
    spare = [RD.random_story(rng, "x%d-" % k, int(rng.integers(5, 40)), min(n_par, 1)) for k in range(n_spare)]
    return [RD.packed_story(s) for s in base + edits + spare]


def layout_for(stories, fields):
    child = max(p.child_nibbles() for p in stories) if fields & A.F_CHILD else 0
    return make_layout(max(p.S for p in stories), child, fields)


def random_records(rng, L, stories, slots):
    """state records of runs on the given stories / slots: progress-shaped phases, every code the layout holds"""
    n, W32 = len(stories), 32 * L.words
    phase, cond, dec = (np.zeros((n, W32), np.uint8) for _ in range(3))
    child = np.zeros((n, max(L.child_nibbles, 1)), np.uint8)
    reg = np.zeros(n, np.uint64)
    for r, ps in enumerate(stories):
        S = ps.S
        prog = int(rng.integers(0, S + 1))
        phase[r, :prog] = rng.choice([3, 13, 4, 2, 8, 1], size=prog, p=[0.75, 0.05, 0.05, 0.08, 0.04, 0.03])
        phase[r, prog:S] = rng.choice([0, 14, 9], size=S - prog, p=[0.9, 0.06, 0.04])
        cond[r, :S] = rng.choice(4, size=S, p=[0.55, 0.2, 0.15, 0.1])
        dec[r, :S] = rng.integers(0, 4, size=S)
        cf = ps.child_first()
        for q in range(len(ps.par_steps)):
            if rng.random() < 0.6:
                reg[r] |= np.uint64(1) << np.uint64(q)
            if L.off_child != A.OFF_NONE:
                b = len(ps.par_branches[q])
                child[r, int(cf[q]):int(cf[q]) + b] = rng.choice([0, 2, 3, 3, 3, 4, 13], size=b)
    rflags = (rng.random(n) < 0.5).astype(np.uint8) * A.RF_FAIL_FAST | (rng.random(n) < 0.2).astype(np.uint8) * A.RF_TOPOLOGY_TERMINATED
    return pack_state(L, np.asarray(slots, np.uint32), rflags, phase, cond if L.off_cond != A.OFF_NONE else None,
                      dec if L.off_decision != A.OFF_NONE else None, child if L.off_child != A.OFF_NONE else None, reg)


class Rig:
    """one ctx and its model; batches are addressed by their model (RM.Batch) objects"""

    def __init__(self, fr, stories, label=""):
        self.fr, self.reg = fr, RM.Registry(stories)
        self.ts1 = [topology_set([p]) for p in stories]   # one TopologySet per pool Story, for bf_topology_put
        self.handles = {}
        self.log, self.label = [], label
        # schedules: their own generator (the drivers' draws stay as they were), the last accepted tick as (batch, n_runs, kind,
        # the call before it), and the compared schedules counted by that tick's kind and by the call before the tick
        self.srng = np.random.default_rng(zlib.crc32(label.encode()))
        self.prior, self.after = None, None
        self.compared = Counter()
        self.rotation = 0

    # -------------------------------------------------------------- failure reports name the sequence
    def where(self):
        return "%s op %d\n  %s" % (self.label, len(self.log) - 1, "\n  ".join(self.log[-60:]))

    def check(self, cond, what):
        if not cond:
            raise AssertionError("%s: %s" % (what, self.where()))

    def _call(self, dev, model):
        """run the model, then the device; a call the model refuses must fail on the device with the same status"""
        try:
            want = model()
        except RM.Refused as e:
            try:
                dev()
            except A.FrontierError as d:
                self.check(d.status == e.status, "status %d, want %d (%s)" % (d.status, e.status, e))
                return None, True
            self.check(False, "the device accepted a call the contract refuses (%s)" % e)
        try:
            got = dev()
        except A.FrontierError as d:
            self.check(False, "the device refused a valid call: %s" % d)
        return (got, want), False

    def sync(self):
        """every batch's device state equals the model's"""
        for b, h in self.handles.items():
            st = self.fr.resident_download(h, 0, b.cap, b.L.state_stride)
            if not np.array_equal(st, b.state):
                bad = np.nonzero((st != b.state).any(axis=1))[0]
                self.check(False, "device state differs from the model in runs %s" % bad[:10].tolist())

    # -------------------------------------------------------------- topologies
    def put(self, k):
        self.log.append("put story %d" % k)
        slot = int(self.fr.put_topologies(self.ts1[k])[0])
        want = self.reg.put(k)
        self.check(slot == want, "put returned slot %d, want %d" % (slot, want))
        return slot

    def drop(self, slot):
        self.log.append("drop %d" % slot)
        self._call(lambda: self.fr.drop_topology(slot), lambda: self.reg.drop(slot))

    # -------------------------------------------------------------- batches
    def create(self, L, cap):
        b = RM.Batch(self.reg, L, cap)
        self.handles[b] = self.fr.resident_create(L, cap)
        self.log.append("create batch %d cap %d S %d" % (self.handles[b], cap, L.steps_max))
        return b

    def destroy(self):
        for h in self.handles.values():
            self.fr.resident_destroy(h)
        self.handles = {}

    def upload(self, b, first, recs):
        self.log.append("upload b%d [%d, %d)" % (self.handles[b], first, first + recs.shape[0]))
        self._call(lambda: self.fr.resident_upload(self.handles[b], first, recs), lambda: b.upload(first, recs))
        self.sync()

    def apply(self, b, d):
        self.log.append("apply b%d %d deltas" % (self.handles[b], len(d)))
        self._call(lambda: self.fr.resident_apply(self.handles[b], d), lambda: b.apply(d))
        self.sync()

    def tick(self, b, kind, n_runs, d=NONE, flags=0, max_iter=0, runs_cap=None, events_cap=None, pinned=False):
        """kind: dense / eval / compact / changed / touched -> the touched tick's output dict (touched), else None"""
        h, fr = self.handles[b], self.fr
        before = self.after or (self.log[-1].split()[0] if self.log else "start")
        self.after = None
        self.log.append("%s b%d n %d deltas %d flags %d iter %d caps %s/%s%s" % (kind, h, n_runs, len(d), flags, max_iter, runs_cap,
                                                                          events_cap, " pinned" if pinned else ""))
        out, r = None, None
        if kind in ("dense", "eval"):
            if kind == "dense":
                r, _ = self._call(lambda: fr.resident_tick(h, b.L, n_runs, d, flags=flags, max_iterations=max_iter),
                                  lambda: b.tick(d, n_runs, flags, max_iter))
            else:
                if len(d):
                    self.apply(b, d)
                r, _ = self._call(lambda: fr.resident_eval(h, b.L, n_runs, flags=flags, max_iterations=max_iter),
                                  lambda: b.tick(NONE, n_runs, flags, max_iter))
            if r:
                (res, counts), (wres, wcounts) = r
                self.check(np.array_equal(res, wres), "result records differ")
                self.check(counts == wcounts, "counts %s, want %s" % (counts, wcounts))
        elif kind in ("compact", "changed"):
            fl = flags | (A.EVAL_CHANGED_ONLY if kind == "changed" else 0)
            r, _ = self._call(lambda: fr.resident_tick_compact(h, n_runs, d, 4_000_000, flags=fl, max_iterations=max_iter),
                              lambda: b.tick_compact(d, n_runs, fl, max_iter))
            if r:
                (head, ev, n_ev, counts, listed), (whead, wev, wlisted, wcounts) = r
                self.check(np.array_equal(head, whead), "heads differ in runs %s" % np.nonzero(head != whead)[0][:10].tolist())
                self.check(n_ev == len(wev) and np.array_equal(ev, wev), "events differ")
                self.check(listed == wlisted and counts == wcounts, "listed %d / %s, want %d / %s" % (listed, counts, wlisted, wcounts))
        else:
            runs_cap = n_runs if runs_cap is None else runs_cap
            events_cap = 4_000_000 if events_cap is None else events_cap
            bufs = {}
            if pinned:
                bufs = {"runs": fr.alloc_pinned(max(runs_cap, 1) * 4).view(np.uint32),
                        "head": fr.alloc_pinned(max(runs_cap, 1) * 4).view(np.uint32),
                        "events": fr.alloc_pinned(max(events_cap, 1) * 2).view(np.uint16)}

            def dev():
                o = fr.resident_tick_touched(h, n_runs, d, runs_cap, events_cap, flags=flags, max_iterations=max_iter, **bufs)
                return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in o.items()}
            try:
                r, _ = self._call(dev, lambda: b.tick_touched(d, n_runs, flags, max_iter))
            finally:
                for v in bufs.values():
                    fr.free_pinned(v.view(np.uint8))
            if r:
                out, want = r
                self.check(out["full"] == want["full"], "touched full = %d, the model says %d" % (out["full"], want["full"]))
                self.check(out["n_listed"] == len(want["runs"]) and out["n_evaluated"] == want["n_evaluated"],
                           "listed / evaluated %d / %d, want %d / %d" % (out["n_listed"], out["n_evaluated"], len(want["runs"]),
                                                                         want["n_evaluated"]))
                self.check(np.array_equal(out["runs"], want["runs"][:runs_cap]),
                           "listed runs %s, want %s" % (out["runs"][:12].tolist(), want["runs"][:12].tolist()))
                self.check(np.array_equal(out["head"], want["head"][:runs_cap]), "touched heads differ")
                self.check(out["n_events"] == len(want["events"]) and np.array_equal(out["events"], want["events"][:events_cap]),
                           "touched events differ")
                if not flags & A.EVAL_NO_COUNTS:
                    self.check(out["counts"] == want["counts"], "counts %s, want %s" % (out["counts"], want["counts"]))
        if r:
            self.prior = (b, n_runs, kind, before)
        self.sync()
        return out

    def schedule(self, b, n_runs):
        """bf_schedule with random sched runs and tables (tests/schedref.py generators); accepted or refused as the model says, and
        when accepted, equal to the reference over the model's current result and state records"""
        g = self.srng
        ns, nq = int(g.choice([0, 1, 7, 40, 600])), int(g.choice([0, 1, 3, 9, 300]))
        sched = SR.random_sched(g, n_runs, ns, nq, out_of_range=float(g.choice([0.0, 0.05])))
        tables = SR.random_tables(g, ns, nq, n_runs, maxprio_base=bool(g.random() < 0.5))
        self.log.append("schedule b%d n %d tables %d/%d" % (self.handles[b], n_runs, ns, nq))
        ok = b.schedule_ok(n_runs)
        try:
            got = self.fr.schedule(b.L, n_runs, sched, **tables)
        except A.FrontierError:
            got = None
        self.check((got is not None) == ok, "bf_schedule %s, the model says %s" % ("accepted" if got is not None else "refused",
                                                                                    "accept" if ok else "refuse"))
        if got is None:
            return
        want = SR.expected(b.L, b.state[:n_runs], b.cur[:n_runs], SR.from_registry(self.reg), sched, tables)
        try:
            SR.assert_schedule(got, want)
        except AssertionError as e:
            self.check(False, str(e))
        _, _, kind, before = self.prior
        self.compared["tick " + kind] += 1
        self.compared["after " + before] += 1

    def tick_and_schedule(self, b, n_runs, after, flags=0, max_iter=0):
        """a tick of the next kind in turn (no deltas) over the batch, then a schedule compared after it and counted as following
        the call `after`"""
        kind = TICK_KINDS[self.rotation % len(TICK_KINDS)]
        self.rotation += 1
        self.after = after
        self.tick(b, kind, n_runs, NONE, flags, max_iter)
        self.schedule_last()

    def schedule_last(self):
        """bf_schedule over the batch and n_runs of the last accepted tick (accepted unless a call since ended the snapshot)"""
        if self.prior is not None:
            self.schedule(*self.prior[:2])

    def migrate(self, b, old, new, n_runs):
        ps_old, ps_new = self.reg.stories[self.reg.live[old]], self.reg.stories[self.reg.live[new]] if new in self.reg.live else None
        smap = M.migration_map(ps_old, ps_new)[0] if ps_new is not None else np.arange(ps_old.S, dtype=np.uint16)
        self.log.append("migrate b%d %d -> %d n %d" % (self.handles[b], old, new, n_runs))
        r, refused = self._call(lambda: self.fr.resident_migrate(self.handles[b], old, new, smap, n_runs),
                                lambda: b.migrate(old, new, smap, n_runs))
        if r:
            self.check(r[0] == r[1], "migrated %d runs, want %d" % r)
        self.sync()
        return None if refused else r[1]

    def redrive(self, b, req):
        self.log.append("redrive b%d %d requests" % (self.handles[b], len(req)))
        r, _ = self._call(lambda: self.fr.resident_redrive(self.handles[b], req), lambda: b.redrive(req))
        if r:
            (st, ap), (wst, wap) = r
            self.check(np.array_equal(st, wst) and ap == wap, "redrive statuses differ")
        self.sync()

    def reshape(self, b, T, cap):
        self.log.append("reshape b%d S %d -> %d child %d fields %#x cap %d -> %d" % (self.handles[b], b.L.steps_max, T.steps_max,
                                                                                   T.child_nibbles, T.fields, b.cap, cap))
        self._call(lambda: self.fr.resident_reshape(self.handles[b], T, cap), lambda: b.reshape(T, cap))
        self.sync()

    def retire(self, b, n_runs, runs, cap=0):
        self.log.append("retire b%d n %d retire %d cap %d" % (self.handles[b], n_runs, len(runs), cap))
        r, refused = self._call(lambda: self.fr.resident_retire(self.handles[b], n_runs, np.asarray(runs, np.uint32), cap),
                                lambda: b.retire(n_runs, runs, cap))
        if r:
            (m, mf, mt), (wm, wf, wt) = r
            self.check(m == wm and np.array_equal(mf, wf) and np.array_equal(mt, wt), "retire moves differ")
        self.sync()
        return None if refused else r[1][0]
