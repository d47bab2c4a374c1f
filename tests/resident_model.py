"""A host model of resident batches: every lifecycle call (upload, deltas, the five tick kinds, migrate, redrive, reshape,
retire, topology put / drop, bf_schedule) restated in numpy from include/bobrafrontier.h, with no GPU call.

The model holds what the contract makes observable: per ctx the slot registry (live slots, the LIFO free list, the next new
index, the slot changes a touched tick must notice) and the snapshot bf_schedule refers to; per batch the layout, the state
records, the current result records (those changed-only and touched ticks compare with), the touched and must-list runs, and
the touched-tick baseline (run count of the last full evaluation, runs uploaded since, the flags and iteration cap of the last
tick, whether a reshape forced a full tick, whether a changed-only tick can compare and over how many runs).  From that it
predicts every output of every call, the `full` flag of touched ticks included, and which calls are refused.
"""
from __future__ import annotations

import numpy as np

from bobrapet_b200 import _abi as A
from oracle import packed as PK
from tests import redrive as RD
from tests import reshape as RS
from tests import retire as RT
from tests.packing import topology_set

NONE_OFF = A.OFF_NONE


class Refused(Exception):
    """a call the contract refuses, with the status it must return; the call changes nothing"""

    def __init__(self, status, why):
        super().__init__("%d: %s" % (status, why))
        self.status = status


def _fits(L, ps):
    return ps.S <= L.steps_max and (L.off_child == NONE_OFF or ps.child_nibbles() <= L.child_nibbles)


class Registry:
    """the topology slots of one ctx over a pool of PackedStory objects (tests/packing.py)"""

    def __init__(self, stories):
        self.stories = list(stories)
        self.ts = topology_set(self.stories)
        self.pt = PK.PackedTopologies(self.ts)      # row k of its table: pool story k (the pointers stay valid with self.ts)
        self.live = {}                              # slot -> pool index
        self.free = []                              # dropped slots, the last one on top
        self.n_index = 0                            # slot indices ever created
        self.changes = 0                            # drops and reuses: each one changes what the runs on the slot evaluate to
        self.last = None                            # (batch, n_runs) of the pass bf_schedule refers to

    def put(self, k):
        if self.free:
            slot = self.free.pop()
            self.changes += 1
        else:
            slot = self.n_index
            self.n_index += 1
        self.live[slot] = k
        return slot

    def drop(self, slot):
        if slot not in self.live:
            raise Refused(A.BF_ETOPO, "drop of an unknown slot")
        del self.live[slot]
        self.free.append(slot)
        self.changes += 1

    def story(self, slot):
        return self.stories[self.live[slot]]

    def evaluate(self, L, state, flags, max_iter):
        """-> (result records, counts) of a pass over `state`: runs on a slot that is not alive are dead (summary all ones, no
        bits, counted nowhere)"""
        n = state.shape[0]
        slots = np.ascontiguousarray(state[:, 0:4]).view("<u4").reshape(n)
        live = np.isin(slots, np.fromiter(self.live, np.int64, len(self.live)))
        res = np.zeros((n, L.result_stride), np.uint8)
        counts = dict(ready=0, skip=0, expansion=0, evals=0)
        if live.any():
            view = PK.PackedTopologies.__new__(PK.PackedTopologies)
            view.n_slots = max(self.live) + 1
            view.table = np.zeros(view.n_slots, PK.ORC_TOPO_DTYPE)
            for s, k in self.live.items():
                view.table[s] = self.pt.table[k]
            idx = np.nonzero(live)[0]
            res[idx], counts = PK.evaluate(view, L, np.ascontiguousarray(state[idx]), flags & A.EVAL_FIXPOINT, max_iter, threads=8)
        res[~live, 0:4] = 0xFF
        return res, counts


def _set_plane(rec, off, W, nbits, idx, code):
    words = rec[off:off + nbits * W * 4].view("<u4")
    for b in range(nbits):
        w = b * W + idx // 32
        words[w] = (int(words[w]) & ~(1 << (idx % 32))) | (((code >> b) & 1) << (idx % 32))


def _get_plane(rec, off, W, nbits, S):
    from bobrapet_b200.records import _unpack_planes
    return _unpack_planes(rec[None, off:off + nbits * W * 4], W, nbits, S)[0]


def _nibble(rec, off, i, code=None):
    b, sh = off + i // 2, 4 * (i & 1)
    if code is None:
        return (int(rec[b]) >> sh) & 0xF
    rec[b] = (int(rec[b]) & ~(0xF << sh) & 0xFF) | ((code & 0xF) << sh)


class Batch:
    """one resident batch of a ctx"""

    def __init__(self, reg, L, cap):
        self.reg, self.L, self.cap = reg, L, cap
        self.state = np.zeros((cap, L.state_stride), np.uint8)
        self.cur = np.zeros((cap, L.result_stride), np.uint8)
        self.touched, self.must = set(), set()
        self.full_runs, self.uploaded = 0, set()
        self.need_full, self.last_fix, self.last_max, self.changes_seen = True, 0, 0, 0
        self.prev_valid, self.prev_runs = False, 0

    def _end_snapshot(self):
        if self.reg.last and self.reg.last[0] is self:
            self.reg.last = None

    # ------------------------------------------------------------------ state
    def upload(self, first, recs):
        n = recs.shape[0]
        if first + n > self.cap:
            raise Refused(A.BF_EINVAL, "run range outside the resident batch")
        if n == 0:
            return
        self._end_snapshot()
        self.prev_valid = False
        self.state[first:first + n] = recs
        rr = set(range(first, first + n))
        self.touched |= rr
        self.must |= rr
        self.uploaded |= set(range(max(first, self.full_runs), first + n))

    def apply(self, d):
        """valid deltas only (the generators draw no rejected ones)"""
        if len(d) == 0:
            return
        self._end_snapshot()
        L, W = self.L, self.L.words
        for run, idx, f, code in zip(d["run"].tolist(), d["index"].tolist(), d["field"].tolist(), d["code"].tolist()):
            rec = self.state[run]
            if f == A.DELTA_PHASE:
                _set_plane(rec, L.off_phase, W, 4, idx, code)
            elif f == A.DELTA_COND:
                _set_plane(rec, L.off_cond, W, 2, idx, code)
            elif f == A.DELTA_DECISION:
                _set_plane(rec, L.off_decision, W, 2, idx, code)
            elif f == A.DELTA_CHILD:
                _nibble(rec, L.off_child, idx, code)
            elif f == A.DELTA_RUN_FLAGS:
                rec[4] = code
            elif f == A.DELTA_REGISTERED:
                v = rec[8:16].view("<u8")
                v[0] = (int(v[0]) & ~(1 << idx)) | (code << idx)
            elif f == A.DELTA_TOPO_SLOT:
                rec[0:4] = np.array([idx | (code << 16)], "<u4").view(np.uint8)
            else:
                raise AssertionError(f)
            self.touched.add(run)

    def slots(self, n):
        return np.ascontiguousarray(self.state[:n, 0:4]).view("<u4").reshape(n)

    # ------------------------------------------------------------------ ticks
    def _full(self, n_runs, flags, max_iter):
        res, counts = self.reg.evaluate(self.L, self.state[:n_runs], flags, max_iter)
        self.prev_valid, self.prev_runs = True, n_runs
        self.need_full, self.full_runs = False, n_runs
        self.last_fix, self.last_max, self.changes_seen = flags & A.EVAL_FIXPOINT, max_iter, self.reg.changes
        self.uploaded = set()
        self.touched, self.must = set(), set()
        self.reg.last = (self, n_runs)
        return res, counts

    def tick(self, d, n_runs, flags=0, max_iter=0):
        """bf_resident_tick / _eval (d empty) -> (result records, counts)"""
        self.reg.last = None
        if n_runs > self.cap:
            raise Refused(A.BF_EINVAL, "n_runs exceeds the resident batch")
        self.apply(d)
        res, counts = self._full(n_runs, flags, max_iter)
        self.cur[:n_runs] = res
        return res, counts

    def tick_compact(self, d, n_runs, flags=0, max_iter=0):
        """bf_resident_tick_compact -> (head, events, n_listed, counts); flags may carry BF_EVAL_CHANGED_ONLY"""
        self.reg.last = None
        if n_runs > self.cap:
            raise Refused(A.BF_EINVAL, "n_runs exceeds the resident batch")
        changed = bool(flags & A.EVAL_CHANGED_ONLY)
        compare = changed and self.prev_valid and self.prev_runs == n_runs
        prev = self.cur[:n_runs].copy() if compare else None
        self.apply(d)
        res, counts = self._full(n_runs, flags & ~A.EVAL_CHANGED_ONLY, max_iter)
        head, ev, listed = PK.compact_events(self.L, res, prev)
        self.cur[:n_runs] = res
        return head, ev, listed, counts

    def full_due(self, n_runs, flags, max_iter):
        """would a touched tick over n_runs with these parameters evaluate and list every run?"""
        covered = all(i in self.uploaded for i in range(self.full_runs, n_runs))
        return (self.need_full or self.reg.changes != self.changes_seen or (flags & A.EVAL_FIXPOINT) != self.last_fix or
                max_iter != self.last_max or (n_runs > self.full_runs and not covered))

    def tick_touched(self, d, n_runs, flags=0, max_iter=0):
        """bf_resident_tick_touched -> dict(full, runs, head, events, n_listed, n_evaluated, counts) before the caps"""
        if flags & ~(A.EVAL_FIXPOINT | A.EVAL_NO_COUNTS):
            raise Refused(A.BF_EINVAL, "touched ticks take BF_EVAL_FIXPOINT and BF_EVAL_NO_COUNTS only")
        if n_runs > self.cap:
            raise Refused(A.BF_EINVAL, "n_runs exceeds the resident batch")
        if self.full_due(n_runs, flags, max_iter):
            head, ev, _, counts = self.tick_compact(d, n_runs, flags & A.EVAL_FIXPOINT, max_iter)
            return dict(full=1, runs=np.arange(n_runs, dtype=np.uint32), head=head, events=ev, n_evaluated=n_runs, counts=counts)
        self.reg.last = None
        self.apply(d)
        want, _ = self.reg.evaluate(self.L, self.state[:n_runs], flags, max_iter)
        evaluated = sorted(r for r in self.touched if r < n_runs)
        listed = np.array([r for r in evaluated if r in self.must or not np.array_equal(want[r], self.cur[r])], np.int64)
        head, ev, _ = PK.compact_events(self.L, want[listed])
        ix = np.array(evaluated, np.int64)
        _, counts = self.reg.evaluate(self.L, np.ascontiguousarray(self.state[ix]), flags, max_iter)
        self.cur[ix] = want[ix]
        self.touched -= set(evaluated)
        self.must -= set(evaluated)
        self.reg.last = (self, n_runs)
        return dict(full=0, runs=listed.astype(np.uint32), head=head, events=ev, n_evaluated=len(evaluated), counts=counts)

    def schedule_ok(self, n_runs):
        return self.reg.last == (self, n_runs)

    # ------------------------------------------------------------------ lifecycle
    def migrate(self, old, new, step_map, n_runs):
        """bf_resident_migrate -> runs migrated"""
        reg, L, W = self.reg, self.L, self.L.words
        if n_runs > self.cap:
            raise Refused(A.BF_EINVAL, "n_runs exceeds the resident batch")
        if old not in reg.live or new not in reg.live:
            raise Refused(A.BF_ETOPO, "migration between unknown topology slots")
        if old == new:
            raise Refused(A.BF_EINVAL, "migration from a slot to itself")
        po, pn = reg.story(old), reg.story(new)
        if len(step_map) != po.S:
            raise Refused(A.BF_EINVAL, "step_map length")
        if not (_fits(L, po) and _fits(L, pn)):
            raise Refused(A.BF_ETOPO, "topology does not fit the batch layout")
        inv = {}
        for i, t in enumerate(int(x) for x in step_map):
            if t == A.MIGRATE_GONE:
                continue
            if t >= pn.S or t in inv:
                raise Refused(A.BF_EINVAL, "step_map")
            inv[t] = i
        descs = []   # (old desc, new desc, branches)
        for q, stp in enumerate(pn.par_steps):
            o = inv.get(stp)
            if o is None or o not in po.par_steps:
                continue
            p = po.par_steps.index(o)
            if len(po.par_branches[p]) != len(pn.par_branches[q]):
                raise Refused(A.BF_EINVAL, "parallel step changes its branch count")
            descs.append((p, q, len(pn.par_branches[q])))
        self._end_snapshot()
        on = np.nonzero(self.slots(n_runs) == old)[0]
        cfo, cfn = po.child_first(), pn.child_first()
        for r in on.tolist():
            rec = self.state[r]
            for off, nbits in ((L.off_phase, 4), (L.off_cond, 2), (L.off_decision, 2)):
                if off == NONE_OFF:
                    continue
                codes = _get_plane(rec, off, W, nbits, 32 * W)
                rec[off:off + nbits * W * 4] = 0
                for t, i in inv.items():
                    _set_plane(rec, off, W, nbits, t, int(codes[i]))
            reg_old = int(rec[8:16].view("<u8")[0])
            reg_new = 0
            kids = []
            for p, q, b in descs:
                reg_new |= ((reg_old >> p) & 1) << q
                if L.off_child != NONE_OFF:
                    kids.append((q, [_nibble(rec, L.off_child, int(cfo[p]) + k) for k in range(b)]))
            if L.off_child != NONE_OFF:
                for i in range(L.child_nibbles):
                    _nibble(rec, L.off_child, i, 0)
                for q, ks in kids:
                    for k, v in enumerate(ks):
                        _nibble(rec, L.off_child, int(cfn[q]) + k, v)
            rec[8:16] = np.array([reg_new], "<u8").view(np.uint8)
            rec[0:4] = np.array([new], "<u4").view(np.uint8)
        self.touched |= set(on.tolist())
        self.must |= set(on.tolist())
        return len(on)

    def redrive(self, req):
        """bf_resident_redrive(requests of Frontier.REDRIVE_DTYPE) -> (status, applied)"""
        reg, L = self.reg, self.L
        for q in req:
            if int(q["run"]) >= self.cap:
                raise Refused(A.BF_EINVAL, "run outside the resident batch")
            if int(q["reserved"]):
                raise Refused(A.BF_EINVAL, "reserved")
            if int(q["slot"]) not in reg.live:
                raise Refused(A.BF_ETOPO, "unknown topology slot")
            ps = reg.story(int(q["slot"]))
            if int(q["step"]) != A.REDRIVE_ALL and int(q["step"]) >= ps.S:
                raise Refused(A.BF_EINVAL, "step index out of range")
            if not _fits(L, ps):
                raise Refused(A.BF_ETOPO, "topology does not fit the batch layout")
        if len(req) == 0:
            return np.zeros(0, np.uint8), 0
        self._end_snapshot()
        status = np.zeros(len(req), np.uint8)
        for i, q in enumerate(req):
            run, slot, step = int(q["run"]), int(q["slot"]), int(q["step"])
            if int(self.state[run, 0:4].view("<u4")[0]) != slot:
                continue
            status[i] = 1
            RD.reset_packed(L, self.state[run], reg.story(slot), None if step == A.REDRIVE_ALL else step)
            self.touched.add(run)
        return status, int(status.sum())

    def reshape(self, T, capacity):
        F = self.L
        if capacity < self.cap:
            raise Refused(A.BF_EINVAL, "reshape cannot lower the capacity")
        if T.steps_max < F.steps_max or F.fields & ~T.fields:
            raise Refused(A.BF_EINVAL, "reshape cannot lower steps_max or drop a field")
        if F.off_child != NONE_OFF and T.child_nibbles < F.child_nibbles:
            raise Refused(A.BF_EINVAL, "reshape cannot shrink the child area")
        added = [n for n in ("off_decision", "off_fail", "off_needs_cond", "off_skip_dep", "off_phase_out")
                 if getattr(F, n) == NONE_OFF and getattr(T, n) != NONE_OFF]
        self._end_snapshot()
        self.state = RS.reshape_state(F, T, self.state, capacity)
        self.cur = RS.reshape_result(F, T, self.cur, capacity)
        self.L, self.cap = T, capacity
        if added:
            self.need_full = True

    def retire(self, n_runs, runs, capacity=0):
        """-> (m, moves_from, moves_to)"""
        if n_runs > self.cap:
            raise Refused(A.BF_EINVAL, "n_runs exceeds the resident batch")
        runs = [int(r) for r in runs]
        if any(r >= n_runs for r in runs) or len(set(runs)) != len(runs):
            raise Refused(A.BF_EINVAL, "runs")
        m = n_runs - len(runs)
        cap = capacity or self.cap
        if cap < m or cap > self.cap:
            raise Refused(A.BF_EINVAL, "capacity")
        if not runs and cap == self.cap:
            return m, np.zeros(0, np.uint32), np.zeros(0, np.uint32)
        self._end_snapshot()
        _, src, dst = RT.moves(n_runs, runs)
        self.state = RT.retire_records(self.state, n_runs, runs, cap)
        cur = self.cur.copy()
        cur[dst] = self.cur[src]
        self.cur = cur[:cap]
        gone = set(range(m, n_runs)) | set(range(cap, self.cap))
        self.touched = (self.touched - gone) | set(dst.tolist())
        self.must = (self.must - gone) | set(dst.tolist())
        self.cap = cap
        self.full_runs = min(self.full_runs, m)
        self.uploaded = {i for i in self.uploaded if i < m} | {int(t) for t in dst if t >= self.full_runs}
        if self.prev_valid and self.prev_runs == n_runs:
            self.prev_runs = m
        else:
            self.prev_valid = False
        return m, src, dst
