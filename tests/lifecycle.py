"""One host model of a resident batch with every per-run side area at once: its state records, its step-timer slots
(tests/timers.py), its limiter inputs and schedule baselines (tests/sched_resident.py) and its run-control records
(tests/runctl.py), each present or absent (an area set, a subset of TIMERS | SCHED | RUNCTL).  Every lifecycle call that moves,
resets or re-lays runs is routed through each present area's model in the contract's order (include/bobrafrontier.h, and
RunAreas in bobrapet_b200/csrc/ctx.h), so that a test can compare every area of every batch with the device after each call.
The per-area rules are not restated here; only how they compose:
  - retire: each area follows its own retire; a new capacity keeps the first `capacity` entries of every area;
  - transfer: a source with limiter inputs needs a destination with them (refused with no unfit run); then a run is unfit when
    it has more armed timer slots than the destination's K (0 without a timer area), or a run-control record that is not the
    default and no run-control area to arrive in; arrivals take the defaults of the areas the source lacks, and lose their
    schedule baseline; the source follows retire; into a batch of another ctx, each arrival's header slot goes through the
    caller's slot map and nothing else differs;
  - reshape: every area grows to the new capacity with its defaults, and a change of words drops every schedule baseline;
  - narrow: the areas are kept, and a change of words drops every schedule baseline;
  - migrate: the timers are re-keyed and the migrated runs lose their schedule baseline;
  - redrive: the record reset of the redrive section, then the run-control record is lifted (the saved flags byte returns)
    and the timers are emptied."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import pack_state
from tests import runctl as R
from tests import sched_resident as SRM
from tests import timers as T
from tests.transfer import map_slots, relay_state

TIMERS, SCHED, RUNCTL = 1, 2, 4
SUBSETS = tuple(range(8))
# the runs a directed transfer moves, in this order, from a batch seeded by seed_requests: 2 has only limiter inputs, 6 one
# armed slot, 5 min(K, 4) armed slots and a story deadline, 13 a drain deadline and an armed slot, 10 a story deadline, 3 a stop
MOVED = [2, 6, 5, 13, 10, 3]


def subset_name(subset, K=0):
    parts = (["timers%d" % K] if subset & TIMERS else []) + (["sched"] if subset & SCHED else []) + \
            (["runctl"] if subset & RUNCTL else [])
    return "+".join(parts) or "bare"


def area_sets(ks=(2, 5)):
    """every (subset, K): the subsets with timers once per K, the others with K = 0"""
    return [(s, k) for s in SUBSETS for k in (ks if s & TIMERS else (0,))]


def template_records(L, slots, S):
    """two state records, one on each of two slots of S[0] and S[1] steps: steps 0-4 Succeeded, step 2's decision SUCCEED,
    step 6's cond HOLD, the rest 0; run_flags FAIL_FAST and REALTIME | TOPOLOGY_TERMINATED (a stop saves them, a redrive
    restores them without TOPOLOGY_TERMINATED)"""
    ph = np.zeros((2, L.steps_max), np.uint8)
    ph[:, :5] = A.PHASE_SUCCEEDED
    dec = np.zeros_like(ph)
    dec[:, 2] = A.DEC_SUCCEED
    cond = np.zeros_like(ph)
    cond[:, 6] = 2
    for t in range(2):
        ph[t, S[t]:] = dec[t, S[t]:] = cond[t, S[t]:] = 0
    flags = np.array([A.RF_FAIL_FAST, A.RF_REALTIME | A.RF_TOPOLOGY_TERMINATED], np.uint8)
    return pack_state(L, np.asarray(slots, np.uint32), flags, ph, cond, dec)


def records_of(templates, n):
    """n runs: run r holds the second template when r % 4 == 2, else the first"""
    return np.ascontiguousarray(templates[[1 if r % 4 == 2 else 0 for r in range(n)]])


def seed_requests(n, K, last_step, now):
    """non-default entries for every area of a batch of n runs, as (limiter puts, timer arms, run-control puts), to be applied
    in that order: inputs on every run, equal for runs of equal r % 4 (so that runs 1 and 13 get equal schedule records: a
    retire of run 1 moves 13 there, and a schedule baseline kept by mistake would go unlisted); run 1 armed at step 1 and
    last_step, run 5 at min(K, 4) steps, runs 6 and 13 at one, run 3 at one that its stop empties; run r stopped when r % 4 == 3 (reasons TIMEOUT, CANCEL, HOST in turn), a story deadline
    when r % 5 == 0 and a drain deadline when r % 6 == 1"""
    p = SRM.defaults(n)
    r = np.arange(n)
    p["run"], p["story_key"], p["queue_key"] = r, r % 4, r % 2
    p["priority"], p["queued_since"], p["run_phase"] = 3 * (r % 4) - 4, now - 10 * (r % 4), 2
    arms = []
    for run, steps in ((1, [1, last_step]), (5, [2, 9, 15, 19]), (6, [4]), (13, [6]), (3, [0])):
        for k, s in enumerate(steps[:min(K, 4)]):
            if run < n:
                arms.append((run, s, (A.DEC_SUCCEED, A.DEC_PENDING, A.DEC_TIMED_OUT)[k % 3], 0, now + 100 + s, 0))
    arms = np.array(arms, np.dtype([("run", "<u4"), ("step", "<u2"), ("code", "u1"), ("reserved", "u1"), ("deadline", "<u4"),
                                    ("reserved2", "<u4")]))
    q = np.zeros(n, R.PUT_DTYPE)
    for i in range(n):
        q[i] = (i, now + 200 + i if i % 5 == 0 else R.NONE, now + 50 if i % 6 == 1 else R.NONE,
                1 + (i // 4) % 3 if i % 4 == 3 else 0, (0, 0, 0))
    return p, arms, q


def seeded(L, cap, subset, K, records, last_step, now):
    """a model batch holding `records` with every area of `subset` seeded by seed_requests -> (batch, requests)"""
    b = AreaBatch(L, cap, subset, K)
    b.upload(0, records)
    p, arms, q = seed_requests(len(records), b.K, last_step, now)
    if b.sched is not None:
        b.put_sched(p)
    if b.K:
        assert b.arm(arms) == 0
    if b.runctl is not None:
        assert b.put_runctl(q)[0] == 0
    return b, (p, arms, q)


def beyond_requests(b, now):
    """entries for the indices of b at or above its runs (records a put may reach ahead of an upload): a story deadline, limiter
    inputs and one armed slot each, for the areas b has -> (limiter puts, timer arms, run-control puts); an arrival there must
    overwrite every one of them"""
    idx = np.arange(b.n, b.cap)
    p = SRM.defaults(idx.size)
    p["run"], p["story_key"], p["priority"] = idx, 1, 7
    arms = np.zeros(idx.size if b.K else 0, np.dtype([("run", "<u4"), ("step", "<u2"), ("code", "u1"), ("reserved", "u1"),
                                                       ("deadline", "<u4"), ("reserved2", "<u4")]))
    if b.K:
        arms["run"], arms["step"], arms["deadline"] = idx, 3, now + 77
    q = np.zeros(idx.size, R.PUT_DTYPE)
    q["run"], q["story_deadline"], q["drain_deadline"] = idx, now + 999, R.NONE
    return p, arms, q


class Refused(Exception):
    """a refused transfer: `unfit` is the position of the first unfit run (A.EXTENT_NO_RUN for a refusal of the whole call),
    `lost` what that run would lose ({"timers", "runctl"})"""

    def __init__(self, why, unfit=A.EXTENT_NO_RUN, lost=()):
        super().__init__(why)
        self.unfit, self.lost = unfit, set(lost)


def _clear_step(L, rec, s):
    """every input code of step s back to 0, as a migration to a map that drops s leaves it"""
    T._set(rec, L.off_phase, L.words, 4, s, 0)
    for off in (L.off_cond, L.off_decision):
        if off != A.OFF_NONE:
            T._set(rec, off, L.words, 2, s, 0)


class AreaBatch:
    """a resident batch: layout L, `cap` state records (zero as after create), runs [0, n) and the side areas of `subset`"""

    def __init__(self, L, cap, subset, K=0):
        self.L, self.subset, self.n = L, subset, 0
        self.K = K if subset & TIMERS else 0
        self.state = np.zeros((cap, L.state_stride), np.uint8)
        self.timers = T.empty_area(cap, self.K) if self.K else None
        self.sched = SRM.Batch(L, cap) if subset & SCHED else None
        self.runctl = R.defaults(cap) if subset & RUNCTL else None

    @property
    def cap(self):
        return self.state.shape[0]

    @property
    def inputs(self):
        return None if self.sched is None else self.sched.inputs

    # -- calls on one batch
    def upload(self, first, records):
        R.upload(self.runctl, self.state, first, records)
        if self.sched is not None:
            self.sched.upload(first, len(records))
        self.n = max(self.n, first + len(records))

    def arm(self, reqs):
        """-> the status bf_resident_timers_arm returns"""
        return T.arm(self.timers, self.L, reqs)

    def put_runctl(self, reqs):
        """-> (status, runs stopped now)"""
        return R.put(self.runctl, self.state, reqs, self.timers, self.inputs)

    def put_sched(self, reqs):
        self.sched.put(reqs)

    # -- calls that move, reset or re-lay runs
    def retire(self, N, runs, capacity=0):
        """bf_resident_retire -> (m, {from: to})"""
        m, mv = T.retire_moves(N, runs)
        st = self.state.copy()
        for f, t in mv.items():
            st[t] = self.state[f]
        st[m:N] = 0
        self.state = st[:capacity].copy() if capacity else st
        if self.timers is not None:
            self.timers = T.retire(self.timers, N, runs, capacity)
        if self.runctl is not None:
            self.runctl = R.retire(self.runctl, N, runs, capacity)
        if self.sched is not None:
            self.sched.retire(N, runs)
            if capacity:
                self.sched.resize(capacity)
        self.n = m
        return m, mv

    def lost_by(self, dst, r):
        """what run r would lose on its way to dst: {"timers"} when its armed slots exceed dst's K, {"runctl"} when its
        run-control record is not the default and dst has no area for it"""
        lost = set()
        if not T.fits(self.timers, r, dst.K):
            lost.add("timers")
        if not R.fits(self.runctl, dst.runctl, r):
            lost.add("runctl")
        return lost

    def transfer(self, dst, dst_first, runs, slot_map=None):
        """bf_resident_transfer of `runs` (source runs [0, self.n)) to dst at dst_first, the fit of the areas only (both
        layouts must hold every run) -> (m, {from: to}); raises Refused, nothing changed.  slot_map: bf_resident_transfer_ctx,
        dst in another ctx: each arrival's header slot becomes slot_map[its source slot] (every moved slot mapped), the rest as
        within one ctx"""
        runs = [int(r) for r in runs]
        if runs and self.sched is not None and dst.sched is None:
            raise Refused("the source has limiter inputs and the destination no area for them")
        for i, r in enumerate(runs):
            lost = self.lost_by(dst, r)
            if lost:
                raise Refused("run %d does not fit" % r, i, lost)
        if not runs:
            return self.n, {}
        k, ix = len(runs), np.asarray(runs, np.int64)
        dst.state[dst_first:dst_first + k] = relay_state(self.L, dst.L, self.state[ix])
        if slot_map is not None:
            map_slots(dst.state[dst_first:dst_first + k], slot_map)
        if dst.timers is not None:
            dst.timers = T.transfer(self.timers, dst.timers, self.n, dst_first, runs)[1]
        if dst.runctl is not None:
            dst.runctl = R.transfer(self.runctl, dst.runctl, self.n, dst_first, runs)[1]
        if dst.sched is not None:
            dst.sched.receive(dst_first, SRM.defaults(k) if self.sched is None else self.sched.inputs[ix].copy())
        dst.n = dst_first + k
        return self.retire(self.n, runs)

    def reshape(self, L, capacity):
        """bf_resident_reshape to layout L and `capacity` (>= cap)"""
        st = np.zeros((capacity, L.state_stride), np.uint8)
        st[:self.cap] = relay_state(self.L, L, self.state)
        if self.timers is not None:
            self.timers = T.reshape(self.timers, capacity)
        if self.runctl is not None:
            self.runctl = R.reshape(self.runctl, capacity)
        if self.sched is not None:
            if capacity > self.cap:
                self.sched.resize(capacity)
            self.sched.relayout(L)
        self.state, self.L = st, L

    def narrow(self, L):
        """bf_resident_narrow to layout L, accepted"""
        self.state = relay_state(self.L, L, self.state)
        if self.sched is not None:
            self.sched.relayout(L)
        self.L = L

    def migrate(self, old_slot, new_slot, step_map):
        """bf_resident_migrate over runs [0, n) with a map that keeps every step's index or drops it (GONE) -> migrated runs"""
        slots = np.ascontiguousarray(self.state[:self.n, 0:4]).view("<u4")[:, 0]
        runs = [int(r) for r in np.nonzero(slots == old_slot)[0]]
        for r in runs:
            assert all(int(t) in (s, T.MIGRATE_GONE) for s, t in enumerate(step_map))
            for s, t in enumerate(step_map):
                if int(t) == T.MIGRATE_GONE:
                    _clear_step(self.L, self.state[r], s)
            self.state[r, 0:4] = np.array([new_slot], "<u4").view(np.uint8)
        if self.timers is not None:
            self.timers = T.migrate(self.timers, runs, step_map)
        if self.sched is not None:
            self.sched.lose_baseline(runs)
        return runs

    def redrive(self, requests, status, resets, has_if):
        """bf_resident_redrive of topologies without parallel steps: resets[i] is request i's reset set R as an int step mask
        (every step for BF_REDRIVE_ALL, else bf_topology_closure's), has_if[i] the HAS_IF steps of its slot.  The steps of R
        get phase 0, decision PENDING, and cond HOLD where they have an `if`, else PASS; TOPOLOGY_TERMINATED is cleared; then
        the run-control record is lifted (the saved flags byte returns) and the timers are emptied"""
        W, L = self.L.words, self.L
        for q, st, m, hi in zip(requests, status, resets, has_if):
            if not st:
                continue
            r = int(q["run"])
            row = self.state[r]
            for off, nbits in ((L.off_phase, 4), (L.off_decision, 2), (L.off_cond, 2)):
                if off == A.OFF_NONE:
                    continue
                for b in range(nbits):
                    lo = off + 4 * W * b
                    v = int.from_bytes(row[lo:lo + 4 * W].tobytes(), "little") & ~m
                    if off == L.off_cond and b == 1:
                        v |= m & hi
                    row[lo:lo + 4 * W] = np.frombuffer(v.to_bytes(4 * W, "little"), np.uint8)
            row[4] &= ~np.uint8(R.RF_TOPOLOGY_TERMINATED)
        R.redrive(self.runctl, self.state, requests, status)
        if self.timers is not None:
            self.timers = T.redrive(self.timers, requests, status)
