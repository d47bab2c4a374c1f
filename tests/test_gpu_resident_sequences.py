"""Random sequences of resident-batch calls in the order a batcher makes them (INTEGRATION.md: put, create, upload, tick; put an
edited Story, migrate, drop the old one; redrive; reshape an outgrown batch; retire finished runs), two batches on one ctx,
checked after every call against the host model of tests/resident_model.py: the device state, every tick output, the `full`
flag of every touched tick, the moves, statuses and counts, which calls are refused, and every accepted bf_schedule against
tests/schedref.py over the model's records.  Then directed cases for the
combinations the random draws reach rarely."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import retire as RT
from tests.seqrig import NONE, TICK_KINDS, Rig, layout_for, random_records, story_pool

pytestmark = pytest.mark.gpu

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT
# shape: (steps lo, hi, parallel steps per Story, layout fields, runs of batch A, runs of batch B, grow steps_max to)
SHAPES = {"cfg3": (200, 256, 0, 0, 1200, 300, None),                       # phase planes only, no cond
          "cfg4": (200, 256, 2, COND | DEC | OUT | CHILD, 1000, 300, None),  # every field
          "parallel": (20, 120, 6, CHILD | OUT, 1000, 300, None),          # parallel steps and a child area
          "wide": (513, 700, 2, COND | DEC | OUT | CHILD, 500, 200, None),  # S > 512: the general kernel
          "grow": (200, 256, 2, COND | OUT | CHILD, 800, 200, 288)}          # one reshape 256 -> 288 moves the pass to another kernel
SEEDS = 6
N_BASE = 5
OPS = {"apply": 8, "upload": 6, "tick": 10, "touched": 22, "migrate": 6, "redrive": 7, "reshape": 4, "retire": 8, "slots": 7,
       "params": 5, "schedule": 4, "invalid": 3}   # weights


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _deltas(rng, rig, b, n, k):
    """k coalesced valid deltas on runs of [0, n): every field the layout has, now and then a slot delta to a live Story that fits"""
    L, reg = b.L, rig.reg
    fields = [A.DELTA_PHASE] * 6 + [A.DELTA_RUN_FLAGS, A.DELTA_REGISTERED]
    fields += [A.DELTA_COND] * (L.off_cond != A.OFF_NONE) + [A.DELTA_DECISION] * (L.off_decision != A.OFF_NONE)
    fields += [A.DELTA_CHILD] * (L.off_child != A.OFF_NONE and L.child_nibbles > 0)
    fits = [s for s, kk in reg.live.items() if reg.stories[kk].S <= L.steps_max and
            (L.off_child == A.OFF_NONE or reg.stories[kk].child_nibbles() <= L.child_nibbles)]
    recs = {}
    for _ in range(k):
        r = int(rng.integers(0, n))
        f = A.DELTA_TOPO_SLOT if (fits and rng.random() < 0.01) else int(rng.choice(fields))
        key = None
        if f == A.DELTA_PHASE:
            idx, code = int(rng.integers(0, 32 * L.words)), int(rng.choice([0, 1, 2, 3, 3, 4, 9, 13, 14]))
        elif f in (A.DELTA_COND, A.DELTA_DECISION):
            idx, code = int(rng.integers(0, 32 * L.words)), int(rng.integers(0, 4))
        elif f == A.DELTA_CHILD:
            idx, code = int(rng.integers(0, L.child_nibbles)), int(rng.choice([0, 2, 3, 4, 13]))
        elif f == A.DELTA_RUN_FLAGS:
            idx, code = 0, int(rng.choice([0, A.RF_FAIL_FAST, A.RF_FAIL_FAST | A.RF_REALTIME, A.RF_TOPOLOGY_TERMINATED]))
        elif f == A.DELTA_TOPO_SLOT:
            new = int(rng.choice(fits))
            idx, code, key = new & 0xFFFF, new >> 16, 0
        else:
            idx, code = int(rng.integers(0, 64)), int(rng.integers(0, 2))
        recs[(r, f, idx if key is None else key)] = (idx, code)
    d = np.zeros(len(recs), dtype=Frontier.DELTA_DTYPE)
    for i, ((r, f, _), (idx, code)) in enumerate(recs.items()):
        d[i] = (r, idx, f, code)
    return d


class Driver:
    def __init__(self, fr, rng, shape, seed):
        lo, hi, n_par, fields, nA, nB, self.grow = SHAPES[shape]
        self.rng, self.fields = rng, fields
        pool = story_pool(rng, lo, hi, n_par, N_BASE)
        self.rig = rig = Rig(fr, pool, "seed %d shape %s" % (seed, shape))
        self.base = [rig.put(k) for k in range(N_BASE)]
        self.edited, self.migrated = set(), set()   # slots of edited Stories; base Stories already edited
        L = layout_for(pool[:N_BASE], fields)
        self.bs = []
        for n in (nA, nB):
            b = rig.create(L, n + n // 4)
            rig.upload(b, 0, self._fresh(L, n))
            self.bs.append([b, n])
        self.flags, self.max_iter = 0, 0
        self.followed = set()

    def follow(self, bi, op):
        """after a resident operation: the first time for each kind of operation and then now and then, a tick over the batch and
        a schedule compared after it"""
        if op in self.followed and self.rig.srng.random() >= 0.5:
            return
        self.followed.add(op)
        b, n = self.bs[bi]
        self.rig.tick_and_schedule(b, n, op, self.flags, self.max_iter)

    def _fresh(self, L, n):
        live = [s for s in self.rig.reg.live if s in self.base or s in self.edited]
        slots = [int(self.rng.choice(live)) for _ in range(n)]
        return random_records(self.rng, L, [self.rig.reg.story(s) for s in slots], slots)

    def step(self):
        rng, rig = self.rng, self.rig
        bi = 0 if rng.random() < 0.75 else 1
        b, n = self.bs[bi]
        op = rng.choice(list(OPS), p=np.array(list(OPS.values())) / sum(OPS.values()))
        if op == "apply":
            rig.apply(b, _deltas(rng, rig, b, max(n, 1), int(rng.integers(1, 300))))
        elif op == "upload":
            if rng.random() < 0.5 and n < b.cap:   # new runs in the tail
                k = int(rng.integers(1, b.cap - n + 1))
                rig.upload(b, n, self._fresh(b.L, k))
                self.bs[bi][1] = n + k
            elif n:                                  # a resync of a few runs, same bytes
                first = int(rng.integers(0, n))
                k = int(rng.integers(1, min(40, n - first) + 1))
                rig.upload(b, first, b.state[first:first + k].copy())
        elif op == "tick":
            kind = str(rng.choice(["dense", "eval", "compact", "changed", "changed"]))
            rig.tick(b, kind, n, _deltas(rng, rig, b, max(n, 1), int(rng.integers(0, 200))) if n else NONE, self.flags, self.max_iter)
            if rig.srng.random() < 0.5:
                rig.schedule_last()
        elif op == "touched":
            u = rng.random()   # mostly the live runs; sometimes fewer, or more (records the batch holds past its live runs)
            nr = n if u < 0.8 else int(rng.integers(0, n + 1)) if u < 0.93 else int(rng.integers(n, b.cap + 1))
            d = _deltas(rng, rig, b, max(nr, 1), int(rng.integers(0, 400))) if nr else NONE
            caps = rng.random() < 0.2
            rig.tick(b, "touched", nr, d, self.flags | (A.EVAL_NO_COUNTS if rng.random() < 0.1 else 0), self.max_iter,
                     runs_cap=int(rng.integers(0, 50)) if caps else None, events_cap=int(rng.integers(0, 500)) if caps else None,
                     pinned=rng.random() < 0.2)
            if rig.srng.random() < 0.5:
                rig.schedule_last()
        elif op == "migrate":
            todo = [k for k in range(N_BASE) if k not in self.migrated and self.base[k] in rig.reg.live]
            if todo:
                k = int(rng.choice(todo))
                new = rig.put(N_BASE + k)
                if rig.migrate(b, self.base[k], new, n) is not None:
                    self.edited.add(new)
                    self.migrated.add(k)
                    other = self.bs[1 - bi]
                    rig.migrate(other[0], self.base[k], new, other[1])
                    if rng.random() < 0.7:
                        rig.drop(self.base[k])
                else:
                    rig.drop(new)
                self.follow(bi, "migrate")
        elif op == "redrive" and n:
            k = int(rng.integers(1, 40))
            runs = rng.integers(0, n, size=k)
            runs = np.concatenate([runs, runs[:k // 4]])   # duplicates
            slots = b.slots(b.cap)[runs]
            req = np.zeros(len(runs), dtype=Frontier.REDRIVE_DTYPE)
            req["run"] = runs
            live = list(rig.reg.live)
            req["slot"] = [s if (s in rig.reg.live and rng.random() < 0.9) else int(rng.choice(live)) for s in slots.tolist()]
            req["step"] = [A.REDRIVE_ALL if rng.random() < 0.3 else int(rng.integers(0, rig.reg.story(int(s)).S)) for s in req["slot"]]
            rig.redrive(b, req)
            self.follow(bi, "redrive")
        elif op == "reshape":
            L = b.L
            S = L.steps_max + (32 if rng.random() < 0.3 else 0)
            if self.grow and L.steps_max < self.grow:
                S = self.grow
            f = L.fields | int(rng.choice([0, COND, DEC, A.F_OUT_FAIL, A.F_OUT_NEEDS_COND, A.F_OUT_SKIP_DEP]))
            child = L.child_nibbles + (8 if (L.off_child != A.OFF_NONE and rng.random() < 0.3) else 0)
            rig.reshape(b, make_layout(S, child, f), b.cap + int(rng.choice([0, 0, 16, b.cap])))
            self.follow(bi, "reshape")
        elif op == "retire" and n:
            k = int(rng.integers(0, n // 3 + 1))
            runs = rng.choice(n, size=k, replace=False)
            m = n - k
            cap = int(rng.choice([0, m, (m + b.cap + 1) // 2])) if m else 0
            if rig.retire(b, n, runs, cap) is not None:
                self.bs[bi][1] = m
            self.follow(bi, "retire")
        elif op == "slots":
            if rng.random() < 0.5:   # drop a slot runs still hold (not one of the base Stories the generators draw from)
                held = [s for s in rig.reg.live if s not in self.base and s not in self.edited]
                if not held:
                    held = [s for s in self.edited if s in rig.reg.live][:1]
                    self.edited -= set(held)
                if held:
                    rig.drop(int(rng.choice(held)))
            else:                    # a put that may reuse a dropped slot; some runs are re-pointed at it
                s = rig.put(len(rig.reg.stories) - 1 - int(rng.integers(0, 2)))
                if n and rng.random() < 0.5:
                    k = int(rng.integers(1, min(n, 20) + 1))
                    d = np.zeros(k, dtype=Frontier.DELTA_DTYPE)
                    d["run"], d["index"], d["field"], d["code"] = rng.choice(n, k, replace=False), s & 0xFFFF, A.DELTA_TOPO_SLOT, s >> 16
                    rig.apply(b, d)
        elif op == "params":
            self.flags = int(rng.choice([0, A.EVAL_FIXPOINT]))
            self.max_iter = int(rng.choice([0, 0, 1, 3])) if self.flags else 0
        elif op == "schedule" and n:   # mostly over the last tick's batch and n_runs; sometimes a batch or count it did not evaluate
            if rig.srng.random() < 0.85:
                rig.schedule_last()
            else:
                rig.schedule(b, n)
        elif op == "invalid":
            kind = int(rng.integers(0, 6))
            if kind == 0 and n:
                rig.retire(b, n, [0, 0])
            elif kind == 1:
                rig.reshape(b, b.L, max(b.cap - 1, 0))
            elif kind == 2:
                rig.migrate(b, self.base[0] if self.base[0] in rig.reg.live else next(iter(rig.reg.live)),
                            self.base[0] if self.base[0] in rig.reg.live else next(iter(rig.reg.live)), n)
            elif kind == 3:
                rig.tick(b, "touched", n, NONE, A.EVAL_CHANGED_ONLY)
            elif kind == 4:
                rig.upload(b, b.cap, b.state[:1].copy())
            else:
                rig.tick(b, "compact", b.cap + 1)


@pytest.mark.parametrize("seed", range(SEEDS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_random_sequences(fr, shape, seed):
    rng = np.random.default_rng(9000 + 100 * list(SHAPES).index(shape) + seed)
    dr = Driver(fr, rng, shape, seed)
    try:
        for b, n in dr.bs:
            dr.rig.tick(b, "touched", n)
        for _ in range(int(rng.integers(60, 101))):
            dr.step()
        for b, n in dr.bs:   # a closing tick of each kind over the batch as it ends
            dr.rig.tick(b, "touched", n, NONE, dr.flags, dr.max_iter)
            dr.rig.tick(b, "changed", n, NONE, dr.flags, dr.max_iter)
        close_with_schedules(dr)
    finally:
        dr.rig.destroy()
    assert_schedules_compared(dr)


def close_with_schedules(dr):
    """a tick of every kind over batch A as it ends, each followed by a compared schedule"""
    b, n = dr.bs[0]
    for kind in TICK_KINDS:
        dr.rig.tick(b, kind, n, NONE, dr.flags, dr.max_iter)
        dr.rig.schedule_last()


def assert_schedules_compared(dr):
    """the sequence compared schedules after every tick kind, and after every kind of resident operation it made"""
    c = dr.rig.compared
    missing = ["tick " + k for k in TICK_KINDS if not c["tick " + k]] + ["after " + op for op in sorted(dr.followed) if not c["after " + op]]
    assert not missing, "no schedule compared for %s; compared: %s" % (missing, dict(c))


# ------------------------------------------------------------------------------------------------ directed cases
def _rig(fr, seed, lo=60, hi=120, n_par=2, fields=COND | DEC | OUT | CHILD, n=600, cap=None, n_base=3):
    rng = np.random.default_rng(seed)
    pool = story_pool(rng, lo, hi, n_par, n_base)
    rig = Rig(fr, pool, "directed seed %d" % seed)
    slots = [rig.put(k) for k in range(n_base)]
    L = layout_for(pool, fields)
    b = rig.create(L, cap or n)
    story = rng.integers(0, n_base, n)
    rig.upload(b, 0, random_records(rng, L, [pool[k] for k in story], [slots[k] for k in story]))
    return rng, rig, b, slots


def test_reused_slot_re_points_its_runs(fr):
    """drop a slot runs hold, a full tick (they evaluate dead), a put that reuses the slot: the next touched tick must be full,
    because those runs now evaluate against the new topology"""
    rng, rig, b, slots = _rig(fr, 1)
    n = 600
    try:
        rig.tick(b, "touched", n)
        rig.drop(slots[1])
        out = rig.tick(b, "touched", n)
        assert out["full"] == 1 and (out["head"] & 0x7FFF == 0x7FFF).any()
        rig.tick(b, "touched", n, NONE)
        s = rig.put(len(rig.reg.stories) - 1)
        assert s == slots[1]   # the last freed slot comes back first
        out = rig.tick(b, "touched", n)
        assert out["full"] == 1
        assert not (out["head"] & 0x7FFF == 0x7FFF).any()
        assert rig.tick(b, "touched", n)["full"] == 0
        # a put of a new index is not a change: the touched tick after it stays incremental
        rig.put(len(rig.reg.stories) - 2)
        assert rig.tick(b, "touched", n)["full"] == 0
    finally:
        rig.destroy()


def test_never_put_slot_index_stays_dead_until_touched(fr):
    """a run may hold only a slot a put returned: one re-pointed at an index no put has created evaluates dead, and a put that
    creates that index later does not make the next touched tick full; re-sending the slot delta touches the run again"""
    rng, rig, b, slots = _rig(fr, 2)
    n = 600
    try:
        rig.tick(b, "touched", n)
        ghost = rig.reg.n_index
        d = np.zeros(3, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"], d["field"], d["code"] = [5, 77, 300], ghost, A.DELTA_TOPO_SLOT, 0
        out = rig.tick(b, "touched", n, d)
        assert out["full"] == 0 and list(out["runs"]) == [5, 77, 300] and (out["head"] & 0x7FFF == 0x7FFF).all()
        assert rig.put(len(rig.reg.stories) - 1) == ghost
        out = rig.tick(b, "touched", n)
        assert out["full"] == 0 and out["n_evaluated"] == 0   # (the runs keep their dead rows)
        out = rig.tick(b, "touched", n, d)
        assert out["full"] == 0 and list(out["runs"]) == [5, 77, 300] and not (out["head"] & 0x7FFF == 0x7FFF).any()
    finally:
        rig.destroy()


def test_reshape_double_capacity_upload_then_retire_across(fr):
    rng, rig, b, slots = _rig(fr, 3, n=500)
    try:
        rig.tick(b, "touched", 500)
        rig.reshape(b, b.L, 1000)
        recs = random_records(rng, b.L, [rig.reg.story(slots[0])] * 500, [slots[0]] * 500)
        rig.upload(b, 500, recs)
        assert rig.tick(b, "touched", 1000)["full"] == 0
        runs = np.concatenate([rng.choice(500, 150, replace=False), 500 + rng.choice(500, 150, replace=False)])
        m = rig.retire(b, 1000, runs)
        assert m == 700
        out = rig.tick(b, "touched", m, NONE)
        assert out["full"] == 0
        rig.tick(b, "changed", m)
    finally:
        rig.destroy()


def test_migrate_retire_moves_migrated_runs_then_redrive(fr):
    rng, rig, b, slots = _rig(fr, 4, n=600)
    n = 600
    try:
        rig.tick(b, "touched", n)
        new = rig.put(3)   # the edit of Story 0
        assert rig.migrate(b, slots[0], new, n) > 0
        on_new = np.nonzero(b.slots(n) == new)[0]
        tail = on_new[on_new >= n - 200]
        runs = rng.choice(n - 200, 200, replace=False)   # the last 200 runs, migrated ones among them, move
        m, mf, mt = n - 200, *RT.moves(n, runs)[1:]
        assert rig.retire(b, n, runs) == m and len(tail) and set(tail.tolist()) <= set(mf.tolist())
        out = rig.tick(b, "touched", m)
        assert out["full"] == 0 and set(mt.tolist()) <= set(out["runs"].tolist())
        req = np.zeros(len(mt), dtype=Frontier.REDRIVE_DTYPE)
        req["run"], req["slot"] = mt, b.slots(m)[mt]
        req["step"] = A.REDRIVE_ALL
        rig.redrive(b, req)
        assert rig.tick(b, "touched", m)["full"] == 0
    finally:
        rig.destroy()


def test_reshape_adding_decision_planes_then_retire_keeps_full(fr):
    rng, rig, b, slots = _rig(fr, 5, fields=COND | OUT | CHILD, n=400)
    try:
        rig.tick(b, "touched", 400)
        rig.reshape(b, make_layout(b.L.steps_max, b.L.child_nibbles, b.L.fields | DEC), b.cap)
        rig.retire(b, 400, rng.choice(400, 50, replace=False))
        assert rig.tick(b, "touched", 350)["full"] == 1
        assert rig.tick(b, "touched", 350)["full"] == 0
    finally:
        rig.destroy()


def test_changed_only_after_a_retire_the_last_tick_did_not_cover(fr):
    """the last tick covered fewer runs than the retire's n_runs: a changed-only tick lists every run"""
    rng, rig, b, slots = _rig(fr, 6, n=500)
    try:
        rig.tick(b, "changed", 400)
        rig.retire(b, 500, rng.choice(500, 60, replace=False))
        rig.tick(b, "changed", 440)
        assert b.prev_valid
        rig.tick(b, "changed", 440)
    finally:
        rig.destroy()


def test_retire_shrinking_capacity_then_touched_and_changed_only(fr):
    rng, rig, b, slots = _rig(fr, 7, n=500, cap=640)
    try:
        rig.tick(b, "changed", 500)
        rig.tick(b, "touched", 500, NONE)
        runs = rng.choice(500, 120, replace=False)
        assert rig.retire(b, 500, runs, 380) == 380
        assert rig.tick(b, "touched", 380)["full"] == 0
        rig.tick(b, "changed", 380)
        rig.tick(b, "touched", 380)
    finally:
        rig.destroy()


def test_retire_counts_moved_runs_as_uploaded_and_lowers_the_full_run_count(fr):
    """the last full tick covered 500 of 600 runs and the rest were re-uploaded but for run 550, which a retire then fills with a
    moved run: it counts as uploaded, so a touched tick over the 598 runs left stays incremental.  After a full tick over 570, a
    retire down to 550 lowers the run count of the last full evaluation: a touched tick over 560 is full"""
    rng, rig, b, slots = _rig(fr, 8, n=600)
    try:
        rig.tick(b, "touched", 600)
        rig.tick(b, "compact", 500)
        rig.upload(b, 500, b.state[500:550].copy())
        rig.upload(b, 551, b.state[551:600].copy())
        assert rig.retire(b, 600, [550, 10]) == 598
        assert rig.tick(b, "touched", 598)["full"] == 0
        assert rig.retire(b, 598, rng.choice(598, 40, replace=False)) == 558
        assert rig.tick(b, "touched", 558)["full"] == 0
        assert rig.tick(b, "touched", 570)["full"] == 1
        assert rig.retire(b, 570, rng.choice(570, 20, replace=False)) == 550
        assert rig.tick(b, "touched", 550)["full"] == 0
        assert rig.tick(b, "touched", 560)["full"] == 1
    finally:
        rig.destroy()
