"""Random side-area resyncs interleaved with the calls that change a resident batch's areas: fires, timer arms, tick commits that
arm the timers of the sleeps, gates and waits they launch, retires, transfers, migrations, redrives and stops, on two batches of
one ctx with every area (tests/lifecycle.AreaBatch as the model).  Each resync goes to the device and to tests/resync_areas.py:
items, drifted runs and n_written must agree, and after every step the state records and every area of both batches over the
whole capacity must be the model's.

The caller's areas of a resync are what a batcher would hold: right after a fire, the timer slots as they were before it (the
annotation keeps a fired slot until its step is terminal; the fire disarmed it, pruned the slots of terminal steps and may have
stopped runs on their story deadline, which the batcher persisted from the fired list) and the drain deadlines before it; else the
device's own areas; either perturbed.  fired_now is the `now` of the batch's last fire.  A commit's writes reach the model through
its journal, as they reach a batcher's persisted state."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import randgen
from tests import resync_areas as M
from tests import runctl as R
from tests import timers as T
from tests.lifecycle import RUNCTL, SCHED, TIMERS, Refused
from tests.test_gpu_resync_areas import Batch, perturb
from tests.test_gpu_run_areas import NOW, TABLES, Env

pytestmark = pytest.mark.gpu

ALL = TIMERS | SCHED | RUNCTL
K, N, CAP = 4, 16, 24
OPS = ["fire", "fire", "arm", "commit", "commit", "retire", "transfer", "migrate", "redrive", "stop",
       "resync", "resync", "resync", "resync"]
TIMING_CODE = {A.STEP_SLEEP: A.DEC_SUCCEED, A.STEP_GATE: A.DEC_TIMED_OUT, A.STEP_WAIT: A.DEC_PENDING}


def _timings(fr, ts, slots, rng):
    """a timing for every sleep, gate and wait step of each slot, so that the commits arm them"""
    at = 0
    for i, slot in enumerate(slots):
        S = int(ts.S[i])
        ents = [(s, TIMING_CODE[int(f) & A.SF_TYPE_MASK], int(rng.integers(0, 20)))
                for s, f in enumerate(ts.step_flags[at:at + S]) if int(f) & A.SF_TYPE_MASK in TIMING_CODE]
        fr.put_timings(int(slot), ents)
        at += S


class Seq:
    def __init__(self, fr, seed):
        self.fr, self.rng = fr, np.random.default_rng(seed)
        self.env = env = Env(fr)
        # timers only at steps every topology has: a fire writes a decision code at its step, and a migration zeroes the codes
        # past the new topology's steps, which the model (identity maps) does not restate
        self.S = min(env.S)
        _timings(fr, env.ts, env.slots, self.rng)
        S0 = env.S[0]
        nt = randgen.random_topologies(np.random.default_rng(seed + S0), 1, S0, S0, parallel=False)
        self.alt = int(fr.put_topologies(nt)[0])   # migrations move runs between slots[0] and this one
        env.add(nt, [self.alt])
        self.bs = [Batch(env, ALL, K, N, CAP), Batch(env, ALL, K, N, CAP)]
        self.now = NOW
        self.fired_now = [A.TIMER_NONE, A.TIMER_NONE]
        self.prefire = [None, None]   # (timers, runctl) of the model just before the batch's last fire, while no call re-keyed it
        self.log = []

    def check(self, what):
        for i, b in enumerate(self.bs):
            b.check("%s (batch %d) after %s" % (what, i, self.log[-8:]))

    def changed(self, i):
        self.prefire[i] = None

    # -- the calls
    def fire(self, i):
        b = self.bs[i]
        self.now += int(self.rng.integers(1, 30))
        pre = (b.m.timers.copy(), b.m.runctl.copy())
        want = R.fire(b.m.runctl, b.m.L, b.m.state, b.m.timers, b.n, self.now, b.m.inputs)
        got = self.fr.resident_fire(b.h, b.n, self.now, fired_cap=4 * b.n + 8)
        assert [tuple(int(v) for v in x) for x in got["fired"]] == want["fired"], (got["fired"], want["fired"])
        self.fired_now[i], self.prefire[i] = self.now, pre

    def arm(self, i):
        b, rng = self.bs[i], self.rng
        runs = rng.choice(b.n, size=int(rng.integers(1, 5)), replace=False)
        req = np.zeros(runs.size, Frontier.TIMER_DTYPE)
        req["run"], req["step"] = runs, rng.integers(0, self.S, runs.size)
        req["code"], req["deadline"] = rng.integers(0, 4, runs.size), self.now + rng.integers(-5, 40, runs.size)
        rc, _ = T.check_arm(b.m.timers, b.m.L, req)
        if rc:
            with pytest.raises(A.FrontierError):
                self.fr.resident_timers_arm(b.h, req)
            return
        assert b.m.arm(req) == 0
        self.fr.resident_timers_arm(b.h, req)
        self.changed(i)

    def commit(self, i):
        """a dense tick, the schedule, then a journaled commit that arms; its journal is applied to the model"""
        b, fr = self.bs[i], self.fr
        fr.resident_tick(b.h, b.m.L, b.n, np.zeros(0, Frontier.DELTA_DTYPE))
        fr.resident_schedule([dict(handle=b.h, n_runs=b.n, runs_cap=b.n, events_cap=1 << 14)], TABLES, self.now)
        try:
            got = fr.resident_commit(b.h, b.n, now=self.now, journal_cap=1 << 14)
        except A.FrontierError:   # a launched stop step without an entry: refused, nothing changed
            return
        L = b.m.L
        for it in got["items"]:
            r, s, f = int(it["run"]), int(it["index"]), int(it["field"])
            if f == A.DELTA_PHASE:
                T._set(b.m.state[r], L.off_phase, L.words, 4, s, int(it["after"]))
            elif f == A.COMMIT_WRITE_TIMER:
                e = {st: (d, c) for st, d, c in T.armed(b.m.timers[r])}
                e[s] = (int(it["after"]), int(it["code"]))
                b.m.timers[r] = T.canonical(e, b.m.K)
            else:
                raise AssertionError("unexpected journal item %s" % (it,))
        if got["n_armed"]:
            self.changed(i)

    def retire(self, i):
        b, rng = self.bs[i], self.rng
        if b.n <= 6:
            return
        gone = sorted(int(x) for x in rng.choice(b.n, size=int(rng.integers(1, 3)), replace=False))
        N = b.n
        m, mv = b.m.retire(N, gone)
        got = self.fr.resident_retire(b.h, N, np.array(gone, np.uint32))
        assert got[0] == m and dict(zip(got[1].tolist(), got[2].tolist())) == mv
        self.changed(i)

    def transfer(self, i):
        a, d = self.bs[i], self.bs[1 - i]
        if a.n <= 6:
            return
        room = d.m.cap - d.n
        moved = [int(x) for x in self.rng.choice(a.n, size=min(room, int(self.rng.integers(1, 3))), replace=False)]
        moved = [r for r in moved if not a.m.lost_by(d.m, r)]
        if not moved:
            return
        src_n, dst_n = a.n, d.n
        try:
            a.m.transfer(d.m, dst_n, moved)
        except Refused:
            return
        out = self.fr.resident_transfer(a.h, d.h, src_n, dst_n, moved)
        assert (out["src_n_runs"], out["dst_n_runs"]) == (a.n, d.n)
        self.changed(0)
        self.changed(1)

    def migrate(self, i):
        b, env = self.bs[i], self.env
        old, new = (env.slots[0], self.alt) if self.rng.random() < 0.5 else (self.alt, env.slots[0])
        S = env.S[0]
        step_map = np.arange(S, dtype=np.uint16)
        step_map[self.rng.choice(S, size=2, replace=False)] = T.MIGRATE_GONE
        runs = b.m.migrate(old, new, step_map)
        assert self.fr.resident_migrate(b.h, old, new, step_map, b.n) == len(runs)
        self.changed(i)

    def redrive(self, i):
        b, rng = self.bs[i], self.rng
        runs = rng.choice(b.n, size=2, replace=False)
        rq = np.zeros(2, Frontier.REDRIVE_DTYPE)
        for k, r in enumerate(runs):
            slot = int(b.m.state[r, :4].view("<u4")[0])
            rq[k] = (r, slot, A.REDRIVE_ALL if rng.random() < 0.5 else 0, 0)
        status, _ = self.fr.resident_redrive(b.h, rq)
        b.m.redrive(rq, status, *self.env.resets(rq, b.m.L.words))
        self.changed(i)

    def stop(self, i):
        b, rng = self.bs[i], self.rng
        r = int(rng.integers(0, b.n))
        q = np.zeros(1, R.PUT_DTYPE)
        q[0] = (r, self.now + int(rng.integers(0, 60)), self.now + 30 if rng.random() < 0.5 else R.NONE, int(rng.integers(0, 4)),
                (0, 0, 0))
        assert b.m.put_runctl(q)[0] == 0
        self.fr.resident_runctl_put(b.h, q)
        self.changed(i)

    def resync(self, i):
        b, rng = self.bs[i], self.rng
        n = b.n
        runs = None if rng.random() < 0.4 else np.flatnonzero(rng.random(n) < 0.5).astype(np.uint32)
        listed = np.arange(n) if runs is None else runs
        t, s, c = M.device_areas(b.m, runs=listed)
        if self.prefire[i] is not None and rng.random() < 0.7:   # what the batcher persisted across the last fire
            pt, pc = self.prefire[i]
            t = pt[listed].copy().view(M.SLOT_DTYPE)
            c["drain_deadline"] = pc["drain_deadline"][listed]
        fired_now = self.fired_now[i]
        t, s, c = perturb(rng, b.m, listed, share=float(rng.choice([0.0, 0.1, 0.4])),
                          fired_now=self.now if fired_now == A.TIMER_NONE else fired_now, areas=(t, s, c), step_hi=self.S)
        sel = int(rng.integers(1, 8))
        t, s, c = (t if sel & 1 else None), (s if sel & 2 else None), (c if sel & 4 else None)
        check = rng.random() < 0.3
        self.log[-1] += " %#x%s" % (sel, " check" if check else "")
        want = M.resync(b.m, n, runs=runs, timers=t, sched=s, runctl=c, fired_now=fired_now, check=check)
        assert want["status"] == 0
        got = self.fr.resident_resync_areas(b.h, n, runs=runs, timers=t, sched=s, runctl=c, fired_now=fired_now, check=check)
        assert got["n_items"] == want["items"].size and got["items"].tobytes() == want["items"].tobytes(), \
            (got["items"][:6], want["items"][:6])
        assert got["drifted"].tolist() == want["drifted"].tolist()
        assert got["n_written"] == want["n_written"]
        if want["n_written"]:
            self.changed(i)

    def step(self, k):
        op = OPS[int(self.rng.integers(0, len(OPS)))]
        i = int(self.rng.integers(0, 2))
        self.log.append("%d:%s b%d" % (k, op, i))
        getattr(self, op)(i)
        self.check(op)


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


@pytest.mark.parametrize("seed", range(6))
def test_random_resync_area_sequences(fr, seed):
    q = Seq(fr, seed)
    done = set()
    for k in range(60):
        q.step(k)
        done.add(q.log[-1].split(":")[1].split()[0])
    assert {"fire", "commit", "resync"} <= done
