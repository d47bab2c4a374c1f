"""Touched ticks (bf_resident_tick_touched): only the runs that received a delta or an upload since they were last evaluated are
evaluated, and of those the ones whose record changed (or that were uploaded) are listed.  Every tick is checked three ways:
against the packed oracle's records through compact_events, against a BF_EVAL_CHANGED_ONLY compact tick of a twin batch that
received the same deltas, and by replaying the listed rows into a row cache that must equal the full compact form."""
import os

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier, synth
from bobrapet_b200.records import make_layout
from oracle import packed as PK
from tests import randgen

pytestmark = pytest.mark.gpu

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000


@pytest.fixture
def fr():   # a ctx of its own per test: the kernel a pass takes depends on every topology of the ctx
    f = Frontier(0)
    yield f
    f.close()


def _batch(fr, shape, rng):
    """-> (ts, slots, L, state) of a batch shaped like `shape`"""
    if shape in ("cfg2", "cfg3", "cfg4"):
        cfg = int(shape[3])
        n, S = {2: (3000, 64), 3: (5003, 256), 4: (4001, 256)}[cfg]
        ts = synth.topologies(cfg, 0, n, S)
        slots = fr.put_topologies(ts)
        L = make_layout(S, 0, ALL if cfg == 4 else (A.F_ALL_OUT if cfg == 2 else 0))
        return ts, slots, L, synth.state(cfg, 0, n, L, slots, ts)
    s_lo, s_hi, par = {"parallel": (20, 300, True), "wide": (513, 1000, True), "rand": (30, 256, False)}[shape]
    if shape == "parallel":   # a live topology without parallel steps: the packed-lanes kernel takes the pass, deferring every run
        fr.put_topologies(randgen.random_topologies(rng, 2, 2, 20, parallel=False))
    ts = randgen.random_topologies(rng, 30, s_lo, s_hi, max_deg=4, parallel=par, fill=0.5)
    slots = fr.put_topologies(ts)
    L, state, _ = randgen.random_state(rng, ts, slots, 3001, ALL, phase_mix="progress")
    return ts, slots, L, state


def _deltas(rng, L, ts, slots, n, k, clustered):
    """k deltas (coalesced: one per (run, field, index)) over every field, on a few runs or spread over all of them"""
    runs = rng.choice(n, size=max(1, min(n, k // 40 + 1)), replace=False) if clustered else None
    W32 = 32 * L.words
    fields = [A.DELTA_PHASE] * 6 + [A.DELTA_RUN_FLAGS, A.DELTA_REGISTERED, A.DELTA_TOPO_SLOT]
    if L.off_cond != 0xFFFFFFFF:
        fields += [A.DELTA_COND, A.DELTA_DECISION]
    if L.off_child != 0xFFFFFFFF and L.child_nibbles:
        fields += [A.DELTA_CHILD]
    recs = {}
    for _ in range(k):
        r = int(rng.choice(runs)) if clustered else int(rng.integers(0, n))
        f = int(rng.choice(fields))
        key = None
        if f == A.DELTA_PHASE:
            idx, code = int(rng.integers(0, W32)), int(rng.choice([0, 1, 2, 3, 3, 4, 9, 13, 14]))
        elif f in (A.DELTA_COND, A.DELTA_DECISION):
            idx, code = int(rng.integers(0, W32)), int(rng.integers(0, 4))
        elif f == A.DELTA_CHILD:
            idx, code = int(rng.integers(0, L.child_nibbles)), int(rng.choice([0, 2, 3, 4, 13]))
        elif f == A.DELTA_RUN_FLAGS:
            idx, code = 0, int(rng.choice([0, A.RF_FAIL_FAST, A.RF_FAIL_FAST | A.RF_REALTIME, A.RF_TOPOLOGY_TERMINATED]))
        elif f == A.DELTA_TOPO_SLOT:
            new = int(rng.choice(slots))
            idx, code, key = new & 0xFFFF, new >> 16, 0
        else:
            idx, code = int(rng.integers(0, 64)), int(rng.integers(0, 2))
        recs[(r, f, idx if key is None else key)] = (idx, code)
    d = np.zeros(len(recs), dtype=Frontier.DELTA_DTYPE)
    for i, ((r, f, _), (idx, code)) in enumerate(recs.items()):
        d[i] = (r, idx, f, code)
    return d


class Twin:
    """Batch T takes the ticks under test, batch C the same deltas through changed-only compact ticks.  The host side tracks
    what the contract says: which runs are touched, which must be listed, and each run's current record."""

    def __init__(self, fr, ts, slots, L, state, cap=None):
        self.fr, self.L, self.pt = fr, L, PK.PackedTopologies(ts, slots)
        self.n = state.shape[0]
        cap = cap or self.n
        self.hT, self.hC = fr.resident_create(L, cap), fr.resident_create(L, cap)
        fr.resident_upload(self.hT, 0, state)
        fr.resident_upload(self.hC, 0, state)
        self.cur = np.zeros((cap, L.result_stride), np.uint8)   # the device's current records, as the contract defines them
        self.touched, self.must = set(range(self.n)), set(range(self.n))
        self.c_prev_runs, self.c_comparable = None, False
        self.cache_head, self.cache_ev = {}, {}
        self.n_full = 0

    def close(self):
        self.fr.resident_destroy(self.hT)
        self.fr.resident_destroy(self.hC)

    def upload(self, first, recs):
        self.fr.resident_upload(self.hT, first, recs)
        self.fr.resident_upload(self.hC, first, recs)
        rr = range(first, first + recs.shape[0])
        self.touched |= set(rr)
        self.must |= set(rr)
        self.c_comparable = False

    def apply(self, d):
        self.fr.resident_apply(self.hT, d)
        self.fr.resident_apply(self.hC, d)
        self.touched |= set(int(r) for r in d["run"])

    def _oracle(self, n_runs, flags, max_iter):
        state = self.fr.resident_download(self.hT, 0, n_runs, self.L.state_stride)
        assert np.array_equal(state, self.fr.resident_download(self.hC, 0, n_runs, self.L.state_stride))
        want, _ = PK.evaluate(self.pt, self.L, state, flags & A.EVAL_FIXPOINT, max_iter, threads=8)
        return state, want

    def _changed_only(self, d, n_runs, flags, max_iter):
        comparable = self.c_comparable and self.c_prev_runs == n_runs
        head, ev, n_ev, _, _ = self.fr.resident_tick_compact(self.hC, n_runs, d, BIG, flags=flags | A.EVAL_CHANGED_ONLY,
                                                             max_iterations=max_iter)
        self.c_prev_runs, self.c_comparable = n_runs, True
        starts = np.concatenate(([0], np.cumsum(head >> A.HEAD_COUNT_SHIFT))).astype(np.int64)
        return head, ev, starts, comparable

    def tick(self, d, n_runs=None, flags=0, max_iter=0, runs_cap=None, events_cap=None, pinned=False, kernel=None, full=None):
        fr, L = self.fr, self.L
        n_runs = self.n if n_runs is None else n_runs
        self.touched |= set(int(r) for r in d["run"])
        chead, cev, cstarts, comparable = self._changed_only(d, n_runs, flags, max_iter)
        runs_cap = n_runs if runs_cap is None else runs_cap
        events_cap = BIG if events_cap is None else events_cap
        bufs = {}
        if pinned:
            bufs = {"runs": fr.alloc_pinned(max(runs_cap, 1) * 4).view(np.uint32), "head": fr.alloc_pinned(max(runs_cap, 1) * 4).view(np.uint32),
                    "events": fr.alloc_pinned(max(events_cap, 1) * 2).view(np.uint16)}
        try:
            out = fr.resident_tick_touched(self.hT, n_runs, d, runs_cap, events_cap, flags=flags, max_iterations=max_iter, **bufs)
            out = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in out.items()}
        finally:
            for v in bufs.values():
                fr.free_pinned(v.view(np.uint8))
        state, want = self._oracle(n_runs, flags, max_iter)
        whead, wev, _ = PK.compact_events(L, want)
        wstarts = np.concatenate(([0], np.cumsum(whead >> A.HEAD_COUNT_SHIFT))).astype(np.int64)
        if full is not None:
            assert out["full"] == int(full), out
        if out["full"]:
            self.n_full += 1
            evaluated = list(range(n_runs))
            expect = evaluated
        else:
            evaluated = sorted(r for r in self.touched if r < n_runs)
            expect = [r for r in evaluated if r in self.must or not np.array_equal(want[r], self.cur[r])]
            if kernel is not None and evaluated:
                assert fr.stats()["last_kernel"] == kernel, fr.stats()
            # a changed-only tick on the same device state lists the same runs (when nothing was uploaded since its last tick)
            # with the same heads and events
            clisted = np.nonzero(chead & A.HEAD_LISTED)[0]
            if comparable:
                assert np.array_equal(clisted, np.array(expect, dtype=clisted.dtype)), (clisted[:20], expect[:20])
            for r in set(expect) & set(clisted.tolist()):
                assert chead[r] == whead[r]
                assert np.array_equal(cev[cstarts[r]:cstarts[r + 1]], wev[wstarts[r]:wstarts[r + 1]])
        assert out["n_evaluated"] == len(evaluated) and out["n_listed"] == len(expect), (out["n_evaluated"], len(evaluated), out["n_listed"], len(expect))
        exp = np.array(expect, dtype=np.int64)
        ev_want = np.concatenate([wev[wstarts[r]:wstarts[r + 1]] for r in expect]) if expect else np.zeros(0, np.uint16)
        assert out["n_events"] == len(ev_want)
        assert np.array_equal(out["runs"], exp[:runs_cap]) and np.array_equal(out["head"], whead[exp[:runs_cap]])
        assert np.array_equal(out["events"], ev_want[:events_cap])
        if not flags & A.EVAL_NO_COUNTS:
            sub = np.ascontiguousarray(state[np.array(evaluated, dtype=np.int64)]) if evaluated else state[:0]
            _, wc = PK.evaluate(self.pt, L, sub, flags & A.EVAL_FIXPOINT, max_iter, threads=8) if evaluated else (None, dict(ready=0, skip=0, expansion=0, evals=0))
            assert out["counts"] == wc, (out["counts"], wc)
        # replay the listed rows into a row cache: it must equal the full compact form (a tick whose lists did not fit the
        # caller's capacities is followed by a resync of the cache, as a batcher would do)
        complete = events_cap >= len(ev_want) and runs_cap >= len(expect)
        pos = 0
        for r, hw in zip(out["runs"], out["head"]):
            c = int(hw) >> A.HEAD_COUNT_SHIFT
            self.cache_head[int(r)] = hw
            self.cache_ev[int(r)] = out["events"][pos:pos + c]
            pos += c
        for r in range(n_runs):
            if complete:
                assert self.cache_head[r] == whead[r] and np.array_equal(self.cache_ev[r], wev[wstarts[r]:wstarts[r + 1]]), r
            else:
                self.cache_head[r], self.cache_ev[r] = whead[r], wev[wstarts[r]:wstarts[r + 1]]
        self._evaluated(evaluated, want, full=bool(out["full"]))
        return out

    def _evaluated(self, evaluated, want, full):
        for r in evaluated:
            self.cur[r] = want[r]
        if full:
            self.touched, self.must = set(), set()
        else:
            self.touched -= set(evaluated)
            self.must -= set(evaluated)

    def full_tick(self, kind, d, flags=0, max_iter=0):
        """a tick of another kind on batch T (the twin takes its changed-only tick as always); the row cache is refilled"""
        fr, L = self.fr, self.L
        n = self.n
        self.touched |= set(int(r) for r in d["run"])
        self._changed_only(d, n, flags, max_iter)
        if kind == "dense":
            res, _ = fr.resident_tick(self.hT, L, n, d, flags=flags, max_iterations=max_iter)
        elif kind == "eval":
            if len(d):
                fr.resident_apply(self.hT, d)
            res, _ = fr.resident_eval(self.hT, L, n, flags=flags, max_iterations=max_iter)
        else:
            head, ev, n_ev, _, _ = fr.resident_tick_compact(self.hT, n, d, BIG, flags=flags | (A.EVAL_CHANGED_ONLY if kind == "changed" else 0),
                                                            max_iterations=max_iter)
        _, want = self._oracle(n, flags, max_iter)
        if kind in ("dense", "eval"):
            assert np.array_equal(res, want)
        else:
            # a changed-only tick compares with the batch's current records, which the touched ticks before it kept up to date:
            # it lists exactly the runs whose record differs from the one the host tracked for them
            chead, cev, _ = PK.compact_events(L, want, self.cur[:n] if kind == "changed" else None)
            assert np.array_equal(head, chead) and n_ev == len(cev) and np.array_equal(ev, cev), kind
        whead, wev, _ = PK.compact_events(L, want)
        wstarts = np.concatenate(([0], np.cumsum(whead >> A.HEAD_COUNT_SHIFT))).astype(np.int64)
        for r in range(n):
            self.cache_head[r] = whead[r]
            self.cache_ev[r] = wev[wstarts[r]:wstarts[r + 1]]
        self._evaluated(range(n), want, full=True)


SHAPES = [("cfg2", 4, None), ("cfg3", 4, None), ("cfg4", 4, None), ("parallel", 5, None), ("wide", 3, None),
          ("rand", 3, "general"), ("fixpoint", 3, None)]


@pytest.mark.parametrize("shape,kernel,knob", SHAPES, ids=[s[0] for s in SHAPES])
def test_touched_sequences(fr, shape, kernel, knob):
    rng = np.random.default_rng(700 + [s[0] for s in SHAPES].index(shape))
    ts, slots, L, state = _batch(fr, "parallel" if shape == "fixpoint" else shape, rng)
    flags = A.EVAL_FIXPOINT if shape == "fixpoint" else 0
    n = state.shape[0]
    old = os.environ.get("BF_KERNEL")
    if knob:
        os.environ["BF_KERNEL"] = knob
    tw = Twin(fr, ts, slots, L, state)
    try:
        for it, max_iter in enumerate([0, 2, 0] if flags else [0]):
            out = tw.tick(NONE, flags=flags, max_iter=max_iter, full=True)   # the first tick / a new iteration cap: every run
            assert out["n_listed"] == n
            for k, clustered in ((0, False), (1, False), (40, True), (40, False), (500, True), (500, False), (3000, True), (3000, False)):
                tw.tick(_deltas(rng, L, ts, slots, n, k, clustered), flags=flags, max_iter=max_iter, kernel=kernel, full=False,
                        pinned=(k == 500))
        # list lengths: fewer than R, one group per CTA (132 SMs), several, every run
        for k in (3, 132 * 4 + 1, 132 * 4 * 9, 4 * n):
            tw.tick(_deltas(rng, L, ts, slots, n, k, False), flags=flags, max_iter=max_iter, kernel=kernel, full=False)
        # deltas through bf_resident_apply between ticks, then a tick without deltas
        tw.apply(_deltas(rng, L, ts, slots, n, 300, False))
        tw.tick(NONE, flags=flags, max_iter=max_iter, kernel=kernel, full=False)
        # capacities smaller than the lists
        d = _deltas(rng, L, ts, slots, n, 2000, False)
        tw.tick(d, flags=flags, max_iter=max_iter, runs_cap=7, events_cap=101, full=False)
        tw.tick(_deltas(rng, L, ts, slots, n, 2000, False), flags=flags, max_iter=max_iter, runs_cap=0, events_cap=0, full=False, pinned=True)
        tw.tick(_deltas(rng, L, ts, slots, n, 500, False), flags=flags | A.EVAL_NO_COUNTS, max_iter=max_iter, full=False)
        # a re-upload of a few runs (unchanged records): listed although their records did not change, no full tick
        tw.upload(10, state[10:14].copy())
        out = tw.tick(NONE, flags=flags, max_iter=max_iter, full=False)
        assert set([10, 11, 12, 13]) <= set(out["runs"].tolist())
        # a resync re-uploads everything: every run listed, still not a full tick
        tw.upload(0, state)
        out = tw.tick(NONE, flags=flags, max_iter=max_iter, kernel=kernel, full=False)
        assert out["n_listed"] == n
    finally:
        tw.close()
        if knob:
            if old is None:
                del os.environ["BF_KERNEL"]
            else:
                os.environ["BF_KERNEL"] = old


def test_touched_baseline_rules_and_carried_runs(fr):
    rng = np.random.default_rng(4242)
    ts, slots, L, state = _batch(fr, "cfg3", rng)
    n = state.shape[0]
    tw = Twin(fr, ts, slots, L, state, cap=n + 1000)
    try:
        tw.tick(NONE, full=True)
        tw.upload(n, state[:1000].copy())   # records beyond n_runs; the full ticks below end their "uploaded since"
        tw.tick(_deltas(rng, L, ts, slots, n, 100, False), full=False)
        # runs at or above n_runs stay touched for a later tick that covers them
        d = _deltas(rng, L, ts, slots, n, 600, False)
        tw.tick(d, n_runs=n // 2, full=False)
        assert any(r >= n // 2 for r in tw.touched)
        tw.tick(NONE, full=False)
        assert not any(r < n for r in tw.touched)
        # a topology drop on the ctx (of a slot no run uses)
        spare = fr.put_topologies(randgen.random_topologies(rng, 1, 5, 10, parallel=False))
        tw.tick(NONE, full=False)
        fr.drop_topology(int(spare[0]))
        tw.tick(_deltas(rng, L, ts, slots, n, 50, False), full=True)
        tw.tick(NONE, full=False)
        # the fixpoint flag and the iteration cap
        tw.tick(_deltas(rng, L, ts, slots, n, 50, False), flags=A.EVAL_FIXPOINT, full=True)
        tw.tick(_deltas(rng, L, ts, slots, n, 50, False), flags=A.EVAL_FIXPOINT, full=False, kernel=3)
        tw.tick(NONE, flags=A.EVAL_FIXPOINT, max_iter=3, full=True)
        tw.tick(_deltas(rng, L, ts, slots, n, 50, False), full=True)
        # a larger n_runs: full, unless every run beyond the last full evaluation was uploaded since
        tw.upload(n, state[1000:1400].copy())
        tw.n = n + 400
        tw.tick(NONE, full=False)
        tw.tick(_deltas(rng, L, ts, slots, n + 400, 300, False), full=False)
        tw.n = n + 1000
        tw.tick(NONE, full=True)
        tw.tick(NONE, full=False)
        assert tw.n_full >= 5
    finally:
        tw.close()


def test_touched_flags_are_checked(fr):
    rng = np.random.default_rng(5)
    ts, slots, L, state = _batch(fr, "cfg2", rng)
    h = fr.resident_create(L, state.shape[0])
    try:
        fr.resident_upload(h, 0, state)
        for bad in (A.EVAL_CHANGED_ONLY, A.EVAL_EXPANSION, A.EVAL_VALIDATE, A.EVAL_COUNTS_SET, A.EVAL_PIPELINED):
            with pytest.raises(A.FrontierError):
                fr.resident_tick_touched(h, state.shape[0], NONE, 10, 10, flags=bad)
    finally:
        fr.resident_destroy(h)


@pytest.mark.parametrize("shape", ["cfg3", "cfg4", "parallel"])
def test_touched_interleaved_with_other_ticks_and_schedule(fr, shape):
    from oracle import limiters as LM
    rng = np.random.default_rng(77 + len(shape))
    ts, slots, L, state = _batch(fr, shape, rng)
    n = state.shape[0]
    tw = Twin(fr, ts, slots, L, state)
    sched = np.zeros(n, dtype=LM.SCHED_RUN_DTYPE)
    sched["story_key"], sched["queue_key"] = np.arange(n) % 7, np.arange(n) % 3
    sched["priority"], sched["queued_elapsed_s"], sched["run_phase"] = np.arange(n) % 5, LM.NONE_U32, 2
    story_limit = np.array([0, 1, 50, 400, 0, 3, 2000], np.int32)
    queue_limit, queue_aging = np.array([0, 300, 5000], np.int32), np.array([60, 0, 30], np.int32)
    try:
        tw.tick(NONE, full=True)
        for kind in ["touched", "dense", "touched", "touched", "compact", "touched", "changed", "touched", "touched", "eval",
                     "touched", "changed", "touched", "dense", "changed", "touched"]:
            d = _deltas(rng, L, ts, slots, n, int(rng.integers(0, 800)), bool(rng.integers(0, 2)))
            if kind == "touched":
                tw.tick(d, full=False)
                # bf_schedule after a touched tick sees the complete current records: the same as after a full pass
                got = fr.schedule(L, n, sched, story_limit, queue_limit, queue_aging, global_limit=20000)
                fr.resident_eval(tw.hC, L, n)
                want = fr.schedule(L, n, sched, story_limit, queue_limit, queue_aging, global_limit=20000)
                tw.c_comparable = False   # (the full pass on the twin is not a changed-only tick)
                for k in got:
                    assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k
            else:
                tw.full_tick(kind, d)
    finally:
        tw.close()


def test_c_program_runs_the_go_call_sequence(tmp_path):
    """tests/c_touched_harness.c: Resident.TickTouched's call sequence through go/frontier/shim.h, compiled as C, against a
    changed-only tick of a twin batch"""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, "bobrapet_b200", "lib")
    exe = str(tmp_path / "c_touched_harness")
    cmd = ["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(root, "include"), "-I" + os.path.join(root, "go", "frontier"),
           os.path.join(root, "tests", "c_touched_harness.c"), "-L" + lib, "-lbobrafrontier", "-Wl,-rpath," + lib, "-o", exe]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "c_touched_harness: ok" in out.stdout, (out.stdout, out.stderr)


def test_touched_grid_follows_the_last_tick_not_the_history(fr):
    """the host's bound on the list (which sizes the pass's grid) restarts from each tick's own deltas and carried runs: after
    many ticks with several deltas per run, a tick with three deltas on one run is still planned as one group of one CTA"""
    rng = np.random.default_rng(31)
    ts, slots, L, state = _batch(fr, "cfg3", rng)
    n = state.shape[0]
    tw = Twin(fr, ts, slots, L, state)
    try:
        tw.tick(NONE, full=True)
        for _ in range(6):
            runs = rng.choice(n, size=400, replace=False)
            d = np.zeros(3 * len(runs), dtype=Frontier.DELTA_DTYPE)
            d["run"], d["index"], d["field"] = np.repeat(runs, 3), np.tile([0, 1, 2], len(runs)), A.DELTA_PHASE
            d["code"] = rng.choice([0, 2, 3, 4], size=len(d))
            tw.tick(d, full=False)
        d = np.zeros(3, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"], d["field"], d["code"] = 17, [0, 1, 2], A.DELTA_PHASE, 3
        out = tw.tick(d, full=False, kernel=4)
        assert out["n_evaluated"] == 1
        assert fr.stats()["last_grid"] == 1, fr.stats()
    finally:
        tw.close()
