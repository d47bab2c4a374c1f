"""In passes without cond and decision codes the packed-lanes kernel neither stages nor walks the needs rows of a word whose
dependency floor (1 + the smallest real dependency of the word's walked steps, the per-slot cut table of device_record.h)
lies above every step of the run that is TERMINAL (or RT_SAT, realtime runs): every candidate there waits on an unsatisfied
step, so met = fd = 0 without a walk (frontier_pack.cu, the floor cut).

These batches are progress-shaped, so the cut fires, and put next to that what must keep it from firing: a satisfied,
skipped or failed step far above the frontier, long-range needs and forward references (small floors), CSR and u16 steps
without needs (floor "never"), NODEP steps, fresh runs (nothing terminal), RT_SAT codes above the frontier of realtime runs,
topology-terminated, fail-fast and host-group runs, and topologies with compensation or finally steps (all-zero rows).
Cond and decision passes do not take the cut and must be unchanged.  A slot dropped and re-used by another topology and
an arena compaction between passes check that the floors follow their slots; touched and compact resident ticks run the
run-list and head-word builds.  Every comparison is on whole result records (or head words) against the packed oracle,
with the packed-lanes kernel checked to have run.
"""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import _pack_planes
from oracle import packed as PK
from tests import randgen

pytestmark = pytest.mark.gpu

FIELDS = {"plain": 0, "out": A.F_ALL_OUT, "cond-dec": A.F_COND | A.F_DECISION | A.F_ALL_OUT}
DONE = [3, 3, 3, 3, 13, 4, 11]          # below the frontier: finished, a few skipped / failed
OPEN = [0, 0, 0, 14, 9, 10]             # from the frontier on
TERMINAL = {3, 4, 5, 6, 7, 11, 12, 13}
RT_SAT = {1, 2, 3, 8, 14}
GROUP_MASK = np.uint8(3 << A.SF_GROUP_SHIFT)


def _concat(a: TopologySet, b: TopologySet) -> TopologySet:
    return TopologySet(np.concatenate((a.S, b.S)), np.concatenate((a.E, b.E)), np.concatenate((a.row_ptr, b.row_ptr)),
                       np.concatenate((a.col_idx, b.col_idx)), np.concatenate((a.step_flags, b.step_flags)))


def _topos(rng, case, count=40):
    """main-only topologies without parallel steps; the needs of a step lie in a window below it (as in synth.c) except in
    case "forward" (forward references, long-range needs)"""
    def rt(n, lo, hi, deg, fill, fwd=False):
        return randgen.random_topologies(rng, n, lo, hi, max_deg=deg, groups=False, parallel=False, forward_refs=fwd, fill=fill)
    if case == "byte4-256":
        return rt(count, 256, 256, 4, 0.9)
    if case == "byte2-odd":      # S not a multiple of 32
        return rt(count, 200, 250, 2, 0.8)
    if case == "u16-512":
        return _concat(rt(count // 2, 257, 512, 2, 0.9), rt(count // 2, 257, 512, 4, 0.7))
    if case == "mixed-csr":      # byte rows and CSR records (rows of five needs) inside the same groups
        return _concat(rt(count // 2, 100, 256, 4, 0.9), rt(count // 2, 100, 256, 5, 0.3))
    # forward references and long-range needs: small floors
    return _concat(rt(count // 2, 200, 256, 4, 0.9, fwd=True), rt(count // 2, 257, 400, 4, 0.6, fwd=True))


def _with_groups(rng, ts: TopologySet) -> TopologySet:
    fl = ts.step_flags & ~GROUP_MASK
    pos = 0
    for S in ts.S.astype(np.int64):
        b = int(rng.integers(S // 2, S))
        a = int(rng.integers(S // 4, b + 1))
        fl[pos + a:pos + b] |= np.uint8(1 << A.SF_GROUP_SHIFT)
        fl[pos + b:pos + S] |= np.uint8(2 << A.SF_GROUP_SHIFT)
        pos += S
    return TopologySet(ts.S, ts.E, ts.row_ptr, ts.col_idx, fl)


def _state(rng, ts, slots, n, fields):
    """random_state's run flags with phases per run kind: 0-2 progress (finished below p, open from p); 3 one satisfied,
    skipped or failed step far above p; 4 fresh (all open); 5 RT_SAT codes above p"""
    L, state, topo = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
    s_max = int(ts.S.max())
    phase = np.zeros((n, s_max), np.uint8)
    kind = rng.integers(0, 6, size=n)
    for r in range(n):
        S = int(ts.S[topo[r]])
        p = int(rng.integers(0, min(64, S)))
        k = int(kind[r])
        phase[r, :p] = rng.choice(DONE, size=p)
        phase[r, p:S] = rng.choice(OPEN, size=S - p)
        if k == 3:
            phase[r, int(rng.integers(min(S - 1, p + 64), S))] = rng.choice([3, 13, 4, 6])
        elif k == 4:
            phase[r, :S] = rng.choice(OPEN, size=S)
        elif k == 5:
            phase[r, rng.integers(p, S, size=3)] = rng.choice([1, 2, 8, 14], size=3)
    state[:, L.off_phase:L.off_phase + L.words * 16] = _pack_planes(phase, L.words, 4)
    return L, state, topo, phase


def _floors(ts: TopologySet, i: int):
    """dependency floors of topology i (device_record.h), or None when its row is all zero"""
    off = int(np.cumsum(np.concatenate(([0], ts.S.astype(np.int64))))[i])
    rp0 = int(np.cumsum(np.concatenate(([0], ts.S.astype(np.int64) + 1)))[i])
    S = int(ts.S[i])
    if (ts.step_flags[off:off + S] & GROUP_MASK).any():
        return None
    rp = ts.row_ptr[rp0:rp0 + S + 1].astype(np.int64)
    e0 = int(np.cumsum(np.concatenate(([0], ts.E.astype(np.int64))))[i])
    ci = ts.col_idx[e0:e0 + int(ts.E[i])].astype(np.int64)
    out = []
    for w in range((S + 31) // 32):
        deps = [ci[rp[j]:rp[j + 1]] for j in range(32 * w, min(S, 32 * w + 32))]
        out.append(None if any(d.size == 0 for d in deps) else 1 + min(int(d.min()) for d in deps if d.size))
    return out


def _cut_words(ts, state, topo, phase):
    """(run, word) pairs with an open step whose floor lies above every TERMINAL (RT_SAT: realtime) step: the words the
    cut leaves out, counted on the runs it applies to (not topology-terminated; fail-fast runs with a failure may count)"""
    rf = state[:, 4]
    fl = {}
    n = 0
    for r in range(state.shape[0]):
        if rf[r] & A.RF_TOPOLOGY_TERMINATED:
            continue
        t = int(topo[r])
        if t not in fl:
            fl[t] = _floors(ts, t)
        if fl[t] is None:
            continue
        S = int(ts.S[t])
        codes = set(TERMINAL) | (RT_SAT if rf[r] & A.RF_REALTIME else set())
        b = np.nonzero(np.isin(phase[r, :S], list(codes)))[0]
        hs = int(b.max()) + 1 if b.size else 0
        for w, f in enumerate(fl[t]):
            if f is not None and f > hs and np.isin(phase[r, 32 * w:min(S, 32 * w + 32)], [0, 9, 10, 14]).any():
                n += 1
    return n


def _check(f, ts, slots, L, state):
    want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=8)
    got, gcounts = f.eval(L, state, flags=A.EVAL_VALIDATE)
    assert f.stats()["last_kernel"] == 1, f.stats()
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, (bad.size, bad[:10])
    assert gcounts == wcounts
    return want


@pytest.fixture(autouse=True)
def _default_formats(monkeypatch):
    monkeypatch.delenv("BF_KERNEL", raising=False)
    monkeypatch.delenv("BF_TOPO_FORMAT", raising=False)


@pytest.mark.parametrize("fields", list(FIELDS))
@pytest.mark.parametrize("case", ["byte4-256", "byte2-odd", "u16-512", "mixed-csr", "forward"])
def test_floor_cut_matches_oracle(case, fields):
    rng = np.random.default_rng(9100 + 10 * list(FIELDS).index(fields) + len(case))
    ts = _topos(rng, case)
    f = Frontier(0)
    try:
        slots = f.put_topologies(ts)
        L, state, topo, phase = _state(rng, ts, slots, 6001, FIELDS[fields])
        if case != "forward":
            assert _cut_words(ts, state, topo, phase) > 500
        _check(f, ts, slots, L, state)
    finally:
        f.close()


@pytest.mark.parametrize("fields", ["plain", "cond-dec"])
def test_floor_cut_compensation_and_finally(fields):
    rng = np.random.default_rng(9201 if fields == "plain" else 9202)
    ts = _concat(_topos(rng, "byte4-256", 30), _with_groups(rng, _topos(rng, "byte4-256", 30)))
    f = Frontier(0)
    try:
        slots = f.put_topologies(ts)
        L, state, topo, phase = _state(rng, ts, slots, 6001, FIELDS[fields])
        _check(f, ts, slots, L, state)
    finally:
        f.close()


def test_floor_cut_slot_reuse_and_compaction():
    """a dropped slot re-used by a topology with long-range needs, then by one with finally steps, must carry its new
    floors; an arena compaction moves records and leaves the floors with their slots"""
    rng = np.random.default_rng(9301)
    f = Frontier(0)
    try:
        a = _topos(rng, "byte4-256", 60)
        slots_a = f.put_topologies(a)
        _check(f, a, slots_a, *_state(rng, a, slots_a, 4001, 0)[:2])
        for s in slots_a:
            f.drop_topology(int(s))
        b = _topos(rng, "forward", 60)
        slots_b = f.put_topologies(b)
        assert set(slots_b.tolist()) == set(slots_a.tolist())
        _check(f, b, slots_b, *_state(rng, b, slots_b, 4001, 0)[:2])
        for s in slots_b:
            f.drop_topology(int(s))
        c = _with_groups(rng, _topos(rng, "byte4-256", 60))
        slots_c = f.put_topologies(c)
        _check(f, c, slots_c, *_state(rng, c, slots_c, 4001, 0)[:2])

        keep = _topos(rng, "byte4-256", 40)
        slots_keep = f.put_topologies(keep)
        gone = _topos(rng, "byte4-256", 1200)
        for s in f.put_topologies(gone):
            f.drop_topology(int(s))
        before = f.stats()["arena_compactions"]
        late = _topos(rng, "u16-512", 40)
        slots_late = f.put_topologies(late)
        assert f.stats()["arena_compactions"] == before + 1
        ts = _concat(_concat(c, keep), late)
        slots = np.concatenate((slots_c, slots_keep, slots_late))
        L, state, topo, phase = _state(rng, ts, slots, 6001, 0)
        assert _cut_words(ts, state, topo, phase) > 300
        _check(f, ts, slots, L, state)
    finally:
        f.close()


def test_floor_cut_resident_compact_and_touched_ticks():
    """a compact tick (fused head words) over the whole batch, then a touched tick (run-list build) over the runs a
    handful of deltas changed: head words and events against the oracle on the downloaded state"""
    rng = np.random.default_rng(9401)
    ts = _topos(rng, "byte4-256", 40)
    f = Frontier(0)
    try:
        slots = f.put_topologies(ts)
        n = 8001
        L, state, topo, phase = _state(rng, ts, slots, n, 0)
        pt = PK.PackedTopologies(ts, slots)
        h = f.resident_create(L, n)
        f.resident_upload(h, 0, state)
        none = np.zeros(0, dtype=f.DELTA_DTYPE)
        head, events, _, _, n_listed = f.resident_tick_compact(h, n, none, 1 << 22)
        want, _ = PK.evaluate(pt, L, f.resident_download(h, 0, n, L.state_stride), threads=8)
        whead, wev, _ = PK.compact_events(L, want)
        assert n_listed == n and np.array_equal(head, whead) and np.array_equal(events, wev)
        f.resident_tick_touched(h, n, none, n, 1 << 22)   # the first touched tick is a full one
        d = np.zeros(300, dtype=f.DELTA_DTYPE)
        d["run"] = rng.choice(n, size=300, replace=False)
        d["index"] = rng.integers(0, 256, size=300)
        d["field"] = A.DELTA_PHASE
        d["code"] = rng.choice([3, 4, 13, 0, 14], size=300)
        out = f.resident_tick_touched(h, n, d, n, 1 << 22)
        assert not out["full"] and f.stats()["last_kernel"] in (4, 5), (out["full"], f.stats())
        want, _ = PK.evaluate(pt, L, f.resident_download(h, 0, n, L.state_stride), threads=8)
        whead, _, _ = PK.compact_events(L, want)
        k = out["n_listed"]
        runs = out["runs"][:k]
        assert k > 0 and np.array_equal(out["head"][:k], whead[runs])
        f.resident_destroy(h)
    finally:
        f.close()
