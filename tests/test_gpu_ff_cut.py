"""The packed-lanes kernel stages no needs rows for a fail-fast run that already has a Failed main step without allowFailure
in a topology without compensation or finally steps (frontier_pack.cu, the cut; the per-slot fail-fast masks of
device_record.h), and in passes without decision codes it stages the type planes from AF on.

These batches put failures of every code of TERMINAL \\ COMPLETED0 (4, 5, 6, 7, 11, 12) above and below the first word
that can hold a candidate, on allowFailure steps only, and nowhere at all, over fail-fast, host-group, realtime and
topology-terminated runs, with and without cond / decision codes (passes with them do not take the skip: they check
that the rest of the cut is unchanged there).  Topologies with compensation or finally steps (whose
masks are zero), a slot dropped and re-used by such a topology, and an arena compaction between passes check that the
masks follow the slots.  Every comparison is on whole result records against the packed oracle, with the packed-lanes
kernel checked to have run.
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

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
FIELDS = {"plain": 0, "out": A.F_ALL_OUT, "cond": A.F_COND | A.F_ALL_OUT, "cond-dec": ALL}
FAILED = [4, 5, 6, 7, 11, 12]                  # TERMINAL \ COMPLETED0
FINISHED = [3, 13, 2, 8, 1]                    # finished or running, not failed
FINISHED_P = [0.8, 0.05, 0.07, 0.04, 0.04]
OPEN = [0, 9, 10, 14]
GROUP_MASK = np.uint8(3 << A.SF_GROUP_SHIFT)


def _concat(a: TopologySet, b: TopologySet) -> TopologySet:
    return TopologySet(np.concatenate((a.S, b.S)), np.concatenate((a.E, b.E)), np.concatenate((a.row_ptr, b.row_ptr)),
                       np.concatenate((a.col_idx, b.col_idx)), np.concatenate((a.step_flags, b.step_flags)))


def _main_only(rng, case, count=40):
    if case == "byte4-256":
        return randgen.random_topologies(rng, count, 225, 256, max_deg=4, groups=False, parallel=False, fill=0.9)
    if case == "byte2-256":
        return randgen.random_topologies(rng, count, 200, 256, max_deg=2, groups=False, parallel=False, fill=0.8)
    if case == "u16-512":
        return _concat(randgen.random_topologies(rng, count // 2, 257, 512, max_deg=2, groups=False, parallel=False, fill=0.9),
                       randgen.random_topologies(rng, count // 2, 257, 512, max_deg=4, groups=False, parallel=False, fill=0.9))
    # byte rows and CSR records (rows of five needs) inside the same groups
    return _concat(randgen.random_topologies(rng, count // 2, 100, 256, max_deg=4, groups=False, parallel=False, fill=0.9),
                   randgen.random_topologies(rng, count // 2, 100, 256, max_deg=5, groups=False, parallel=False, fill=0.3))


def _with_groups(rng, ts: TopologySet) -> TopologySet:
    """the same graphs with a compensation range and a non-empty finally range at the end of every topology"""
    fl = ts.step_flags & ~GROUP_MASK
    pos = 0
    for S in ts.S.astype(np.int64):
        b = int(rng.integers(S // 2, S))           # finally: [b, S), at least one step
        a = int(rng.integers(S // 4, b + 1))       # compensation: [a, b), possibly empty
        fl[pos + a:pos + b] |= np.uint8(1 << A.SF_GROUP_SHIFT)
        fl[pos + b:pos + S] |= np.uint8(2 << A.SF_GROUP_SHIFT)
        pos += S
    return TopologySet(ts.S, ts.E, ts.row_ptr, ts.col_idx, fl)


def _flags_of(ts: TopologySet):
    off = np.concatenate(([0], np.cumsum(ts.S.astype(np.int64))))
    return [ts.step_flags[off[i]:off[i + 1]] for i in range(ts.count)]


def _ff_state(rng, ts, slots, n, fields):
    """random_state's runs (flags, cond and decision codes) with progress-shaped phases and failures placed per run:
    0: one failure on a step without allowFailure, anywhere; 1: failures on allowFailure steps only; 2: a failure in the
    last word and open steps from the first; 3: a failure in the first word and open steps from a later one; 4: RUNNING /
    PENDING / PAUSED prefix (stage-G gates) and no failure; 5: no failure"""
    L, state, topo = randgen.random_state(rng, ts, slots, n, fields, phase_mix="progress")
    flags = _flags_of(ts)
    s_max = int(ts.S.max())
    phase = np.zeros((n, s_max), np.uint8)
    kind = rng.integers(0, 6, size=n)
    for r in range(n):
        S = int(ts.S[topo[r]])
        W = (S + 31) // 32
        af = (flags[topo[r]] & A.SF_ALLOW_FAILURE) != 0
        p = int(rng.integers(0, S + 1))
        phase[r, :S] = rng.choice(FINISHED, size=S, p=FINISHED_P)
        phase[r, p:S] = np.where(rng.random(S - p) < 0.7, rng.choice(OPEN, size=S - p), phase[r, p:S])
        k = int(kind[r])
        strict = np.nonzero(~af)[0]
        if k == 0 and strict.size:
            phase[r, rng.choice(strict)] = rng.choice(FAILED)
        elif k == 1 and af.any():
            idx = np.nonzero(af)[0]
            phase[r, rng.choice(idx, size=min(3, idx.size), replace=False)] = rng.choice(FAILED, size=min(3, idx.size))
        elif k == 2 and W > 1:
            phase[r, :32] = rng.choice(OPEN, size=32)
            hi = [i for i in strict if i >= 32 * (W - 1)]
            if hi:
                phase[r, rng.choice(hi)] = rng.choice(FAILED)
        elif k == 3 and W > 1:
            lo = [i for i in strict if i < 32]
            if lo:
                phase[r, :32] = rng.choice(FINISHED, size=32, p=FINISHED_P)
                phase[r, rng.choice(lo)] = rng.choice(FAILED)
                j = int(rng.integers(1, W))
                phase[r, 32 * j:S] = rng.choice(OPEN, size=S - 32 * j)
        elif k == 4:
            phase[r, :p] = rng.choice([2, 2, 2, 1, 8], size=p)
    state[:, L.off_phase:L.off_phase + L.words * 16] = _pack_planes(phase, L.words, 4)
    return L, state, topo, phase


def _skippable(ts, state, topo, phase):
    """runs whose rows the kernel does not stage: fail-fast, group not set by the host, no compensation / finally step,
    a failure code on a step without allowFailure"""
    flags = _flags_of(ts)
    rf = state[:, 4]
    out = 0
    for r in range(state.shape[0]):
        f = flags[topo[r]]
        if (rf[r] & (A.RF_FAIL_FAST | A.RF_HOST_GROUP)) != A.RF_FAIL_FAST or (f & GROUP_MASK).any():
            continue
        S = f.shape[0]
        out += bool((np.isin(phase[r, :S], FAILED) & ((f & A.SF_ALLOW_FAILURE) == 0)).any())
    return out


def _check(f, ts, slots, L, state):
    want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=8)
    got, gcounts = f.eval(L, state, flags=A.EVAL_VALIDATE)
    assert f.stats()["last_kernel"] == 1, f.stats()
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, (bad.size, bad[:10])
    assert gcounts == wcounts


@pytest.fixture(autouse=True)
def _default_formats(monkeypatch):
    monkeypatch.delenv("BF_KERNEL", raising=False)
    monkeypatch.delenv("BF_TOPO_FORMAT", raising=False)


@pytest.mark.parametrize("fields", list(FIELDS))
@pytest.mark.parametrize("case", ["byte4-256", "byte2-256", "u16-512", "mixed-csr"])
def test_ff_cut_matches_oracle(case, fields):
    rng = np.random.default_rng(8100 + 10 * list(FIELDS).index(fields) + len(case))
    ts = _main_only(rng, case)
    f = Frontier(0)
    try:
        slots = f.put_topologies(ts)
        L, state, topo, phase = _ff_state(rng, ts, slots, 6001, FIELDS[fields])
        assert _skippable(ts, state, topo, phase) > 300
        _check(f, ts, slots, L, state)
    finally:
        f.close()


@pytest.mark.parametrize("fields", ["plain", "cond-dec"])
def test_ff_cut_compensation_and_finally(fields):
    """topologies with compensation / finally steps have zero masks: a failed fail-fast run moves to those groups and
    walks their rows; batches mix them with main-only topologies"""
    rng = np.random.default_rng(8201 if fields == "plain" else 8202)
    main = _main_only(rng, "byte4-256", 30)
    ts = _concat(main, _with_groups(rng, _main_only(rng, "byte4-256", 30)))
    f = Frontier(0)
    try:
        slots = f.put_topologies(ts)
        L, state, topo, phase = _ff_state(rng, ts, slots, 6001, FIELDS[fields])
        _check(f, ts, slots, L, state)
    finally:
        f.close()


def test_ff_cut_slot_reuse_and_compaction():
    """a dropped main-only slot re-used by a topology with finally steps must carry a zero mask; an arena compaction
    moves records and leaves the masks with their slots"""
    rng = np.random.default_rng(8301)
    f = Frontier(0)
    try:
        a = _main_only(rng, "byte4-256", 60)
        slots_a = f.put_topologies(a)
        L, state, topo, phase = _ff_state(rng, a, slots_a, 4001, ALL)
        _check(f, a, slots_a, L, state)
        for s in slots_a:
            f.drop_topology(int(s))
        b = _with_groups(rng, _main_only(rng, "byte4-256", 60))
        slots_b = f.put_topologies(b)
        assert set(slots_b.tolist()) == set(slots_a.tolist())
        for fields in ("plain", "cond-dec"):
            L, state, topo, phase = _ff_state(rng, b, slots_b, 4001, FIELDS[fields])
            _check(f, b, slots_b, L, state)

        keep = _main_only(rng, "byte4-256", 40)
        slots_keep = f.put_topologies(keep)
        gone = _main_only(rng, "byte4-256", 1200)
        for s in f.put_topologies(gone):
            f.drop_topology(int(s))
        before = f.stats()["arena_compactions"]
        late = _main_only(rng, "byte2-256", 40)
        slots_late = f.put_topologies(late)
        assert f.stats()["arena_compactions"] == before + 1
        ts = _concat(_concat(b, keep), late)
        slots = np.concatenate((slots_b, slots_keep, slots_late))
        for fields in ("plain", "cond"):
            L, state, topo, phase = _ff_state(rng, ts, slots, 6001, FIELDS[fields])
            assert _skippable(ts, state, topo, phase) > 200
            _check(f, ts, slots, L, state)
    finally:
        f.close()


def test_ff_cut_long_batch_and_pipelined_rotation():
    """70 001 runs (every slot group re-armed many times, so a run without rows finds another topology's rows in its
    buffer), then pipelined passes rotating over three batches with different fields on one stream"""
    import torch
    rng = np.random.default_rng(8401)
    f = Frontier(0)
    try:
        sets = []
        for case, n, fields in (("byte4-256", 70001, "plain"), ("u16-512", 20011, "cond-dec"), ("byte2-256", 30011, "cond")):
            ts = _main_only(rng, case)
            slots = f.put_topologies(ts)
            L, state, topo, phase = _ff_state(rng, ts, slots, n, FIELDS[fields])
            want, wc = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=16)
            if n > 70000:
                got, gc = f.eval(L, state)
                assert f.stats()["last_kernel"] == 1, f.stats()
                bad = np.nonzero((got != want).any(axis=1))[0]
                assert bad.size == 0 and gc == wc, (bad.size, bad[:10], gc, wc)
            sets.append((L, n, state, want, wc))
        dev = torch.device("cuda", 0)
        bufs = [(torch.from_numpy(st).to(dev), torch.zeros((n, L.result_stride), dtype=torch.uint8, device=dev),
                 torch.zeros(4, dtype=torch.int64, device=dev)) for L, n, st, _, _ in sets]
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for _ in range(3):
                for (L, n, _, _, _), (d_state, d_result, d_counts) in zip(sets, bufs):
                    f.eval_device(L, n, d_state.data_ptr(), d_result.data_ptr(), d_counts.data_ptr(), s.cuda_stream,
                                  flags=A.EVAL_COUNTS_SET | A.EVAL_PIPELINED)
        torch.cuda.synchronize()
        assert f.stats()["last_kernel"] == 1, f.stats()
        for (L, n, _, want, wc), (_, d_result, d_counts) in zip(sets, bufs):
            got = d_result.cpu().numpy()
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, (n, bad.size, bad[:10])
            assert d_counts.cpu().numpy().tolist() == [wc["ready"], wc["skip"], wc["expansion"], wc["evals"]]
    finally:
        f.close()
