"""Launch shapes forced through the A/B knobs, each checked against the oracle on whole records and against stats() for
the shape that really ran.  The planner picks one shape per batch; these cases reach the builds and shapes it does not
pick for the suite's other data: the packed-lanes walk paths on groups of one row format, small and large rings, R = 1,
reduced grids, and every general-kernel instance (register budget RB 0 / 1 / 2, fixpoint, run list).  A knob the planner
refuses fails the case: every case asserts the shape it asked for."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from tests import randgen
from tests.test_gpu_parity import _compare

pytestmark = pytest.mark.gpu

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
KNOBS = ("BF_KERNEL", "BF_TOPO_FORMAT", "BF_WARPS", "BF_GROUPS", "BF_STAGES", "BF_BLOCKS_PER_SM", "BF_WQ", "BF_ASSIGN",
         "BF_PACK_CTAS", "BF_E2E_CHUNKS")
BUDGET = 227 * 1024          # shared memory a CTA may use (kSmemBudget, abi.cu)
PACK_MAX_WARPS = 24


def _r16(x):
    return (x + 15) // 16 * 16


def _up(x, a):
    return (x + a - 1) // a * a


@pytest.fixture(scope="module")
def sms():
    f = Frontier(0)
    try:
        return f.stats()["sm_count"]
    finally:
        f.close()


def _fresh(monkeypatch, env, reserve_sms=0):
    """a new ctx under exactly these knobs (BF_TOPO_FORMAT is read at upload, so set before put_topologies); one pass
    per eval, so that stats() describes the whole batch"""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("BF_E2E_CHUNKS", "1")
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    return Frontier(0, reserve_sms=reserve_sms)


def _max_deg(ts, t):
    R_off = np.concatenate(([0], np.cumsum(ts.S.astype(np.int64) + 1)))
    rp = ts.row_ptr[R_off[t]:R_off[t] + int(ts.S[t]) + 1].astype(np.int64)
    return int((rp[1:] - rp[:-1]).max()) if ts.S[t] else 0


def _row_kinds(f, ts, slots, fmt=None):
    """the device row format of each topology without parallel steps, read off its record size (device_record.h);
    fmt: the BF_TOPO_FORMAT of the upload (csr: CSR only, ell16: no byte entries)"""
    kinds = []
    for t in range(ts.count):
        S, E, md = int(ts.S[t]), int(ts.E[t]), _max_deg(ts, t)
        W = (S + 31) // 32
        K = 2 if md <= 2 else 4
        sizes = {"byte%d" % K: _r16(32 + K * 32 * W + _r16(9 * 4 * W)), "u16-%d" % K: _r16(32 + 2 * K * 32 * W + _r16(8 * 4 * W)),
                 "csr%s" % ("4" if md <= 4 else "L"): _r16(32 + _r16(2 * (S + 1)) + _r16(2 * E + 8) + _r16(8 * 4 * W))}
        nbytes = f.topology_record(int(slots[t]))[1]
        allowed = lambda k: (md <= 4 or k.startswith("csr")) and (fmt != "csr" or k.startswith("csr")) and \
            (fmt != "ell16" or not k.startswith("byte"))  # noqa: E731
        hit = [k for k, v in sizes.items() if v == nbytes and allowed(k)]
        assert len(hit) == 1, (t, S, E, md, nbytes, sizes)
        kinds.append(hit[0])
    return kinds


def _pack_plan(f, L, slots, warps=PACK_MAX_WARPS, groups=None, wq_min=0):
    """the packed-lanes plan of abi.cu (plan_pack) for a batch large enough that no CTA is short of groups: (R, warps, slot groups,
    shared memory, bytes per group)"""
    wq = 1
    while wq < L.words:
        wq <<= 1
    while wq < wq_min and wq < 32:
        wq <<= 1
    R = 32 // wq
    stage = L.state_stride + _r16(max(f.topology_record(int(s))[1] for s in slots))
    st_stride = 256 if wq == 8 else 32 * wq + 16
    work = _up(R * st_stride + 128 + 16 * R, 256)

    def groups_for(w):
        fixed = 128 + 768 + 256 + w * work
        return min(64, (BUDGET - fixed) // (R * stage) if fixed < BUDGET else 0)

    nw = max(1, min(warps, PACK_MAX_WARPS))
    while nw > 1 and groups_for(nw) < nw:
        nw -= 1
    ng = min(groups_for(nw), 32 * nw)   # one thread per slot group sets up its barrier
    if groups is not None and nw <= groups <= ng:
        ng = groups
    smem = 128 + _up(ng * 12, 128) + ng * R * stage + 256 + nw * work
    return R, nw, ng, smem


def _assert_pack(st, R, nw, ng, grid, smem):
    assert st["last_kernel"] == 1, st
    assert (st["last_runs_per_trip"], st["last_block"], st["last_stages"], st["last_grid"], st["last_smem_bytes"]) == \
        (R, 32 * nw, ng, grid, smem), st


# ---------------------------------------------------------------------------------------------------------------------
# packed lanes: the eight walk paths (frontier_pack.cu), each with and without failed-dependency bits
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {   # name: (BF_TOPO_FORMAT, S range, max_deg, fill, the row format every topology must get)
    "mixed": (None, (5, 120), 5, 0.0, None),
    "byte4-wq8": (None, (225, 256), 4, 0.9, "byte4"),
    "byte4": (None, (97, 128), 4, 0.9, "byte4"),
    "byte2": (None, (97, 128), 2, 0.9, "byte2"),
    "u16-4": ("ell16", (128, 128), 4, 1.0, "u16-4"),
    "u16-2": ("ell16", (128, 128), 2, 1.0, "u16-2"),
    "csr4": ("csr", (97, 128), 4, 0.5, "csr4"),
    "csrL": (None, (97, 128), 8, 0.6, "csrL"),
}
IO = [0, A.F_COND | A.F_DECISION, A.F_ALL_OUT, ALL]   # <CD, XO> = 00, 10, 01, 11


@pytest.mark.parametrize("any_fd", [False, True])
@pytest.mark.parametrize("walk", list(WALKS))
def test_pack_walk_paths(monkeypatch, walk, any_fd):
    """groups uniform in one row format take that format's walk; `mixed` groups take the any-format walk.  any_fd = False:
    every run fail-fast (no failed-dependency class in any group); True: no run fail-fast (every main-group run has one)"""
    fmt, (smin, smax), deg, fill, kind = WALKS[walk]
    f = _fresh(monkeypatch, {"BF_TOPO_FORMAT": fmt} if fmt else {})
    try:
        i = list(WALKS).index(walk)
        rng = np.random.default_rng(4100 + 2 * i + any_fd)
        ts = randgen.random_topologies(rng, 40, smin, smax, max_deg=deg, parallel=False, fill=fill)
        slots = f.put_topologies(ts)
        kinds = _row_kinds(f, ts, slots, fmt)
        if kind is None:
            assert len(set(kinds)) >= 2, kinds
        else:
            assert set(kinds) == {kind}, kinds
        fields = IO[(2 * i + any_fd) % 4]
        L, state, _ = randgen.random_state(rng, ts, slots, 6000, fields, phase_mix=("any" if i % 2 else "progress"),
                                           fail_fast=not any_fd)
        _compare(f, ts, slots, L, state)
        R, nw, ng, smem = _pack_plan(f, L, slots)
        assert R == (4 if walk == "byte4-wq8" else 8)
        st = f.stats()
        assert st["last_kernel"] == 1 and st["last_runs_per_trip"] == R, st
    finally:
        f.close()


# ---------------------------------------------------------------------------------------------------------------------
# packed lanes: forced shapes (warps, ring depth, runs per trip, grid)
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = {   # name: (env, reserve: "none" | "one" | "all-but-one")
    "w1": ({"BF_WARPS": 1}, "none"),
    "w8": ({"BF_WARPS": 8}, "none"),
    "w24": ({"BF_WARPS": 24}, "none"),
    "w1-ring-min": ({"BF_WARPS": 1, "BF_GROUPS": 8}, "none"),
    "w8-ring-min": ({"BF_WARPS": 8, "BF_GROUPS": 8}, "none"),
    "w24-ring-min": ({"BF_WARPS": 24, "BF_GROUPS": 24}, "none"),
    "R1": ({"BF_WQ": 32}, "none"),
    "R2": ({"BF_WQ": 16}, "none"),
    "reserve-1": ({}, "one"),
    "one-cta": ({}, "all-but-one"),
    "one-cta-ring-min": ({"BF_WARPS": 8, "BF_GROUPS": 8}, "all-but-one"),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_pack_forced_shapes(monkeypatch, sms, shape):
    """every CTA draws at least 4 x NG groups, so that each slot group of its ring is re-armed at least three times"""
    env, reserve = SHAPES[shape]
    k = {"none": 0, "one": 1, "all-but-one": sms - 1}[reserve]
    f = _fresh(monkeypatch, env, reserve_sms=k)
    try:
        rng = np.random.default_rng(4300 + list(SHAPES).index(shape))
        ts = randgen.random_topologies(rng, 50, 225, 256, max_deg=4, parallel=False, fill=0.9)
        slots = f.put_topologies(ts)
        L, _, _ = randgen.random_state(rng, ts, slots, 1, ALL)
        R, nw, ng, smem = _pack_plan(f, L, slots, warps=int(env.get("BF_WARPS", PACK_MAX_WARPS)), groups=env.get("BF_GROUPS"),
                                     wq_min=int(env.get("BF_WQ", 0)))
        if "BF_WARPS" in env:
            assert nw == env["BF_WARPS"], (nw, ng)
        if "BF_GROUPS" in env:
            assert ng == env["BF_GROUPS"], (nw, ng)
        if "BF_WQ" in env:
            assert R == 32 // env["BF_WQ"]
        if shape == "w1":
            assert ng == 32, ng   # 35 slot groups would fit: capped at one per thread of the one-warp CTA
        grid = sms - k
        n = 4 * R * ng * grid + R - 1          # + a partial last group
        L, state, _ = randgen.random_state(rng, ts, slots, n, ALL, phase_mix=("any" if ng % 2 else "progress"))
        _compare(f, ts, slots, L, state)
        _assert_pack(f.stats(), R, nw, ng, grid, smem)
    finally:
        f.close()


# ---------------------------------------------------------------------------------------------------------------------
# the one-run-per-warp kernel: all 36 instances (frontier_kernel.cu)
# ---------------------------------------------------------------------------------------------------------------------
def _general_smem(f, L, slots, wpb, st):
    stage = L.state_stride + _r16(max(f.topology_record(int(s))[1] for s in slots))
    work = _r16(4 * L.words) + 32 * L.words + 16
    return 128 + wpb * (st * stage + work + 64)


def _topologies(rng, ch, smin, smax):
    ts = randgen.random_topologies(rng, 30, smin, smax, max_deg=4, parallel=ch, fill=0.5)
    assert (ts.P.sum() > 0) == ch
    return ts


@pytest.mark.parametrize("rb", [0, 1, 2])
@pytest.mark.parametrize("ch", [False, True])
@pytest.mark.parametrize("io", [0, 1, 2, 3])
def test_general_single_pass_builds(monkeypatch, sms, rb, ch, io):
    """RB 2: 24 warps (the 80-register build, one CTA per SM); RB 1: 16 warps with two CTAs per SM (the 64-register build);
    RB 0: 16 warps whose ring of stages leaves room for one CTA only.  CH: the ctx holds a topology with parallel steps."""
    f = _fresh(monkeypatch, {"BF_KERNEL": "general", "BF_WARPS": 24 if rb == 2 else 16})
    try:
        rng = np.random.default_rng(4500 + 8 * rb + 4 * ch + io)
        ts = _topologies(rng, ch, *((400, 512) if rb == 0 else (10, 64)))
        slots = f.put_topologies(ts)
        n = 2 * sms * 24 + 5
        L, state, _ = randgen.random_state(rng, ts, slots, n, IO[io], phase_mix=("any" if io % 2 else "progress"))
        wpb = 24 if rb == 2 else 16
        if rb == 0:   # the smallest ring that two 16-warp CTAs cannot share an SM with
            fit = [st for st in (1, 2, 3, 4) if 116 * 1024 < _general_smem(f, L, slots, 16, st) <= BUDGET]
            assert fit, [_general_smem(f, L, slots, 16, st) for st in (1, 2, 3, 4)]
            monkeypatch.setenv("BF_STAGES", str(fit[0]))
        _compare(f, ts, slots, L, state, expansion=ch)
        st = f.stats()
        assert st["last_kernel"] == 0 and st["last_block"] == 32 * wpb, st
        assert st["last_grid"] == (2 * sms if rb == 1 else sms), st
        assert st["last_smem_bytes"] == _general_smem(f, L, slots, wpb, st["last_stages"]), st
        if rb == 1:
            assert 2 * (st["last_smem_bytes"] + 1024) <= 228 * 1024, st
    finally:
        f.close()


@pytest.mark.parametrize("ch", [False, True])
@pytest.mark.parametrize("io", [0, 1, 2, 3])
def test_general_fixpoint_builds(monkeypatch, sms, ch, io):
    """the eight fixpoint instances (RB 0 only: the fixpoint is never planned at more than 16 warps)"""
    f = _fresh(monkeypatch, {})
    try:
        rng = np.random.default_rng(4600 + 4 * ch + io)
        ts = _topologies(rng, ch, 10, 200)
        slots = f.put_topologies(ts)
        L, state, _ = randgen.random_state(rng, ts, slots, 2 * sms * 16 + 3, IO[io], phase_mix="progress")
        _compare(f, ts, slots, L, state, flags=A.EVAL_FIXPOINT, expansion=ch)
        st = f.stats()
        assert st["last_kernel"] == 0 and st["last_block"] <= 512, st
    finally:
        f.close()


@pytest.mark.parametrize("io", [0, 1, 2, 3])
def test_general_run_list_builds(monkeypatch, io):
    """the four run-list instances: the second tier of a packed-lanes pass over a ctx where only some topologies have
    parallel steps (the runs of those are deferred to the general kernel)"""
    f = _fresh(monkeypatch, {})
    try:
        rng = np.random.default_rng(4700 + io)
        ts = randgen.random_topologies(rng, 40, 3, 60, max_deg=4, fill=0.5)
        assert 0 < int((ts.P > 0).sum()) < ts.count
        slots = f.put_topologies(ts)
        L, state, _ = randgen.random_state(rng, ts, slots, 5000, IO[io], phase_mix=("any" if io % 2 else "progress"))
        _compare(f, ts, slots, L, state, expansion=True)
        assert f.stats()["last_kernel"] == 2, f.stats()
    finally:
        f.close()


@pytest.mark.parametrize("knob", ["stages-1", "stages-2", "stages-3", "stages-4", "blocked"])
def test_general_ring_depths_and_assignment(monkeypatch, sms, knob):
    env = {"BF_KERNEL": "general", "BF_WARPS": 16}
    if knob == "blocked":
        env["BF_ASSIGN"] = "blocked"
    else:
        env["BF_STAGES"] = int(knob[-1])
    f = _fresh(monkeypatch, env)
    try:
        rng = np.random.default_rng(4800 + len(knob) + int(knob[-1]) if knob != "blocked" else 4899)
        ts = randgen.random_topologies(rng, 30, 20, 100, max_deg=5, fill=0.3)
        slots = f.put_topologies(ts)
        L, state, _ = randgen.random_state(rng, ts, slots, 2 * sms * 16 * 3 + 7, ALL)
        _compare(f, ts, slots, L, state, expansion=True)
        st = f.stats()
        assert st["last_kernel"] == 0 and st["last_block"] == 512, st
        if knob != "blocked":
            assert st["last_stages"] == int(knob[-1]), st
    finally:
        f.close()


def test_general_knobs_follow_on_one_ctx(monkeypatch):
    """the shape knobs are read on every pass: changing one on a ctx that has already planned this batch re-plans it"""
    f = _fresh(monkeypatch, {"BF_KERNEL": "general"})
    try:
        rng = np.random.default_rng(4900)
        ts = randgen.random_topologies(rng, 30, 20, 64, max_deg=4, fill=0.5)
        slots = f.put_topologies(ts)
        L, state, _ = randgen.random_state(rng, ts, slots, 3000, ALL)
        for env, key, want in ((("BF_STAGES", 1), "last_stages", 1), (("BF_STAGES", 3), "last_stages", 3),
                               (("BF_STAGES", 2), "last_stages", 2), (("BF_WARPS", 8), "last_block", 256),
                               (("BF_WARPS", 24), "last_block", 768), (("BF_WARPS", 16), "last_block", 512)):
            monkeypatch.setenv(*map(str, env))
            _compare(f, ts, slots, L, state)
            assert f.stats()[key] == want, (env, f.stats())
    finally:
        f.close()
