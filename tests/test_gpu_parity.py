"""GPU parity: the CUDA path (through the C ABI, bf_eval) vs the packed oracle, bit for bit.

Every comparison is on whole result records (header + every mask + phase_out), so a single
wrong bit anywhere fails.  Integer/bit work: the bar is exact equality.
"""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier, synth
from bobrapet_b200.records import make_layout, unpack_result
from oracle import packed as PK
from tests import randgen

pytestmark = pytest.mark.gpu

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT


@pytest.fixture(scope="module")
def fr():
    f = Frontier(0)
    yield f
    f.close()


@pytest.fixture(params=["pack-ell", "pack-ell16", "pack-csr", "general-ell", "general-ell16", "general-csr"])
def kernel(request, monkeypatch):
    """pack = the default: packed lanes (a group of R runs per warp trip, frontier_pack.cu; runs whose topology has
    parallel steps are deferred to the general kernel), general = the one-run-per-warp kernel forced for every run
    (BF_KERNEL=general).  ell / csr = the row format of the topology records: fixed-width rows where they qualify
    (the default: byte entries up to 256 steps, u16 entries above), fixed-width rows with u16 entries only
    (BF_TOPO_FORMAT=ell16) or CSR only (BF_TOPO_FORMAT=csr, read at upload).  All must equal the oracle."""
    k, fmt = request.param.split("-")
    if k == "general":
        monkeypatch.setenv("BF_KERNEL", "general")
    else:
        monkeypatch.delenv("BF_KERNEL", raising=False)
    if fmt in ("csr", "ell16"):
        monkeypatch.setenv("BF_TOPO_FORMAT", fmt)
    else:
        monkeypatch.delenv("BF_TOPO_FORMAT", raising=False)
    return k


def _compare(fr, ts, slots, L, state, flags=0, max_iter=0, expansion=False, validate=True, cap=None):
    """cap: the expansion capacity (default: room for every tuple); the kernel must keep the oracle's first `cap` tuples
    and still report the full total.  validate=False for records with reserved codes, which the validation rejects."""
    pt = PK.PackedTopologies(ts, slots)
    want, wcounts = PK.evaluate(pt, L, state, flags, max_iter, threads=8)
    vflag = A.EVAL_VALIDATE if validate else 0
    if expansion:
        if cap is None:
            cap = int(wcounts["expansion"]) + 8
        got, gcounts, gexp = fr.eval(L, state, flags=flags | A.EVAL_EXPANSION | vflag, max_iterations=max_iter,
                                     expansion_cap=cap)
        wexp, n = PK.expand(pt, L, state, want, cap)
        assert n == wcounts["expansion"] == gcounts["expansion"]
        assert len(gexp) == len(wexp) == min(cap, n)
        assert np.array_equal(gexp, wexp), "expansion tuples differ"
    else:
        got, gcounts = fr.eval(L, state, flags=flags | vflag, max_iterations=max_iter)
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        r = int(bad[0])
        S = int(ts.S.max())
        g, w = unpack_result(L, got[r:r + 1], S), unpack_result(L, want[r:r + 1], S)
        diff = {k: (g[k][0], w[k][0]) for k in g if not np.array_equal(g[k], w[k])}
        raise AssertionError("%d/%d runs differ; first run %d: %s" % (len(bad), len(got), r, {k: (np.nonzero(np.atleast_1d(a != b))[0][:8], a, b) for k, (a, b) in diff.items()}))
    assert gcounts == wcounts
    return got


def test_child_first_rule_matches_library(fr):
    rng = np.random.default_rng(5)
    ts = randgen.random_topologies(rng, 40, 1, 300)
    slots = fr.put_topologies(ts)
    cfs, _ = randgen.child_layout(ts)
    for t in range(ts.count):
        assert np.array_equal(fr.child_first(int(slots[t])), cfs[t])


@pytest.mark.parametrize("cfg,n,S", [(2, 3000, 64), (3, 3000, 256), (4, 3000, 256), (5, 600, 1024),
                                     (3, 500, 1), (3, 500, 2), (3, 500, 31), (3, 500, 32), (3, 500, 33),
                                     (3, 500, 100), (4, 500, 200), (3, 300, 1000), (4, 300, 1023)])
def test_synthetic_configs(fr, kernel, cfg, n, S):
    ts = synth.topologies(cfg, 0, n, S)
    slots = fr.put_topologies(ts)
    pt = PK.PackedTopologies(ts, slots)
    fields = ALL if cfg in (4, 5) else A.F_ALL_OUT
    child = pt.max_child_nibbles()
    L = make_layout(S, child, fields | (A.F_CHILD if child else 0))
    cf = fr.child_first(int(slots[0])) if child else None
    state = synth.state(cfg, 0, n, L, slots, ts, cf)
    got = _compare(fr, ts, slots, L, state, expansion=(cfg == 5))
    out = unpack_result(L, got, S)
    assert out["ready"].any() or S < 3


# "dirty": records no producer should write but the kernels must read exactly as the oracle does — the reserved phase /
# child code 15 (read as 0) and random codes past each run's S (not read); EVAL_VALIDATE would reject them
EDGES = {"clean": {}, "dirty": {"reserved": 0.05, "padding": True}}


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("mode", ["single", "fixpoint"])
def test_random_adversarial(fr, seed, mode):
    _random_adversarial(fr, seed, mode, "clean")


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("mode", ["single", "fixpoint"])
def test_random_adversarial_dirty(fr, seed, mode):
    _random_adversarial(fr, seed, mode, "dirty")


def _random_adversarial(fr, seed, mode, edges):
    rng = np.random.default_rng(1000 + seed)
    smax = [40, 257, 1024, 96, 600, 33][seed]
    deg, fill = [(5, 0.0), (4, 0.9), (5, 0.0), (2, 0.9), (4, 0.85), (5, 0.0)][seed]
    ts = randgen.random_topologies(rng, 60, 1, smax, max_deg=deg, fill=fill)
    slots = fr.put_topologies(ts)
    L, state, _ = randgen.random_state(rng, ts, slots, 4000, ALL, phase_mix=("any" if seed % 2 else "progress"), **EDGES[edges])
    _compare(fr, ts, slots, L, state, flags=(A.EVAL_FIXPOINT if mode == "fixpoint" else 0), expansion=True,
             validate=(edges == "clean"))


@pytest.mark.parametrize("max_iter", [1, 2, 3, "S+5"])
def test_fixpoint_iteration_cap(fr, max_iter):
    """max_iterations caps the device fixpoint (the loop stops after k iterations, its launch effects kept)"""
    rng = np.random.default_rng(1500)
    ts = randgen.random_topologies(rng, 60, 1, 200, max_deg=3, fill=0.5)
    slots = fr.put_topologies(ts)
    L, state, _ = randgen.random_state(rng, ts, slots, 3000, ALL, phase_mix="progress")
    k = int(ts.S.max()) + 5 if max_iter == "S+5" else max_iter
    got = _compare(fr, ts, slots, L, state, flags=A.EVAL_FIXPOINT, max_iter=k, expansion=True)
    iters = np.ascontiguousarray(got[:, 0:4]).view("<u4")[:, 0] >> A.SUM_ITER_SHIFT
    assert (iters <= k).all()
    if k <= 3:
        assert (iters == k).any()   # some run was still progressing when the cap stopped it


@pytest.mark.parametrize("which", ["zero", "one", "inside", "total-1", "total"])
def test_expansion_cap(fr, which):
    """a cap below the tuple count keeps the oracle's first `cap` tuples (run-major, step / branch order) and still
    reports the full total in counts.expansion"""
    rng = np.random.default_rng(1600)
    ts = randgen.random_topologies(rng, 40, 5, 120, max_deg=3, fill=0.5, branch_choices=(3, 9, 33, 40))
    slots = fr.put_topologies(ts)
    L, state, _ = randgen.random_state(rng, ts, slots, 2000, ALL, phase_mix="progress")
    pt = PK.PackedTopologies(ts, slots)
    want, wc = PK.evaluate(pt, L, state, threads=8)
    total = int(wc["expansion"])
    assert total > 100
    hdr = np.ascontiguousarray(want[:, 0:16]).view("<u4").reshape(-1, 4)
    first = int(np.nonzero(hdr[:, 3] > 2)[0][0])                    # a run with a branch list of several tuples
    inside = int(hdr[:first, 3].sum()) + 1                          # the cap ends inside that run's list
    cap = {"zero": 0, "one": 1, "inside": inside, "total-1": total - 1, "total": total}[which]
    _compare(fr, ts, slots, L, state, expansion=True, cap=cap)


@pytest.mark.parametrize("seed", range(8))
def test_random_adversarial_no_parallel(fr, kernel, seed):
    """all phase codes / groups / flags / FAIL codes, no parallel steps: the packed-lanes kernel's domain"""
    _random_adversarial_no_parallel(fr, kernel, seed, "clean")


@pytest.mark.parametrize("seed", range(8))
def test_random_adversarial_no_parallel_dirty(fr, kernel, seed):
    """the same batches with reserved codes and padding (EDGES)"""
    _random_adversarial_no_parallel(fr, kernel, seed, "dirty")


def _random_adversarial_no_parallel(fr, kernel, seed, edges):
    rng = np.random.default_rng(5000 + seed)
    smax = [40, 257, 1024, 96, 600, 33, 8, 130][seed]
    # seeds 0-2: sparse rows up to 5 needs (CSR, long rows); 3-5: dense rows of <= 4 (fixed-width 4); 6-7: dense <= 2
    deg, fill = [(5, 0.0), (5, 0.0), (5, 0.0), (4, 0.9), (4, 0.85), (4, 0.9), (2, 0.9), (2, 0.8)][seed]
    ts = randgen.random_topologies(rng, 60, 1, smax, max_deg=deg, parallel=False, fill=fill)
    slots = fr.put_topologies(ts)
    n = [4000, 4001, 999, 4003, 1500, 4005, 4006, 4007][seed]
    L, state, _ = randgen.random_state(rng, ts, slots, n, ALL if seed % 3 else (A.F_COND | A.F_ALL_OUT),
                                       phase_mix=("any" if seed % 2 else "progress"), **EDGES[edges])
    _compare(fr, ts, slots, L, state, validate=(edges == "clean"))
    st = fr.stats()
    # the ctx also holds topologies with parallel steps (earlier tests): packed lanes + deferred general; layouts wider
    # than 16 words (S > 512) always take the general kernel
    assert st["last_kernel"] == (2 if kernel == "pack" and L.words <= 16 else 0), st


def test_minimal_layout_outputs_only_ready_skip(fr, kernel):
    rng = np.random.default_rng(77)
    ts = randgen.random_topologies(rng, 30, 5, 200, parallel=False)
    slots = fr.put_topologies(ts)
    L, state, _ = randgen.random_state(rng, ts, slots, 2000, 0)
    _compare(fr, ts, slots, L, state)


def test_shared_topology_mode(fr, kernel):
    """D << N: many runs per topology (records come from L2 instead of HBM)."""
    ts = synth.topologies(3, 0, 8, 256)
    slots = fr.put_topologies(ts)
    n = 5000
    L = make_layout(256, 0, A.F_ALL_OUT)
    big = synth.topologies(3, 0, n, 256)  # only for flags-shaped state generation
    state = synth.state(3, 0, n, L, np.asarray(slots)[np.arange(n) % 8], big)
    # state was generated against `big`'s flags; for cfg 3 flags only carry allowFailure, which state ignores
    _compare(fr, ts, slots, L, state)


def test_invalid_slot_yields_marked_empty_result(fr):
    ts = synth.topologies(3, 0, 4, 64)
    slots = fr.put_topologies(ts)
    L = make_layout(64, 0, 0)
    state = synth.state(3, 0, 4, L, slots, ts)
    state[2, 0:4] = np.frombuffer(np.uint32(0x7FFFFFF0).tobytes(), np.uint8)
    with pytest.raises(A.FrontierError):
        fr.eval(L, state, flags=A.EVAL_VALIDATE)
    got, _ = fr.eval(L, state)   # without validation the kernel marks the run and carries on
    hdr = got[:, 0:4].view("<u4")[:, 0]
    assert hdr[2] == 0xFFFFFFFF and not got[2, 16:].any()
    assert hdr[0] != 0xFFFFFFFF


def test_topology_rejections(fr):
    from bobrapet_b200.frontier import TopologySet
    cyc = TopologySet([2], [2], [0, 1, 2], [1, 0], [0, 0])
    with pytest.raises(A.FrontierError) as e:
        fr.put_topologies(cyc)
    assert e.value.status == A.BF_ETOPO and "cycle" in str(e.value)          # dag_test.go:321
    selfloop = TopologySet([1], [1], [0, 1], [0], [0])
    with pytest.raises(A.FrontierError):
        fr.put_topologies(selfloop)
    unknown = TopologySet([2], [1], [0, 0, 1], [7], [0, 0])
    with pytest.raises(A.FrontierError) as e:
        fr.put_topologies(unknown)
    assert "unknown step dependency" in str(e.value)                          # dag_test.go:206


@pytest.mark.parametrize("fmt", ["ell", "ell16", "csr"])
def test_packed_lanes_only_context(monkeypatch, fmt):
    """a ctx whose topologies have no parallel steps runs the packed-lanes kernel alone (4 runs per trip at S=256, 16 at
    S=64: the ring is planned from the largest record a run of the batch's layout can stage, not the ctx-wide largest)"""
    monkeypatch.delenv("BF_KERNEL", raising=False)
    if fmt in ("csr", "ell16"):
        monkeypatch.setenv("BF_TOPO_FORMAT", fmt)
    else:
        monkeypatch.delenv("BF_TOPO_FORMAT", raising=False)
    f = Frontier(0)
    try:
        ts = synth.topologies(4, 0, 3001, 256)
        slots = f.put_topologies(ts)
        L = make_layout(256, 0, ALL)
        state = synth.state(4, 0, 3001, L, slots, ts)
        _compare(f, ts, slots, L, state)
        st = f.stats()
        assert st["last_kernel"] == 1 and st["last_runs_per_trip"] == 4, st
        _, nbytes = f.topology_record(int(slots[0]))
        # 32 + 256 x 4 + 9 x 32 (byte entries + NODEP plane) | 32 + 528 + 2048 + 256 (CSR: a topology of exactly 8 words never
        # takes u16 fixed-width rows, its PAD index 256 has no status byte in the packed kernel; u16 rows: test_row_formats)
        assert nbytes == {"ell": 1344, "ell16": 2864, "csr": 2864}[fmt], nbytes
        ts2 = synth.topologies(2, 0, 777, 64)
        s2 = f.put_topologies(ts2)
        L2 = make_layout(64, 0, A.F_ALL_OUT)
        _compare(f, ts2, s2, L2, synth.state(2, 0, 777, L2, s2, ts2))
        assert f.stats()["last_runs_per_trip"] == 16, f.stats()
        # runs of mixed step counts and row formats inside one group (S = 5 .. 250, some rows longer than 4)
        rng = np.random.default_rng(4242)
        ts3 = randgen.random_topologies(rng, 25, 5, 250, parallel=False)
        ts3b = randgen.random_topologies(rng, 25, 5, 250, max_deg=4, parallel=False, fill=0.9)
        s3b = f.put_topologies(ts3b)
        L3b, state3b, _ = randgen.random_state(rng, ts3b, s3b, 3001, ALL)
        _compare(f, ts3b, s3b, L3b, state3b)
        s3 = f.put_topologies(ts3)
        L3, state3, _ = randgen.random_state(rng, ts3, s3, 5003, ALL)
        _compare(f, ts3, s3, L3, state3)
        assert f.stats()["last_kernel"] == 1, f.stats()
    finally:
        f.close()


@pytest.mark.parametrize("cfg,n", [(3, 70001), (4, 66003), (2, 300000)])
def test_long_ring_sequences(cfg, n):
    """enough groups per CTA that every warp wraps its prefetch batches and the slot ring many times"""
    f = Frontier(0)
    try:
        S = 64 if cfg == 2 else 256
        synth.set_threads(16)
        ts = synth.topologies(cfg, 0, n, S)
        slots = f.put_topologies(ts)
        L = make_layout(S, 0, ALL if cfg == 4 else 0)
        state = synth.state(cfg, 0, n, L, slots, ts)
        want, wc = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=16)
        got, gc = f.eval(L, state)
        assert f.stats()["last_kernel"] == 1
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert bad.size == 0 and gc == wc, (bad[:10], bad.size, gc, wc)
    finally:
        f.close()


def test_group_tail_and_tiny_batches():
    """batch sizes around the group size R and the CTA count: partial last group, fewer groups than warps / CTAs"""
    f = Frontier(0)
    try:
        ts = synth.topologies(3, 0, 700, 256)
        slots = f.put_topologies(ts)
        L = make_layout(256, 0, A.F_ALL_OUT)
        sms = f.stats()["sm_count"]   # R = 4 runs per group: one group per CTA of the persistent grid around these sizes
        for n in (1, 2, 3, 4, 5, 63, 64, 65, (sms - 1) * 4 + 1, sms * 4, sms * 4 + 3, 147 * 4 + 1, 148 * 4, 148 * 4 + 3, 700):
            state = synth.state(3, 0, n, L, slots[:n], synth.topologies(3, 0, n, 256))
            want, wc = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=4)
            got, gc = f.eval(L, state)
            assert np.array_equal(got, want) and gc == wc, n
            assert f.stats()["last_kernel"] == 1
    finally:
        f.close()


def test_drop_and_reuse_slot(fr):
    ts = synth.topologies(3, 100, 3, 64)
    slots = fr.put_topologies(ts)
    fr.drop_topology(int(slots[1]))
    ts2 = synth.topologies(3, 200, 1, 64)
    s2 = fr.put_topologies(ts2)
    assert int(s2[0]) == int(slots[1])
    L = make_layout(64, 0, A.F_ALL_OUT)
    state = synth.state(3, 200, 1, L, s2, ts2)
    pt = PK.PackedTopologies(ts2, s2)
    want, _ = PK.evaluate(pt, L, state)
    got, _ = fr.eval(L, state)
    assert np.array_equal(got, want)


def test_arena_compaction_keeps_live_topologies():
    """one put + one drop per Story generation must not grow the arena without bound: when dropped records outweigh
    the live ones the arena is re-packed, slots keep their ids and the surviving topologies still evaluate exactly"""
    f = Frontier(0)
    try:
        n = 3000
        ts = synth.topologies(3, 0, n, 256)
        slots = f.put_topologies(ts)
        L = make_layout(256, 0, A.F_ALL_OUT)
        state = synth.state(3, 0, n, L, slots, ts)
        want, wc = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=4)
        used0 = f.stats()["arena_used_bytes"]
        for gen in range(6):   # generations of other stories come and go
            ts2 = synth.topologies(3, 1000000 + gen * n, n, 256)
            s2 = f.put_topologies(ts2)
            for s in s2:
                f.drop_topology(int(s))
        st = f.stats()
        assert st["arena_compactions"] >= 1 and st["n_topologies"] == n
        assert st["arena_used_bytes"] <= 3 * used0, st     # bounded: live records + at most the uncompacted tail
        got, gc = f.eval(L, state)
        assert np.array_equal(got, want) and gc == wc
    finally:
        f.close()


@pytest.mark.parametrize("chunks", [0, 1, 5, 32])
def test_pipelined_host_eval_matches_oracle(fr, monkeypatch, chunks):
    """bf_eval cuts large batches into run chunks whose H2D / kernel / D2H overlap on three streams; any chunking
    (default, serial, uneven, maximum) must give the same records and the same global counts."""
    if chunks:
        monkeypatch.setenv("BF_E2E_CHUNKS", str(chunks))
    else:
        monkeypatch.delenv("BF_E2E_CHUNKS", raising=False)
    n = 20011
    ts = synth.topologies(4, 0, n, 256)
    slots = fr.put_topologies(ts)
    L = make_layout(256, 0, ALL)
    state = synth.state(4, 0, n, L, slots, ts)
    _compare(fr, ts, slots, L, state)
    total = n * (L.state_stride + L.result_stride)
    want_chunks = {0: max(2, (total + (11 << 18)) // (11 << 19)), 1: 1, 5: 5, 32: 32}[chunks]
    assert fr.stats()["last_eval_chunks"] == want_chunks


def test_pipelined_passes_counts_set(fr):
    """BF_EVAL_COUNTS_SET | BF_EVAL_PIPELINED: passes over DIFFERENT batches submitted back to back on one stream (each a
    programmatic dependent of the one before: its start overlaps the previous pass's tail) give the same records as plain
    passes, and every counts block holds exactly its own pass's totals although nobody zeroes it."""
    import torch
    dev = torch.device("cuda", 0)
    L = make_layout(256, 0, 0)
    sets = []
    for k in range(3):
        ts = synth.topologies(3, 1000 + 50_000 * k, 20_000 + 17 * k, 256)
        slots = fr.put_topologies(ts)
        st = synth.state(3, 1000 + 50_000 * k, ts.S.shape[0], L, slots, ts)
        want, wc = PK.evaluate(PK.PackedTopologies(ts, slots), L, st, threads=8)
        sets.append((st.shape[0], torch.from_numpy(st).to(dev), torch.zeros((st.shape[0], L.result_stride), dtype=torch.uint8, device=dev),
                     torch.full((4,), 123456789, dtype=torch.int64, device=dev), want, wc))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for rep in range(4):
            for n, d_state, d_result, d_counts, _, _ in sets:
                fr.eval_device(L, n, d_state.data_ptr(), d_result.data_ptr(), d_counts.data_ptr(), s.cuda_stream,
                               flags=A.EVAL_COUNTS_SET | A.EVAL_PIPELINED)
    torch.cuda.synchronize()
    for n, _, d_result, d_counts, want, wc in sets:
        assert np.array_equal(d_result.cpu().numpy(), want)
        assert d_counts.cpu().numpy().tolist() == [wc["ready"], wc["skip"], wc["expansion"], wc["evals"]]


@pytest.mark.parametrize("case", ["p10-1024", "p10-mixed", "byte4-256", "byte2-256", "u16x2-800", "csr-1024"])
def test_row_formats(case):
    """every device row format on purpose (device_record.h): the record size says which one a topology got; then the records
    go through both passes (single / fixpoint), the device validation (Kahn peel) and the redrive closure, all against the oracle.
    Byte / 10-bit rows have no PAD index: short rows repeat an entry, rows without needs are flagged NODEP."""
    from tests.test_redrive_closure import closure_packed
    from tests import packing as P
    smin, smax, deg, fill, par = {"p10-1024": (1024, 1024, 4, 0.9, True), "p10-mixed": (513, 1024, 3, 0.5, True),
                                  "byte4-256": (256, 256, 4, 0.9, False), "byte2-256": (225, 256, 2, 0.8, False),
                                  "u16x2-800": (700, 900, 2, 0.9, False), "csr-1024": (1000, 1024, 5, 0.3, True)}[case]
    rng = np.random.default_rng({"p10-1024": 11, "p10-mixed": 12, "byte4-256": 13, "byte2-256": 14, "u16x2-800": 15, "csr-1024": 16}[case])
    ts = randgen.random_topologies(rng, 12, smin, smax, max_deg=deg, parallel=par, fill=fill)
    f = Frontier(0)
    try:
        slots = f.put_topologies(ts)
        R_off = np.concatenate(([0], np.cumsum(ts.S.astype(np.int64) + 1)))
        E_off = np.concatenate(([0], np.cumsum(ts.E.astype(np.int64))))
        S_off = np.concatenate(([0], np.cumsum(ts.S.astype(np.int64))))
        for t in range(ts.count):
            S, Pn = int(ts.S[t]), int(ts.P[t])
            W = (S + 31) // 32
            rp = ts.row_ptr[R_off[t]:R_off[t] + S + 1].astype(np.int64)
            md = int((rp[1:] - rp[:-1]).max())
            _, nbytes = f.topology_record(int(slots[t]))
            br = ts.parallel["branches"][int(ts.P[:t].sum()):int(ts.P[:t].sum()) + Pn].astype(np.int64) if Pn else np.zeros(0, np.int64)
            par_bytes = 16 * Pn + 4 * int(((br + 31) // 32 + (br == 0)).sum())
            r16 = lambda x: (x + 15) // 16 * 16  # noqa: E731
            want = {"p10": 32 + 5 * 32 * W + r16(9 * 4 * W), "byte": 32 + (2 if md <= 2 else 4) * 32 * W + r16(9 * 4 * W),
                    "u16": 32 + 2 * (2 if md <= 2 else 4) * 32 * W + r16(8 * 4 * W),
                    "csr": 32 + r16(2 * (S + 1)) + r16(2 * int(ts.E[t]) + 8) + r16(8 * 4 * W)}
            kind = case.split("-")[0].rstrip("24").replace("u16x", "u16")
            if kind == "p10" and md <= 2:
                kind = "u16"      # rows of at most two needs keep u16 pairs (4 bytes per row already)
            assert nbytes == r16(want[kind] + par_bytes), (case, t, S, md, nbytes, {k: r16(v + par_bytes) for k, v in want.items()})
        for flags in (0, A.EVAL_FIXPOINT):
            L, state, _ = randgen.random_state(rng, ts, slots, 1500, ALL, phase_mix="progress")
            _compare(f, ts, slots, L, state, flags=flags, expansion=par)
        assert not (f.check_topologies(slots) & 1).any()          # the device Kahn peel reads the same rows
        for t in range(0, ts.count, 3):
            S = int(ts.S[t])
            ps = P.PackedStory(["s%d" % i for i in range(S)], {}, ts.row_ptr[R_off[t]:R_off[t] + S + 1],
                               ts.col_idx[E_off[t]:E_off[t + 1]], ts.step_flags[S_off[t]:S_off[t] + S])
            starts = rng.integers(0, S, size=8)
            got = f.closure([int(slots[t])] * 8, starts, 32)
            for k, st in enumerate(starts):
                assert np.array_equal(got[k, :(S + 31) // 32], closure_packed(ps, int(st))), (case, t, st)
    finally:
        f.close()


def test_counts_set_on_every_dispatch_shape(fr):
    """BF_EVAL_COUNTS_SET overwrites a counts block full of garbage whatever kernels the pass takes: packed lanes alone (the last
    CTA out publishes), packed lanes + deferred runs, the one-run-per-warp kernel, expansion lists, and an empty batch."""
    import torch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(99)
    cases = []
    f2 = Frontier(0)
    try:
        ts = synth.topologies(3, 0, 3000, 256)                                  # a ctx without parallel steps: packed lanes alone
        cases.append((f2, ts, f2.put_topologies(ts), False))
        tsp = randgen.random_topologies(rng, 40, 20, 250, max_deg=4, fill=0.8)  # fr holds parallel steps: two tiers at S <= 512
        cases.append((fr, tsp, fr.put_topologies(tsp), True))
        tsw = randgen.random_topologies(rng, 12, 600, 1000, max_deg=4, fill=0.8)  # S > 512: the one-run-per-warp kernel
        cases.append((fr, tsw, fr.put_topologies(tsw), True))
        for f, t, slots, exp in cases:
            L, state, _ = randgen.random_state(rng, t, slots, 2500, ALL, phase_mix="progress")
            pt = PK.PackedTopologies(t, slots)
            want, wc = PK.evaluate(pt, L, state, threads=8)
            d_state = torch.from_numpy(state).to(dev)
            d_result = torch.zeros((state.shape[0], L.result_stride), dtype=torch.uint8, device=dev)
            d_counts = torch.full((4,), 0x5A5A5A5A5A, dtype=torch.int64, device=dev)
            cur = torch.cuda.current_stream().cuda_stream
            for _ in range(2):
                f.eval_device(L, state.shape[0], d_state.data_ptr(), d_result.data_ptr(), d_counts.data_ptr(), cur, flags=A.EVAL_COUNTS_SET)
            torch.cuda.synchronize()
            assert np.array_equal(d_result.cpu().numpy(), want)
            assert d_counts.cpu().numpy().tolist() == [wc["ready"], wc["skip"], wc["expansion"], wc["evals"]], f.stats()
            if exp and wc["expansion"]:
                d_exp = torch.zeros((int(wc["expansion"]), 8), dtype=torch.uint8, device=dev)
                d_counts.fill_(77)
                f.eval_device(L, state.shape[0], d_state.data_ptr(), d_result.data_ptr(), d_counts.data_ptr(), cur,
                              flags=A.EVAL_COUNTS_SET | A.EVAL_EXPANSION, expansion_ptr=d_exp.data_ptr(), expansion_cap=int(wc["expansion"]))
                torch.cuda.synchronize()
                assert d_counts.cpu().numpy().tolist() == [wc["ready"], wc["skip"], wc["expansion"], wc["evals"]]
            d_counts.fill_(123)
            f.eval_device(L, 0, d_state.data_ptr(), d_result.data_ptr(), d_counts.data_ptr(), cur, flags=A.EVAL_COUNTS_SET)
            torch.cuda.synchronize()
            assert d_counts.cpu().numpy().tolist() == [0, 0, 0, 0]
    finally:
        f2.close()


@pytest.mark.parametrize("mode", ["single", "fixpoint"])
def test_parallel_steps_with_hundreds_of_branches(mode):
    """stage H classifies eight child nibbles per lane, a sub-warp per descriptor; a step with more than 256 branches does not
    fit a warp's 32 lanes x 8 children and takes the one-child-per-lane path.  Both, mixed in one batch, join + expansion."""
    rng = np.random.default_rng(2024)
    ts = randgen.random_topologies(rng, 30, 20, 60, max_deg=3, fill=0.5, branch_choices=(0, 5, 64, 128, 129, 255, 256, 257, 300, 600))
    f = Frontier(0)
    try:
        slots = f.put_topologies(ts)
        L, state, _ = randgen.random_state(rng, ts, slots, 1200, ALL, phase_mix="progress")
        _compare(f, ts, slots, L, state, flags=(A.EVAL_FIXPOINT if mode == "fixpoint" else 0), expansion=True)
    finally:
        f.close()
