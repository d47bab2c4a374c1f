"""Compact results (bf_eval_compact / bf_resident_tick_compact): the per-run head words and the 16-bit (step | kind << 10) event
list must be exactly what the oracle's mask records say, in run-major / step-ascending order; in changed-only mode exactly the
runs whose record differs from the previous tick's are listed, and replaying the ticks rebuilds every run's row."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier, synth
from bobrapet_b200.records import make_layout, pack_state
from oracle import packed as PK
from tests import randgen

pytestmark = pytest.mark.gpu

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT


@pytest.fixture(scope="module")
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _check(fr, ts, slots, L, state, flags=0, cap=None, want=None, wcounts=None):
    if want is None:
        want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, flags, 0, threads=8)
    whead, wev, wlisted = PK.compact_events(L, want)
    cap = len(wev) + 16 if cap is None else cap
    head, events, n_events, counts = fr.eval_compact(L, state, cap, flags=flags)
    assert n_events == len(wev) and counts == wcounts
    assert np.array_equal(head, whead)
    assert np.array_equal(events, wev[:cap])
    # pinned caller buffers (what the batcher uses)
    n = state.shape[0]
    p_head = fr.alloc_pinned(max(n, 1) * 4).view(np.uint32)
    p_ev = fr.alloc_pinned(max(cap, 1) * 2).view(np.uint16)
    p_head[:] = 0xABABABAB
    try:
        head, events, n_events, counts = fr.eval_compact(L, state, cap, flags=flags, head=p_head, events=p_ev)
        assert n_events == len(wev) and counts == wcounts and np.array_equal(head, whead) and np.array_equal(events, wev[:cap])
    finally:
        fr.free_pinned(p_head.view(np.uint8))
        fr.free_pinned(p_ev.view(np.uint8))
    return n_events


@pytest.mark.parametrize("cfg,n,S,fields", [(3, 5003, 256, 0), (4, 4001, 256, ALL), (2, 3000, 64, A.F_ALL_OUT), (5, 700, 1024, ALL),
                                            (3, 600, 33, A.F_OUT_FAIL), (3, 1, 256, 0), (3, 513, 100, A.F_OUT_SKIP_DEP)])
def test_compact_matches_oracle_masks(fr, cfg, n, S, fields):
    ts = synth.topologies(cfg, 0, n, S)
    slots = fr.put_topologies(ts)
    pt = PK.PackedTopologies(ts, slots)
    child = pt.max_child_nibbles()
    f = fields | (A.F_COND | A.F_DECISION if cfg in (4, 5) else 0) | (A.F_CHILD if child else 0)
    L = make_layout(S, child, f)
    cf = fr.child_first(int(slots[0])) if child else None
    state = synth.state(cfg, 0, n, L, slots, ts, cf)
    assert _check(fr, ts, slots, L, state) > 0 or n < 10


@pytest.mark.parametrize("seed", range(4))
def test_compact_adversarial_and_fixpoint(fr, seed):
    rng = np.random.default_rng(900 + seed)
    ts = randgen.random_topologies(rng, 40, 1, [60, 300, 1024, 130][seed], max_deg=[5, 4, 5, 2][seed], fill=[0, 0.9, 0, 0.9][seed])
    slots = fr.put_topologies(ts)
    L, state, _ = randgen.random_state(rng, ts, slots, 3001, ALL, phase_mix=("any" if seed % 2 else "progress"))
    _check(fr, ts, slots, L, state)
    _check(fr, ts, slots, L, state, flags=A.EVAL_FIXPOINT)


def test_compact_capacity_smaller_than_the_list_and_dead_slot(fr):
    ts = synth.topologies(3, 0, 2000, 256)
    slots = fr.put_topologies(ts)
    L = make_layout(256, 0, 0)
    state = synth.state(3, 0, 2000, L, slots, ts)
    want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, 0, 0, threads=8)
    # run 7 gets a dead topology slot: the kernels mark it (summary all-ones, empty record, nothing counted)
    hdr = want[7, 0:16].view("<u4")
    wcounts = dict(wcounts, ready=wcounts["ready"] - int(hdr[1]), skip=wcounts["skip"] - int(hdr[2]), evals=wcounts["evals"] - 256)
    want[7, :] = 0
    want[7, 0:4] = 0xFF
    state[7, 0:4] = np.frombuffer(np.uint32(0x7FFFFFF0).tobytes(), np.uint8)
    n = _check(fr, ts, slots, L, state, want=want, wcounts=wcounts)
    assert n > 200
    _check(fr, ts, slots, L, state, cap=100, want=want, wcounts=wcounts)  # only the first `cap` events are written, n_events still says how many
    _check(fr, ts, slots, L, state, cap=0, want=want, wcounts=wcounts)
    _check(fr, ts, slots, L, state, want=want, wcounts=wcounts)          # and a larger list after a tiny one (the first D2H slice is a guess)


def test_resident_tick_compact_and_changed_only(fr):
    n, S = 6007, 256
    ts = synth.topologies(4, 0, n, S)
    slots = fr.put_topologies(ts)
    L = make_layout(S, 0, ALL)
    state = synth.state(4, 0, n, L, slots, ts)
    pt = PK.PackedTopologies(ts, slots)
    h = fr.resident_create(L, n)
    try:
        fr.resident_upload(h, 0, state)
        rng = np.random.default_rng(3)
        prev = None
        rows = {}      # the batcher's cache: run -> (head low bits, events), rebuilt from changed-only ticks
        for tick in range(6):
            k = [500, 40, 0, 3000, 1, 500][tick]
            flat = rng.choice(n * S, size=k, replace=False)
            d = np.zeros(k, dtype=fr.DELTA_DTYPE)
            d["run"], d["index"], d["field"] = flat // S, flat % S, A.DELTA_PHASE
            d["code"] = rng.choice([0, 2, 3, 3, 4, 13], size=k)
            changed_only = tick >= 2
            head, events, n_events, counts, n_listed = fr.resident_tick_compact(
                h, n, d, 200000, flags=(A.EVAL_CHANGED_ONLY if changed_only else 0))
            cur = fr.resident_download(h, 0, n, L.state_stride)
            want, wcounts = PK.evaluate(pt, L, cur, 0, 0, threads=8)
            # the first changed-only tick follows full ticks whose records are still on the device: it may already be sparse
            whead, wev, wlisted = PK.compact_events(L, want, prev if changed_only else None)
            assert counts == wcounts and n_events == len(wev) and n_listed == wlisted
            assert np.array_equal(head, whead) and np.array_equal(events, wev)
            if changed_only and k <= 40:
                assert n_listed <= max(4 * k, 1) and n_listed < n // 10      # O(changes), not O(runs)
            # replay into the cache and compare with the full compact form of this tick
            pos = 0
            for r in np.nonzero(head & A.HEAD_LISTED)[0]:
                c = int(head[r]) >> A.HEAD_COUNT_SHIFT
                rows[int(r)] = (int(head[r]) & A.HEAD_SUMMARY_MASK, events[pos:pos + c].copy())
                pos += c
            assert pos == n_events
            fhead, fev, _ = PK.compact_events(L, want)
            pos = 0
            for r in range(n):
                c = int(fhead[r]) >> A.HEAD_COUNT_SHIFT
                assert rows[r][0] == int(fhead[r]) & A.HEAD_SUMMARY_MASK and np.array_equal(rows[r][1], fev[pos:pos + c]), (tick, r)
                pos += c
            prev = want
        # new full records for some runs: the next changed-only tick lists every run again
        fr.resident_upload(h, 10, cur[10:20])
        head, events, n_events, counts, n_listed = fr.resident_tick_compact(h, n, np.zeros(0, dtype=fr.DELTA_DTYPE), 200000,
                                                                             flags=A.EVAL_CHANGED_ONLY)
        assert n_listed == n
    finally:
        fr.resident_destroy(h)


def test_fused_heads_ticks_of_different_sizes():
    """On a ctx without parallel steps a compact tick's pass is the packed-lanes kernel alone and leaves the head words and the
    per-512-run event totals itself (no heads kernel; two totals buffers used in turn, each left zeroed by the other tick's emit
    kernel).  Ticks of very different sizes, changed-only ticks (which keep the heads kernel) and dead slots in between must not
    leave anything behind in either buffer."""
    f = Frontier(0)
    try:
        rng = np.random.default_rng(77)
        batches = []
        for n, S, fields in ((40000, 256, 0), (700, 256, ALL), (9000, 64, A.F_ALL_OUT)):
            ts = synth.topologies(4 if fields == ALL else 3, n, n, S)
            slots = f.put_topologies(ts)
            L = make_layout(S, 0, fields)
            state = synth.state(4 if fields == ALL else 3, n, n, L, slots, ts)
            live5 = state[5, 0:4].copy()
            if n == 700:
                state[5, 0:4] = np.frombuffer(np.uint32(0x7FFFFFF0).tobytes(), np.uint8)   # a dead topology slot
            h = f.resident_create(L, n)
            f.resident_upload(h, 0, state)
            batches.append((n, S, L, PK.PackedTopologies(ts, slots), h, None, live5))
        order = [0, 1, 0, 2, 1, 1, 0, 2, 2, 0]
        for step, b in enumerate(order):
            n, S, L, pt, h, prev, live5 = batches[b]
            k = int(rng.integers(0, 300))
            flat = rng.choice(n * S, size=k, replace=False)
            d = np.zeros(k, dtype=f.DELTA_DTYPE)
            d["run"], d["index"], d["field"] = flat // S, flat % S, A.DELTA_PHASE
            d["code"] = rng.choice([0, 2, 3, 3, 4, 13], size=k)
            if b == 1:
                d = d[d["run"] != 5]
            changed_only = step % 3 == 2 and prev is not None
            p_head = f.alloc_pinned(n * 4).view(np.uint32)
            p_ev = f.alloc_pinned(400000 * 2).view(np.uint16)
            try:
                head, events, n_events, counts, n_listed = f.resident_tick_compact(
                    h, n, d, 400000, flags=(A.EVAL_CHANGED_ONLY if changed_only else 0), head=p_head, events=p_ev)
                cur = f.resident_download(h, 0, n, L.state_stride)
                if b == 1:
                    cur[5, 0:4] = live5      # the oracle takes live slots only; the dead run's record is patched below
                want, wcounts = PK.evaluate(pt, L, cur, 0, 0, threads=8)
                if b == 1:   # the dead run: marked, empty, not counted (as in test_compact_capacity_smaller_than_the_list_and_dead_slot)
                    hdr = want[5, 0:16].view("<u4")
                    wcounts = dict(wcounts, ready=wcounts["ready"] - int(hdr[1]), skip=wcounts["skip"] - int(hdr[2]), evals=wcounts["evals"] - S)
                    want[5, :] = 0
                    want[5, 0:4] = 0xFF
                whead, wev, wlisted = PK.compact_events(L, want, prev if changed_only else None)
                assert counts == wcounts and n_events == len(wev) and n_listed == wlisted, (step, b, n_events, len(wev), n_listed, wlisted)
                assert np.array_equal(head, whead) and np.array_equal(events, wev), (step, b)
                st = f.stats()
                assert st["last_kernel"] == 1, st
            finally:
                f.free_pinned(p_head.view(np.uint8))
                f.free_pinned(p_ev.view(np.uint8))
            batches[b] = (n, S, L, pt, h, want, live5)
    finally:
        f.close()


def _no_deps_topology(S):
    from bobrapet_b200.frontier import TopologySet
    return TopologySet([S], [0], np.zeros(S + 1, np.uint32), np.zeros(0, np.uint16), np.zeros(S, np.uint8))


@pytest.mark.parametrize("pattern", ["all-direct", "alternating"])
def test_compact_direct_and_staged_blocks(fr, pattern):
    """a 512-run block whose slice holds more than 8192 events writes it directly instead of staging it in shared memory:
    S = 1024 steps without needs, all ready, in every block ("all-direct"), or in every other block with 1-2 events per run
    between ("alternating": staged slices at odd and even bases).  Caps inside a direct slice and inside a staged slice that
    starts at an odd base: only the first `cap` events are written, n_events still counts them all."""
    S, n, CB = 1024, 4096, 512
    slots = fr.put_topologies(_no_deps_topology(S))
    ts = _no_deps_topology(S)
    L = make_layout(S, 0, 0)
    phase = np.zeros((n, S), np.uint8)
    heavy = np.ones(n, bool) if pattern == "all-direct" else (np.arange(n) // CB) % 2 == 0
    rng = np.random.default_rng(31)
    for r in np.nonzero(~heavy)[0]:
        phase[r, :] = 3                                      # Succeeded: no event
        phase[r, rng.choice(S, size=(2 if r == CB else 1), replace=False)] = 0   # one ready step (two in run 512: an odd slice)
    state = pack_state(L, np.full(n, slots[0], np.uint32), np.zeros(n, np.uint8), phase)
    want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, 0, 0, threads=8)
    whead, wev, _ = PK.compact_events(L, want)
    per_block = (whead >> A.HEAD_COUNT_SHIFT).reshape(-1, CB).sum(axis=1).astype(np.int64)
    base = np.concatenate(([0], np.cumsum(per_block)))
    direct = per_block > 8192
    assert direct.all() if pattern == "all-direct" else (direct == heavy[::CB]).all()
    assert _check(fr, ts, slots, L, state, want=want, wcounts=wcounts) == len(wev)
    caps = [int(base[np.nonzero(direct)[0][-1]]) + 777]                        # inside a direct slice
    if pattern == "alternating":
        odd = [b for b in np.nonzero(~direct)[0] if base[b] % 2 == 1]
        assert odd, base
        caps += [int(base[odd[0]]) + 1, int(base[odd[0]]) + 2]                 # inside a staged slice at an odd base
        caps += [int(base[1]) + 1]                                               # and at an even one
    for cap in caps:
        _check(fr, ts, slots, L, state, cap=cap, want=want, wcounts=wcounts)


@pytest.mark.parametrize("max_iter", [1, 2, 3, "S+5"])
def test_resident_tick_compact_iteration_cap(fr, max_iter):
    """max_iterations reaches the fixpoint of a compact resident tick"""
    rng = np.random.default_rng(950)
    ts = randgen.random_topologies(rng, 40, 1, 200, max_deg=3, fill=0.5)
    slots = fr.put_topologies(ts)
    n = 3001
    L, state, _ = randgen.random_state(rng, ts, slots, n, ALL, phase_mix="progress")
    k = int(ts.S.max()) + 5 if max_iter == "S+5" else max_iter
    h = fr.resident_create(L, n)
    try:
        fr.resident_upload(h, 0, state)
        head, events, n_events, counts, _ = fr.resident_tick_compact(h, n, np.zeros(0, dtype=fr.DELTA_DTYPE), 2_000_000,
                                                                      flags=A.EVAL_FIXPOINT, max_iterations=k)
        want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, A.EVAL_FIXPOINT, k, threads=8)
        whead, wev, _ = PK.compact_events(L, want)
        assert counts == wcounts and n_events == len(wev)
        assert np.array_equal(head, whead) and np.array_equal(events, wev)
    finally:
        fr.resident_destroy(h)
