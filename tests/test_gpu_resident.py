"""Resident batches (row f2: incremental state upload): the device copy after a stream of deltas must equal, byte for
byte, the records the host would have uploaded, and a pass over it must equal the oracle on those records."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import _unpack_planes, make_layout, pack_state
from oracle import packed as PK
from tests import randgen

pytestmark = pytest.mark.gpu
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT


def _decode(L, state):
    n, W = state.shape[0], L.words
    S = W * 32
    phase = _unpack_planes(state[:, L.off_phase:L.off_phase + 16 * W], W, 4, S)
    cond = _unpack_planes(state[:, L.off_cond:L.off_cond + 8 * W], W, 2, S)
    dec = _unpack_planes(state[:, L.off_decision:L.off_decision + 8 * W], W, 2, S)
    child = None
    if L.off_child != A.OFF_NONE:
        nb = (L.child_nibbles + 1) // 2
        raw = state[:, L.off_child:L.off_child + nb]
        child = np.empty((n, nb * 2), dtype=np.uint8)
        child[:, 0::2] = raw & 0xF
        child[:, 1::2] = raw >> 4
        child = child[:, :L.child_nibbles]
    slots = np.ascontiguousarray(state[:, 0:4]).view("<u4")[:, 0].copy()
    rflags = state[:, 4].copy()
    reg = np.ascontiguousarray(state[:, 8:16]).view("<u8")[:, 0].copy()
    return slots, rflags, phase, cond, dec, child, reg


def _want_with_dead(pt, L, state, dead, flags, max_iter):
    """oracle records of a batch whose runs in `dead` point at a dropped slot: the kernels mark such a run (summary all-ones,
    empty record) and count nothing for it; every other run is independent of them"""
    want = np.zeros((state.shape[0], L.result_stride), dtype=np.uint8)
    live = np.nonzero(~dead)[0]
    want[live], wcounts = PK.evaluate(pt, L, np.ascontiguousarray(state[live]), flags, max_iter, threads=8)
    want[dead, 0:4] = 0xFF
    return want, wcounts


@pytest.mark.parametrize("seed", range(3))
def test_deltas_equal_full_upload(seed):
    """random deltas of every field, including indices in [S, 32 * words) (accepted: the bound is the layout width) and
    DELTA_TOPO_SLOT re-pointing runs at a smaller topology (stale codes stay behind past its S), at one with parallel steps,
    or at a dropped slot (the run is marked dead); fixpoint ticks with and without an iteration cap"""
    rng = np.random.default_rng(8800 + seed)
    fr = Frontier(0)
    try:
        ts = randgen.random_topologies(rng, 30, 1, [70, 300, 1000][seed])
        tslots = fr.put_topologies(ts)
        dropped = int(fr.put_topologies(randgen.random_topologies(rng, 1, 1, 10))[0])
        fr.drop_topology(dropped)
        n = 1500
        L, state, topo = randgen.random_state(rng, ts, tslots, n, ALL, phase_mix="progress")
        pt = PK.PackedTopologies(ts, tslots)
        slots, rflags, phase, cond, dec, child, reg = _decode(L, state)
        # the decoded arrays re-pack to the very same records (so the host copy below is canonical)
        assert np.array_equal(pack_state(L, slots, rflags, phase, cond, dec, child, reg), state)
        h = fr.resident_create(L, n + 7)
        fr.resident_upload(h, 0, state)
        S_run = ts.S[topo].astype(np.int64)
        S_of = {int(tslots[t]): int(ts.S[t]) for t in range(ts.count)}
        with_par = [int(tslots[t]) for t in range(ts.count) if ts.P[t]]
        dead = np.zeros(n, dtype=bool)
        W32 = 32 * L.words
        for tick in range(6):
            k = int(rng.integers(1, 4000))
            recs = {}
            for _ in range(k):
                r = int(rng.integers(0, n))
                f = int(rng.choice([A.DELTA_PHASE] * 6 + [A.DELTA_COND, A.DELTA_DECISION, A.DELTA_CHILD, A.DELTA_RUN_FLAGS, A.DELTA_REGISTERED,
                                                          A.DELTA_TOPO_SLOT]))
                key = None
                if f in (A.DELTA_PHASE, A.DELTA_COND, A.DELTA_DECISION):
                    hi = W32 if (rng.random() < 0.2 and S_run[r] < W32) else S_run[r]   # past S: padding the kernels must not read
                    idx = int(rng.integers(0, hi))
                    code = int(rng.integers(0, 15 if f == A.DELTA_PHASE else 4))
                elif f == A.DELTA_CHILD:
                    if child is None:
                        continue
                    idx, code = int(rng.integers(0, L.child_nibbles)), int(rng.choice([0, 2, 3, 4, 13]))
                elif f == A.DELTA_RUN_FLAGS:
                    idx, code = 0, int(rng.choice([0, A.RF_FAIL_FAST, A.RF_FAIL_FAST | A.RF_REALTIME, A.RF_TOPOLOGY_TERMINATED]))
                elif f == A.DELTA_TOPO_SLOT:
                    kind = rng.integers(0, 8)
                    smaller = [s for s, S in S_of.items() if S < S_run[r]]
                    if kind == 0:
                        new = dropped
                    elif kind <= 3 and smaller:
                        new = int(rng.choice(smaller))
                    elif kind <= 5 and with_par:
                        new = int(rng.choice(with_par))
                    else:
                        new = int(rng.choice(tslots))
                    idx, code, key = new & 0xFFFF, new >> 16, 0     # one slot delta per run and tick
                else:
                    idx, code = int(rng.integers(0, 64)), int(rng.integers(0, 2))
                recs[(r, f, idx if key is None else key)] = (idx, code)   # the host coalesces: last value of the tick wins
            d = np.zeros(len(recs), dtype=Frontier.DELTA_DTYPE)
            for i, ((r, f, _), (idx, code)) in enumerate(recs.items()):
                d[i] = (r, idx, f, code)
                if f == A.DELTA_PHASE: phase[r, idx] = code
                elif f == A.DELTA_COND: cond[r, idx] = code
                elif f == A.DELTA_DECISION: dec[r, idx] = code
                elif f == A.DELTA_CHILD: child[r, idx] = code
                elif f == A.DELTA_RUN_FLAGS: rflags[r] = code
                elif f == A.DELTA_TOPO_SLOT:
                    slots[r] = idx | (code << 16)
                    dead[r] = slots[r] == dropped
                    if not dead[r]:
                        S_run[r] = S_of[int(slots[r])]
                else: reg[r] = (int(reg[r]) & ~(1 << idx)) | (code << idx)
            flags = A.EVAL_FIXPOINT if tick % 2 else 0
            max_iter = {1: 0, 3: 1, 5: 3}.get(tick, 0)
            dp = np.ascontiguousarray(d[rng.permutation(len(d))])
            want_state = pack_state(L, slots, rflags, phase, cond, dec, child, reg)
            if tick % 2:   # the fused call: deltas + pass + results, one synchronisation
                got, gcounts = fr.resident_tick(h, L, n, dp, flags=flags, max_iterations=max_iter)
            else:
                fr.resident_apply(h, dp)
                got, gcounts = fr.resident_eval(h, L, n, flags=flags)
            assert np.array_equal(fr.resident_download(h, 0, n, L.state_stride), want_state), "tick %d: device copy differs" % tick
            want, wcounts = _want_with_dead(pt, L, want_state, dead, flags, max_iter)
            assert np.array_equal(got, want), "tick %d" % tick
            assert gcounts == wcounts
        assert dead.any() and (S_run < W32).any()
        # a delta outside the batch is rejected, the rest of the call still lands
        bad = np.zeros(2, dtype=Frontier.DELTA_DTYPE)
        bad[0] = (n + 1000, 0, A.DELTA_PHASE, 3)
        bad[1] = (0, 0, A.DELTA_PHASE, 3)
        with pytest.raises(A.FrontierError):
            fr.resident_apply(h, bad)
        phase[0, 0] = 3
        assert np.array_equal(fr.resident_download(h, 0, 1, L.state_stride), pack_state(L, slots, rflags, phase, cond, dec, child, reg)[0:1])
        # the limiters accept a resident pass as "the batch just evaluated"
        fr.resident_eval(h, L, n)
        sched = np.zeros(n, dtype=np.dtype([("story_key", "<u4"), ("queue_key", "<u4"), ("priority", "<i4"), ("queued_elapsed_s", "<u4"),
                                            ("run_phase", "<u4"), ("reserved", "<u4", (3,))]))
        out = fr.schedule(L, n, sched, [0], [0], [0])
        assert out["records"].shape[0] == n
        fr.resident_destroy(h)
    finally:
        fr.close()


def test_tick_default_chunk_count(monkeypatch):
    """without BF_E2E_CHUNKS, a dense tick whose result records pass 2 MiB is cut into one chunk per ~2 MiB of them (rounded) and
    returns the oracle's records; a compact tick over the same batch keeps its results on the device and runs as one chunk"""
    monkeypatch.delenv("BF_E2E_CHUNKS", raising=False)
    rng = np.random.default_rng(6120)
    fr = Frontier(0)
    try:
        ts = randgen.random_topologies(rng, 30, 30, 256, parallel=False)
        slots = fr.put_topologies(ts)
        n = int(3.6 * (2 << 20)) // make_layout(int(ts.S.max()), 0, ALL).result_stride
        L, state, _ = randgen.random_state(rng, ts, slots, n, ALL, phase_mix="progress")
        rbytes = n * L.result_stride
        want_chunks = (rbytes + (1 << 20)) // (2 << 20)
        assert L.off_child == A.OFF_NONE and want_chunks == 4
        want, wcounts = PK.evaluate(PK.PackedTopologies(ts, slots), L, state, threads=8)
        h = fr.resident_create(L, n)
        fr.resident_upload(h, 0, state)
        none = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
        got, counts = fr.resident_tick(h, L, n, none)
        assert fr.stats()["last_eval_chunks"] == want_chunks
        assert np.array_equal(got, want) and counts == wcounts
        fr.resident_tick_compact(h, n, none, 1 << 22)
        assert fr.stats()["last_eval_chunks"] == 1
    finally:
        fr.close()


def test_host_mirror_resident_mode_matches_full_upload():
    """two bfh_batches fed the same event stream — one uploads everything every tick, one is resident and sends
    deltas — must return identical result records every tick; the resident one moves O(changes) bytes"""
    from bobrapet_b200 import host as H
    rng = np.random.default_rng(4242)
    fr = Frontier(0)
    hb_full = hb_res = None
    try:
        S, n = 96, 400
        hs = H.HostStory()
        for i in range(S):
            kind = A.STEP_GATE if i % 11 == 5 else (A.STEP_PARALLEL if i % 29 == 7 else A.STEP_ENGRAM)
            needs = ["s%d" % j for j in sorted(set(rng.integers(max(0, i - 9), i, size=min(i, 2)).tolist()))] if i else []
            hs.add_step("s%d" % i, 0, kind, allow_failure=(i % 13 == 0), if_expr=("{{ inputs.x }}" if i % 7 == 3 else None),
                        needs=needs, branches=([("b0", False), ("b1", True), ("b2", False)] if kind == A.STEP_PARALLEL else ()))
        hs.set_policy(continue_on_step_failure=True)
        assert hs.finalize() == 0, hs.error()
        slot = hs.upload(fr)
        _, _, _, n_par = hs.csr()
        fields = A.F_COND | A.F_DECISION | A.F_CHILD | A.F_ALL_OUT
        hb_full = H.HostBatch(fr, S, 8 * n_par, fields, n)
        hb_res = H.HostBatch(fr, S, 8 * n_par, fields, n)
        hb_res.set_resident(True)
        phases = ["", "Pending", "Running", "Succeeded", "Failed", "Paused", "Skipped", "Blocked", "Timeout"]
        for tick in range(6):
            if tick % 2 == 0:      # StoryRuns arrive over time
                for _ in range(n // 3 if tick < 4 else 0):
                    assert hb_full.add_run(hs, slot) == hb_res.add_run(hs, slot)
            live = hb_full._l.bfh_batch_size(hb_full._p)
            for _ in range(int(rng.integers(50, 900))):   # the tick's watch events; repeats on one step coalesce
                r, i = int(rng.integers(0, live)), int(rng.integers(0, S))
                ev = int(rng.integers(0, 7))
                for hb in (hb_full, hb_res):
                    if ev <= 2:
                        ph = phases[(r * 7 + i * 3 + tick + ev) % len(phases)]
                        hb.set_phase(r, i, ph, "Queued due to story concurrency limit (1 running, limit 1)" if (i + tick) % 5 == 0 else "")
                    elif ev == 3:
                        hb.set_cond(r, i, (r + i + tick) % 4)
                    elif ev == 4:
                        hb.set_gate(r, i, ["", "Approved", "Rejected", "Pending"][(r + i) % 4], timed_out=(tick % 2 == 0))
                    elif ev == 5:
                        hb.set_run_flags(r, topology_terminated=bool((r + tick) % 2))
                    else:
                        q = (r + i) % n_par
                        hb._chk(hb._l.bfh_run_register_children(hb._p, r, q, 1), "register")
                        hb._chk(hb._l.bfh_run_set_child_phase(hb._p, r, q, i % 3, phases[2 + (i + tick) % 5].encode()), "child")
            cf, cr = hb_full.eval(A.EVAL_FIXPOINT if tick % 2 else 0), hb_res.eval(A.EVAL_FIXPOINT if tick % 2 else 0)
            assert cf == cr, tick
            nb = live * hb_full.L.result_stride
            import ctypes as C
            a = np.frombuffer((C.c_uint8 * nb).from_address(hb_full._l.bfh_batch_result(hb_full._p)), dtype=np.uint8)
            b = np.frombuffer((C.c_uint8 * nb).from_address(hb_res._l.bfh_batch_result(hb_res._p)), dtype=np.uint8)
            assert np.array_equal(a, b), "tick %d: resident results differ" % tick
        full_bytes, delta_bytes, pending = hb_res.traffic()
        assert pending == 0
        assert full_bytes == live * hb_res.L.state_stride              # every run travelled once as a full record
        assert delta_bytes < 6 * 900 * 8 * 2                            # and afterwards only its changes
    finally:
        for hb in (hb_full, hb_res):
            if hb is not None:
                hb.close()
        fr.close()
