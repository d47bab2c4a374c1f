"""Adversarial random packed batches (all step types, groups, phases, codes) for differential tests."""
from __future__ import annotations

import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import PAR_DTYPE, make_layout, pack_state
from oracle.packed import child_first_of


def random_topologies(rng: np.random.Generator, count: int, s_min: int, s_max: int, max_deg: int = 5,
                      groups: bool = True, parallel: bool = True, forward_refs: bool = True, fill: float = 0.0,
                      branch_choices=(0, 1, 2, 3, 7, 8, 9, 31, 32, 33, 40)) -> TopologySet:
    """fill: probability that a step takes the full max_deg needs (dense low-degree graphs qualify for the
    fixed-width row format of the device records; sparse ones stay CSR)"""
    S_l, E_l, P_l, rp_l, ci_l, fl_l, par_l, allow_bits = [], [], [], [], [], [], [], []
    for _ in range(count):
        S = int(rng.integers(s_min, s_max + 1))
        # acyclic order: deps point to lower rank in a random permutation (so dep index may exceed step index)
        rank = rng.permutation(S) if forward_refs else np.arange(S)
        order = np.argsort(rank)
        rows = []
        for i in range(S):
            r = int(rank[i])
            k = int(min(r, max_deg if rng.random() < fill else rng.integers(0, max_deg + 1)))
            if k and rng.random() < 0.7:  # local window, like real workflows
                lo = max(0, r - 16)
                cands = order[lo:r]
            else:
                cands = order[:r]
            k = min(k, len(cands))
            rows.append(np.sort(rng.choice(cands, size=k, replace=False)) if k else np.zeros(0, np.int64))
        rp = np.zeros(S + 1, np.uint32)
        rp[1:] = np.cumsum([len(r) for r in rows])
        ci = np.concatenate(rows).astype(np.uint16) if rp[-1] else np.zeros(0, np.uint16)
        types = rng.choice(8, size=S, p=[0.45, 0.1, 0.08 if parallel else 0.0, 0.07, 0.03, 0.07, 0.05,
                                         0.15 if parallel else 0.23])
        fl = types.astype(np.uint8)
        fl |= (rng.random(S) < 0.15).astype(np.uint8) * A.SF_ALLOW_FAILURE
        fl |= (rng.random(S) < 0.4).astype(np.uint8) * A.SF_ON_TIMEOUT_SKIP
        fl |= (rng.random(S) < 0.3).astype(np.uint8) * A.SF_HAS_IF
        if groups and rng.random() < 0.7:
            # main ++ compensations ++ finally are contiguous index ranges (allStorySteps, dag.go:3270)
            cuts = np.sort(rng.integers(0, S + 1, size=2))
            g = np.zeros(S, np.uint8)
            g[cuts[0]:cuts[1]] = 1
            g[cuts[1]:] = 2
            fl |= g << A.SF_GROUP_SHIFT
        par_idx = np.nonzero(types == A.STEP_PARALLEL)[0][:A.MAX_PARALLEL]
        # steps typed parallel beyond the 64-desc cap become engrams
        extra = np.nonzero(types == A.STEP_PARALLEL)[0][A.MAX_PARALLEL:]
        fl[extra] &= ~np.uint8(A.SF_TYPE_MASK)
        pd = np.zeros(len(par_idx), PAR_DTYPE)
        for q, stp in enumerate(par_idx):
            B = int(rng.choice(list(branch_choices)))
            pd[q] = (stp, B, len(allow_bits))
            allow_bits.extend((rng.random(B) < 0.3).tolist())
        S_l.append(S); E_l.append(int(rp[-1])); P_l.append(len(par_idx))
        rp_l.append(rp); ci_l.append(ci); fl_l.append(fl); par_l.append(pd)
    bits = np.asarray(allow_bits + [False] * ((-len(allow_bits)) % 8), dtype=bool)
    allow = np.packbits(bits, bitorder="little") if len(allow_bits) else None
    return TopologySet(S_l, E_l, np.concatenate(rp_l), np.concatenate(ci_l) if sum(E_l) else np.zeros(0, np.uint16),
                       np.concatenate(fl_l), P_l, np.concatenate(par_l) if sum(P_l) else None, allow)


def child_layout(ts: TopologySet):
    """per-topology child_first arrays and the max child nibble count"""
    out, pos, mx = [], 0, 0
    for i in range(ts.count):
        p = int(ts.P[i])
        br = ts.parallel["branches"][pos:pos + p].astype(np.int64)
        cf = child_first_of(br)
        out.append(cf)
        if p:
            mx = max(mx, int((int(cf[-1]) + int(br[-1]) + 7) // 8 * 8))
        pos += p
    return out, mx


def random_state(rng: np.random.Generator, ts: TopologySet, slots: np.ndarray, n_runs: int, fields: int,
                 phase_mix: str = "any", fail_codes: bool = True, run_flag_mix: bool = True,
                 reserved: float = 0.0, padding: bool = False, fail_fast=None):
    """-> (layout, state records, topo index per run).  `slots[t]` is the slot of topology t.

    Records no well-behaved producer writes, which the kernels must read exactly as their `cleaned` twin:
    reserved: the rate at which phase codes below S and child nibbles are replaced by the reserved code 15;
    padding: random phase, cond and decision codes in the steps from a run's S up to the layout width (32 * words).
    fail_fast: True / False sets RF_FAIL_FAST on every run instead of the random mix."""
    cfs, child_max = child_layout(ts)
    if child_max:
        fields |= A.F_CHILD
    s_max = int(ts.S.max())
    L = make_layout(s_max, child_max, fields)
    topo = rng.integers(0, ts.count, size=n_runs)
    if phase_mix == "any":
        phase = rng.integers(0, 15, size=(n_runs, s_max)).astype(np.uint8)
    else:  # progress-shaped, closer to live workflows
        prog = rng.integers(0, s_max + 1, size=(n_runs, 1))
        idx = np.arange(s_max)[None, :]
        done = rng.choice([3, 13, 4, 2, 8, 11, 6, 1], size=(n_runs, s_max), p=[0.8, 0.04, 0.03, 0.05, 0.03, 0.01, 0.01, 0.03])
        todo = rng.choice([0, 14, 9, 10], size=(n_runs, s_max), p=[0.93, 0.04, 0.02, 0.01])
        phase = np.where(idx < prog, done, todo).astype(np.uint8)
    pc = [0.55, 0.2, 0.15, 0.1] if fail_codes else [0.6, 0.25, 0.15, 0.0]
    cond = rng.choice(4, size=(n_runs, s_max), p=pc).astype(np.uint8)
    dec = rng.integers(0, 4, size=(n_runs, s_max)).astype(np.uint8)
    child = rng.choice([0, 2, 3, 3, 3, 3, 4, 13, 11, 1], size=(n_runs, max(child_max, 1))).astype(np.uint8)
    all_done = rng.random(n_runs) < 0.5
    child[all_done] = rng.choice([3, 3, 3, 3, 13, 4], size=(int(all_done.sum()), child.shape[1])).astype(np.uint8)
    reg = rng.integers(0, 2**63, size=n_runs, dtype=np.uint64) | (rng.integers(0, 2, size=n_runs, dtype=np.uint64) << np.uint64(63))
    rflags = np.zeros(n_runs, np.uint8)
    if run_flag_mix:
        rflags |= (rng.random(n_runs) < 0.5).astype(np.uint8) * A.RF_FAIL_FAST
        rflags |= (rng.random(n_runs) < 0.25).astype(np.uint8) * A.RF_REALTIME
        rflags |= (rng.random(n_runs) < 0.3).astype(np.uint8) * A.RF_TOPOLOGY_TERMINATED
        hg = rng.random(n_runs) < 0.2
        rflags |= hg.astype(np.uint8) * A.RF_HOST_GROUP
        rflags |= (hg * rng.integers(0, 4, size=n_runs)).astype(np.uint8) << A.RF_HOST_GROUP_SHIFT
    if fail_fast is not None:
        rflags = (rflags & ~np.uint8(A.RF_FAIL_FAST)) | (np.uint8(A.RF_FAIL_FAST) if fail_fast else np.uint8(0))
    # zero the codes beyond each run's own S (padding must not matter, but keep records canonical)
    Srun = ts.S[topo].astype(np.int64)[:, None]
    pad = np.arange(s_max)[None, :] >= Srun
    phase[pad] = 0; cond[pad] = 0; dec[pad] = 0
    if reserved:   # drawn after every canonical field: the same seed gives the same run otherwise
        phase[(rng.random(phase.shape) < reserved) & ~pad] = 15
        child[rng.random(child.shape) < reserved] = 15
    if padding:
        width = 32 * L.words
        wpad = np.arange(width)[None, :] >= Srun
        wide = lambda a: np.concatenate([a, np.zeros((n_runs, width - s_max), np.uint8)], axis=1)  # noqa: E731
        phase, cond, dec = wide(phase), wide(cond), wide(dec)
        phase[wpad] = rng.integers(0, 16, size=int(wpad.sum()), dtype=np.uint8)
        cond[wpad] = rng.integers(0, 4, size=int(wpad.sum()), dtype=np.uint8)
        dec[wpad] = rng.integers(0, 4, size=int(wpad.sum()), dtype=np.uint8)
    state = pack_state(L, np.asarray(slots)[topo], rflags, phase, cond, dec, child if child_max else None, reg)
    return L, state, topo


def cleaned(L, state: np.ndarray, ts: TopologySet, topo: np.ndarray) -> np.ndarray:
    """The canonical twin of a state batch: phase code 15 -> 0, child nibble 15 -> 0, and every phase / cond / decision
    code at or past a run's own S zeroed.  Every evaluator must give a record and its twin the same result."""
    from bobrapet_b200.records import _pack_nibbles, _pack_planes, _unpack_planes
    out = state.copy()
    W = L.words
    pad = np.arange(32 * W)[None, :] >= ts.S[topo].astype(np.int64)[:, None]
    for off, nbits in ((L.off_phase, 4), (L.off_cond, 2), (L.off_decision, 2)):
        if off == A.OFF_NONE:
            continue
        codes = _unpack_planes(out[:, off:off + nbits * W * 4], W, nbits, 32 * W)
        codes[pad] = 0
        if nbits == 4:
            codes[codes == 15] = 0
        out[:, off:off + nbits * W * 4] = _pack_planes(codes, W, nbits)
    if L.off_child != A.OFF_NONE and L.child_nibbles:
        nb = (L.child_nibbles + 1) // 2
        raw = out[:, L.off_child:L.off_child + nb]
        nib = np.stack([raw & 0xF, raw >> 4], axis=2).reshape(raw.shape[0], 2 * nb)
        nib[nib == 15] = 0
        out[:, L.off_child:L.off_child + nb] = _pack_nibbles(nib, nb)
    return out
