"""One-dependency probe batches for the dependency walks of the frontier kernels.

A random batch decides most verdicts by whichever of a row's four or five dependencies is unsatisfied, so a status read at
the wrong address or with the wrong shift flips a verdict only in the rare row where that one misread bit decides it.  Here
every walked reader's verdict rests on exactly one status read:

- ANCHOR steps are held Succeeded (or Skipped) in every run.  The first is a root, the others need earlier anchors.
- TARGET steps (the probes) need anchors only, so their own verdict never depends on a probe.  Each run draws their phase
  codes from satisfied, unsatisfied and failed ones; in cond batches a pending target with cond FAIL turns Failed inside the
  pass (the cond-FAIL fix-up).
- READER steps are pending and need one target d, their probe, plus anchors as fillers.  A u16 row shorter than K carries
  the PAD entry d = 32 W, a byte row repeats an entry.

Targets sit on every word's steps 0, 15, 16 and 31 (the half-word swap of the status words and the word edges), on steps
127, 128 and 255 (the offset bits of the in-place byte-entry walk) and on the last step; readers pick a target below or
above themselves with equal odds (forward references are legal), and the probe's place in the row is drawn too.  The rows
are made dense enough that each topology gets the row format it is meant for (plan_record, topology.cu), which
`row_format` restates.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import make_layout, pack_state

ANCHOR, TARGET, READER = 0, 1, 2

SAT = (3, 13)                          # Succeeded, Skipped: satisfied in every run
UNSAT = (0, 1, 2, 8, 9, 10, 14)        # not satisfied (1, 2, 8 and 14 are satisfied for realtime runs)
FAILED = (4, 5, 6, 7, 11, 12)          # terminal, not completed: a failed dependency under skip-on-failed


def _r16(x):
    return (x + 15) // 16 * 16


def row_format(S: int, E: int, max_deg: int, forced: str | None = None) -> str:
    """the row format plan_record (topology.cu) gives a topology without parallel steps; forced: BF_TOPO_FORMAT"""
    W = (S + 31) // 32
    rows = 32 * W
    csr = _r16(2 * (S + 1)) + _r16(2 * E + 8)
    K = 2 if max_deg <= 2 else (4 if max_deg <= 4 else 0)
    if K and forced != "csr":
        if rows <= 256 and forced != "ell16" and K * rows + 4 * W <= csr:
            return "byte%d" % K
        if K == 4 and W > 16 and forced != "ell16" and 5 * rows + 4 * W <= csr:
            return "p10"
        if 2 * K * rows <= csr and rows != 256:
            return "u16-%d" % K
    return "csr4" if max_deg <= 4 else "csrL"


def forced_format(kinds) -> str | None:
    """the BF_TOPO_FORMAT under which every kind of `kinds` can be had"""
    if "csr4" in kinds and len(set(kinds)) == 1:
        return "csr"
    if any(k.startswith("u16") for k in kinds):
        return "ell16"
    return None


def widths(kind: str, w_max: int, forced: str | None):
    """the topology widths (words) at which `kind` exists under `forced`, up to w_max"""
    if kind.startswith("byte"):
        return [w for w in range(1, min(w_max, 8) + 1)]
    if kind.startswith("u16"):
        return [w for w in range(1, min(w_max, 16) + 1) if w != 8]
    if kind == "csr4" and forced != "csr":
        return []
    return list(range(1, w_max + 1))


@dataclass
class ProbeTopologies:
    ts: TopologySet
    kinds: list        # intended row format of each topology
    roles: list        # per topology: role of each step (ANCHOR / TARGET / READER)
    probes: list       # per topology: probe d of each reader, -1 elsewhere
    af: list           # per topology: allowFailure of each step (targets only)

    @property
    def W(self):
        return (self.ts.S.astype(np.int64) + 31) // 32


def _target_positions(S: int):
    W = (S + 31) // 32
    pos = {32 * k + o for k in range(W) for o in (0, 15, 16, 31)} | {127, 128, 255, S - 1}
    return sorted(p for p in pos if p < S)


def _one(rng, S: int, kind: str, forced: str | None, p_short: float):
    K = 2 if kind.endswith("2") else 4
    long_rows = kind == "csrL"
    targets = _target_positions(S)
    free = np.setdiff1d(np.arange(S), targets)
    extra = rng.choice(free, size=len(free) // 10, replace=False) if len(free) >= 10 else np.zeros(0, np.int64)
    targets = np.union1d(targets, extra).astype(np.int64)
    free = np.setdiff1d(free, extra)
    n_anchor = min(len(free) - 1 if len(free) > 1 else len(free), max(8 if long_rows else K + 1, S // 12))
    anchors = np.sort(rng.choice(free, size=n_anchor, replace=False)) if n_anchor > 0 else np.zeros(0, np.int64)
    role = np.full(S, READER, np.int64)
    role[targets] = TARGET
    role[anchors] = ANCHOR
    probe = np.full(S, -1, np.int64)
    af = np.zeros(S, bool)
    af[targets] = rng.random(len(targets)) < 0.2
    rows = []
    for i in range(S):
        if role[i] == ANCHOR:
            prev = anchors[anchors < i]
            k = min(len(prev), K)
            rows.append(np.sort(rng.choice(prev, size=k, replace=False)) if k else np.zeros(0, np.int64))
        elif role[i] == TARGET:
            k = min(len(anchors), K if rng.random() >= p_short else int(rng.integers(0, K)))
            rows.append(rng.choice(anchors, size=k, replace=False) if k else np.zeros(0, np.int64))
        else:
            lo, hi = targets[targets < i], targets[targets > i]
            side = lo if (len(hi) == 0 or (len(lo) and rng.random() < 0.5)) else hi
            d = int(rng.choice(side))
            probe[i] = d
            if long_rows:
                n = int(rng.integers(1, 9)) if rng.random() < 0.6 else int(rng.integers(5, 9))
            elif kind == "csr4":
                n = int(rng.integers(1, 5))
            else:
                n = K if rng.random() >= p_short else int(rng.integers(1, K))
            n = min(n, len(anchors) + 1)
            fill = rng.choice(anchors, size=n - 1, replace=False) if n > 1 else np.zeros(0, np.int64)
            row = np.concatenate(([d], fill)).astype(np.int64)
            rows.append(rng.permutation(row))
    E = sum(len(r) for r in rows)
    md = max(len(r) for r in rows)
    return rows, role, probe, af, row_format(S, E, md, forced), E


def probe_topologies(rng, kinds, w_choices, forced: str | None = None, count: int = 24, full: float = 0.6) -> ProbeTopologies:
    """`count` probe topologies: topology t has kind t % len(kinds) and takes the widths (words) of w_choices in turn, the
    widest first, the others in random order; a topology is S = 32 W
    steps with probability `full`, else S is drawn in [32 W - 11, 32 W).  Each gets the row format of its kind under
    BF_TOPO_FORMAT = forced (asserted)."""
    S_l, E_l, rp_l, ci_l, fl_l, out_k, out_r, out_p, out_af = [], [], [], [], [], [], [], [], []
    order = [max(w_choices)] + list(rng.permutation([w for w in w_choices if w != max(w_choices)]))
    for t in range(count):
        kind = kinds[t % len(kinds)]
        ws = [w for w in order if w in widths(kind, max(w_choices), forced)]
        assert ws, (kind, w_choices, forced)
        W = int(ws[(t // len(kinds)) % len(ws)])
        S = 32 * W if rng.random() < full else int(rng.integers(32 * W - 11, 32 * W))
        p_short = 0.25
        for a in range(12):   # fewer short rows, then (a narrow u16 topology too short for its rows) all 32 W steps
            rows, role, probe, af, got, E = _one(rng, S, kind, forced, p_short)
            if got == kind:
                break
            p_short = p_short / 2 if p_short > 0.02 else 0.0
            if a == 5:
                S, p_short = 32 * W, 0.25
        assert got == kind, (kind, S, E, got)
        rp = np.zeros(S + 1, np.uint32)
        rp[1:] = np.cumsum([len(r) for r in rows])
        S_l.append(S)
        E_l.append(E)
        rp_l.append(rp)
        ci_l.append(np.concatenate(rows).astype(np.uint16))
        fl = np.zeros(S, np.uint8)                       # engram steps of the main group
        fl |= af.astype(np.uint8) * A.SF_ALLOW_FAILURE
        fl |= (rng.random(S) < 0.3).astype(np.uint8) * A.SF_HAS_IF
        fl_l.append(fl)
        out_k.append(kind)
        out_r.append(role)
        out_p.append(probe)
        out_af.append(af)
    ts = TopologySet(S_l, E_l, np.concatenate(rp_l), np.concatenate(ci_l), np.concatenate(fl_l))
    return ProbeTopologies(ts, out_k, out_r, out_p, out_af)


@dataclass
class ProbeState:
    L: object
    state: np.ndarray
    topo: np.ndarray       # topology of each run
    rflags: np.ndarray
    phase: np.ndarray      # [n, 32 * words] phase codes as packed
    cond: np.ndarray


def probe_state(rng, pt: ProbeTopologies, slots, n: int, words: int, fields: int, any_fd: bool = True,
                topo: np.ndarray | None = None) -> ProbeState:
    """n runs over the probe topologies at layout make_layout(32 * words) (at least as wide as every topology).
    any_fd False: every run fail-fast, so no group has a failed-dependency class.  True: runs fail-fast or skip-on-failed at
    random.  A quarter of the runs are realtime.  Cond batches (F_COND in fields): a pending target has cond FAIL with
    probability 0.4 (the fix-up probe); readers draw PASS / SKIP / HOLD / FAIL."""
    ts = pt.ts
    assert int(ts.S.max()) <= 32 * words
    L = make_layout(32 * words, 0, fields)
    width = 32 * words
    if topo is None:
        topo = rng.integers(0, ts.count, size=n)
    rf = np.zeros(n, np.uint8)
    ff = np.ones(n, bool) if not any_fd else rng.random(n) < 0.4
    rf |= ff.astype(np.uint8) * A.RF_FAIL_FAST
    rt = rng.random(n) < 0.25
    rf |= rt.astype(np.uint8) * A.RF_REALTIME
    rf |= ((rng.random(n) < 0.15) & ~rt).astype(np.uint8) * A.RF_TOPOLOGY_TERMINATED
    rf |= (rng.random(n) < 0.1).astype(np.uint8) * A.RF_HOST_GROUP   # host group MAIN (0 << RF_HOST_GROUP_SHIFT)
    # per-topology role and allowFailure planes, padded to the layout width
    role = np.full((ts.count, width), -1, np.int64)
    afm = np.zeros((ts.count, width), bool)
    for t in range(ts.count):
        S = int(ts.S[t])
        role[t, :S] = pt.roles[t]
        afm[t, :S] = pt.af[t]
    R, AFr = role[topo], afm[topo]
    sat = rng.choice(SAT, size=(n, width))
    uns = rng.choice(UNSAT, size=(n, width))
    fail = rng.choice(FAILED, size=(n, width))
    u = rng.random((n, width))
    # fail-fast runs: a failed main step would mark every pending step Skipped, so their targets fail only with allowFailure
    can_fail = ~ff[:, None] | AFr
    tphase = np.where(u < 0.35, sat, np.where((u < 0.7) | ~can_fail, uns, fail))
    phase = np.zeros((n, width), np.uint8)
    phase[R == ANCHOR] = sat[R == ANCHOR]
    phase[R == TARGET] = tphase[R == TARGET]
    phase[R == READER] = rng.choice([0, 0, 0, 9, 10, 14], size=int((R == READER).sum()))
    cond = None
    if fields & A.F_COND:
        cond = np.zeros((n, width), np.uint8)
        fix = (R == TARGET) & (rng.random((n, width)) < 0.4)
        phase[fix] = 0
        cond[fix] = A.COND_FAIL
        rd = R == READER
        cond[rd] = rng.choice(4, size=int(rd.sum()), p=[0.7, 0.1, 0.1, 0.1])
    dec = np.zeros((n, width), np.uint8) if fields & A.F_DECISION else None
    state = pack_state(L, np.asarray(slots)[topo], rf, phase, cond, dec)
    return ProbeState(L, state, topo, rf, phase, cond if cond is not None else np.zeros_like(phase))
