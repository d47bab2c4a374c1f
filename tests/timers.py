"""A host model of a resident batch's step-timer area (bf_resident_timers*, bf_resident_fire and what the other resident calls do
to the area), written from the contract in include/bobrafrontier.h.

An area is a numpy uint64 array of shape (capacity, K): slot = deadline | step << 32 | code << 48 (bf_timer_slot read as one
little-endian u64), EMPTY = deadline BF_TIMER_NONE with every other byte 0.  A run's armed slots come first, ascending by step.
State records are the uint8 arrays of tests/packing.py (one row per run); fire() reads and writes them in place."""
import numpy as np

NONE = 0xFFFFFFFF
EMPTY = np.uint64(NONE)
LUT_TERMINAL = 0x38F8
DEC_PENDING = 0
EINVAL, ENOMEM = -1, -2
F_DECISION = 0x2
OFF_NONE = 0xFFFFFFFF
MIGRATE_GONE = 0xFFFF


def slot(deadline, step, code):
    return np.uint64(int(deadline) | int(step) << 32 | int(code) << 48)


def unpack(v):
    v = int(v)
    return v & 0xFFFFFFFF, (v >> 32) & 0xFFFF, (v >> 48) & 0xFF


def empty_area(cap, K):
    return np.full((cap, K), EMPTY, dtype=np.uint64)


def armed(row):
    """(step, deadline, code) of a row's armed slots, in slot order"""
    out = []
    for v in row:
        d, s, c = unpack(v)
        if d != NONE:
            out.append((s, d, c))
    return out


def canonical(entries, K):
    """a row from {step: (deadline, code)}: armed slots ascending by step, then empty ones"""
    row = np.full(K, EMPTY, dtype=np.uint64)
    for k, s in enumerate(sorted(entries)):
        row[k] = slot(entries[s][0], s, entries[s][1])
    return row


def grow(area, K):
    """bf_resident_timers on a batch that has an area: K grows, every slot stays where it was"""
    assert K >= area.shape[1]
    out = empty_area(area.shape[0], K)
    out[:, :area.shape[1]] = area
    return out


def check_arm(area, L, reqs):
    """the status bf_resident_timers_arm returns (0, EINVAL or ENOMEM), and on ENOMEM the run named"""
    if area is None:
        return EINVAL, None
    cap, K = area.shape
    seen = set()
    for q in reqs:
        run, step, code = int(q["run"]), int(q["step"]), int(q["code"])
        if run >= cap or step >= L.steps_max or code > 3 or q["reserved"] or q["reserved2"]:
            return EINVAL, None
        if code != DEC_PENDING and L.off_decision == OFF_NONE:
            return EINVAL, None
        if (run, step) in seen:
            return EINVAL, None
        seen.add((run, step))
    for run in sorted({int(q["run"]) for q in reqs}):
        if len(_merged(area[run], [q for q in reqs if int(q["run"]) == run])) > K:
            return ENOMEM, run
    return 0, None


def _merged(row, reqs):
    entries = {s: (d, c) for s, d, c in armed(row)}
    for q in reqs:
        s = int(q["step"])
        if int(q["deadline"]) == NONE:
            entries.pop(s, None)
        else:
            entries[s] = (int(q["deadline"]), int(q["code"]))
    return entries


def arm(area, L, reqs):
    """bf_resident_timers_arm -> status; the area changes only on 0"""
    rc, _ = check_arm(area, L, reqs)
    if rc:
        return rc
    K = area.shape[1]
    for run in sorted({int(q["run"]) for q in reqs}):
        area[run] = canonical(_merged(area[run], [q for q in reqs if int(q["run"]) == run]), K)
    return 0


def _get(rec, off, words, nbits, s):
    w = rec[off:off + 4 * nbits * words].view("<u4")
    return sum((((int(w[b * words + (s >> 5)]) >> (s & 31)) & 1) << b) for b in range(nbits))


def _set(rec, off, words, nbits, s, code):
    w = rec[off:off + 4 * nbits * words].view("<u4")
    for b in range(nbits):
        bit = np.uint32(1 << (s & 31))
        i = b * words + (s >> 5)
        w[i] = (w[i] | bit) if (code >> b) & 1 else (w[i] & ~bit)


def phase(L, rec, s):
    return _get(rec, L.off_phase, L.words, 4, s)


def decision(L, rec, s):
    return _get(rec, L.off_decision, L.words, 2, s) if L.off_decision != OFF_NONE else DEC_PENDING


def fire(area, L, state, n_runs, now):
    """bf_resident_fire over runs [0, n_runs): the area and `state` change in place.
    -> dict(n_fired, n_written, n_pruned, next_deadline, fired [(run, step, code, written)], touched {runs})"""
    K = area.shape[1]
    out = {"n_fired": 0, "n_written": 0, "n_pruned": 0, "next_deadline": NONE, "fired": [], "touched": set()}
    for r in range(n_runs):
        rec = state[r]
        keep = {}
        for s, d, c in armed(area[r]):
            if (LUT_TERMINAL >> phase(L, rec, s)) & 1:
                out["n_pruned"] += 1
                continue
            if d > now:
                keep[s] = (d, c)
                out["next_deadline"] = min(out["next_deadline"], d)
                continue
            w = c != DEC_PENDING and L.off_decision != OFF_NONE and decision(L, rec, s) == DEC_PENDING
            if w:
                _set(rec, L.off_decision, L.words, 2, s, c)
                out["touched"].add(r)
                out["n_written"] += 1
            out["n_fired"] += 1
            out["fired"].append((r, s, c, int(w)))
        area[r] = canonical(keep, K)
    return out


def as_deltas(fired, dtype):
    """the written codes of a fire as BF_DELTA_DECISION deltas (the fire's equivalence)"""
    rows = [(r, s, 2, c) for r, s, c, w in fired if w]
    d = np.zeros(len(rows), dtype=dtype)
    for i, (r, s, f, c) in enumerate(rows):
        d[i] = (r, s, f, c)
    return d


def retire_moves(N, runs):
    """the move rule of bf_resident_retire -> (m, {source: target})"""
    gone = set(int(x) for x in runs)
    m = N - len(gone)
    holes = [i for i in range(m) if i in gone]
    sources = [i for i in range(m, N) if i not in gone]
    return m, dict(zip(sources, holes))


def retire(area, N, runs, capacity=0):
    """bf_resident_retire -> the new area (a new capacity re-allocates it)"""
    m, mv = retire_moves(N, runs)
    out = area.copy()
    for src, dst in mv.items():
        out[dst] = area[src]
    out[m:N] = EMPTY
    if capacity:
        out = out[:capacity].copy()
    return out


def fits(src_area, run, dst_K):
    """a moved run's armed slots fit the destination's K (0 without an area)"""
    return src_area is None or len(armed(src_area[run])) <= dst_K


def transfer(src_area, dst_area, src_N, dst_first, runs):
    """bf_resident_transfer after the fit check -> (source area, destination area); either may be None (no area)"""
    if dst_area is not None:
        dst_area = dst_area.copy()
        K = dst_area.shape[1]
        for i, r in enumerate(runs):
            dst_area[dst_first + i] = canonical({} if src_area is None else {s: (d, c) for s, d, c in armed(src_area[r])}, K)
    if src_area is not None:
        src_area = retire(src_area, src_N, runs)
    return src_area, dst_area


def migrate(area, migrated_runs, step_map):
    """bf_resident_migrate: the slots of each migrated run re-indexed through step_map (gone or unmapped steps cancelled)"""
    out = area.copy()
    K = area.shape[1]
    for r in migrated_runs:
        e = {}
        for s, d, c in armed(area[r]):
            t = int(step_map[s]) if s < len(step_map) else MIGRATE_GONE
            if t != MIGRATE_GONE:
                e[t] = (d, c)
        out[r] = canonical(e, K)
    return out


def redrive(area, requests, status):
    """bf_resident_redrive: every slot of a run with an applied request is emptied"""
    out = area.copy()
    for q, st in zip(requests, status):
        if st:
            out[int(q["run"])] = EMPTY
    return out


def reshape(area, capacity):
    """bf_resident_reshape: a larger capacity extends the area with empty slots"""
    out = empty_area(max(capacity, area.shape[0]), area.shape[1])
    out[:area.shape[0]] = area
    return out


def extent(area):
    """the timers' share of bf_resident_extent: (steps, BF_F_DECISION or 0, lowest record needing those steps or None)"""
    steps, fields, widest = 0, 0, None
    for r in range(area.shape[0]):
        for s, d, c in armed(area[r]):
            if s + 1 > steps:
                steps, widest = s + 1, r
            if c != DEC_PENDING:
                fields |= F_DECISION
    return steps, fields, widest
