"""The limiter reference of the schedule tests: what bf_schedule must return for a batch's state and result records.

A batch's topologies are described per slot (SlotDesc).  Two sources supply that description: a randgen TopologySet with
the slots it was put at (from_topology_set), and the topology registry of the resident sequence model
(tests/resident_model.Registry, from_registry), whose live slots are the only ones a run can count on.

expected() reduces the records to per-run Running counts and demand exactly as the contract of include/bobrafrontier.h
states it (its limiter block lists the edges), then limits the ready masks with schedule_fast, a numpy restatement of
oracle.limiters.schedule_packed.  schedule_packed stays the definition; test_schedref.py checks that the two agree.

schedule_device() runs Frontier.schedule_device over device copies of its inputs, for the tests and tools of the device path.

The generators at the end draw sched runs and tables over the whole input range: every run_phase code and values past
15, int32 priority extremes, elapsed times at the clamp and BF_SCHED_NONE, negative and huge limits and aging, and keys
out of range."""
from __future__ import annotations

from typing import Dict, NamedTuple

import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import _unpack_planes
from oracle import limiters as LM
from tests import randgen

INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


class SlotDesc(NamedTuple):
    S: int
    engram: np.ndarray        # [S] bool: the step owns a StepRun when Running (step type 0)
    branches: np.ndarray      # [P] int64
    child_first: np.ndarray   # [P] int64: first child nibble of each parallel step


def slot_descs(ts, topo_of_slot: Dict[int, int]) -> Dict[int, SlotDesc]:
    """slot -> SlotDesc for the TopologySet rows topo_of_slot names"""
    S_off = np.concatenate(([0], np.cumsum(ts.S.astype(np.int64))))
    P_off = np.concatenate(([0], np.cumsum(ts.P.astype(np.int64))))
    cfs, _ = randgen.child_layout(ts)
    out = {}
    for slot, t in topo_of_slot.items():
        S, P = int(ts.S[t]), int(ts.P[t])
        types = ts.step_flags[S_off[t]:S_off[t] + S] & A.SF_TYPE_MASK
        br = ts.parallel["branches"][P_off[t]:P_off[t] + P].astype(np.int64) if P else np.zeros(0, np.int64)
        out[int(slot)] = SlotDesc(S, types == 0, br, np.asarray(cfs[t], np.int64)[:P])
    return out


def from_topology_set(ts, slots) -> Dict[int, SlotDesc]:
    return slot_descs(ts, {int(s): t for t, s in enumerate(slots)})


def from_registry(reg) -> Dict[int, SlotDesc]:
    """the live slots of a resident_model.Registry (row k of reg.ts is pool Story k)"""
    return slot_descs(reg.ts, {int(s): int(k) for s, k in reg.live.items()})


def running_and_demand(L, state: np.ndarray, descs: Dict[int, SlotDesc]):
    """-> (run_running, run_demand) [n] uint32: Running engram steps + Running children of registered parallel steps, and
    whether some step is Running (2) or queued (14), read from the records as stored.  Runs on slots descs does not hold
    count nothing."""
    n, W = state.shape[0], L.words
    running = np.zeros(n, np.uint32)
    demand = np.zeros(n, np.uint32)
    if n == 0:
        return running, demand
    sid = np.ascontiguousarray(state[:, 0:4]).view("<u4")[:, 0]
    reg = np.ascontiguousarray(state[:, 8:16]).view("<u8")[:, 0]
    codes = _unpack_planes(state[:, L.off_phase:L.off_phase + 16 * W], W, 4, 32 * W)
    nib = None
    if L.off_child != A.OFF_NONE and L.child_nibbles:
        nb = (L.child_nibbles + 1) // 2
        raw = state[:, L.off_child:L.off_child + nb]
        nib = np.stack([raw & 0xF, raw >> 4], axis=2).reshape(n, 2 * nb)
    for slot, d in descs.items():
        rows = np.nonzero(sid == slot)[0]
        if rows.size == 0 or (d.S + 31) // 32 > W:
            continue
        ph = codes[rows, :d.S]
        cnt = ((ph == 2) & d.engram[None, :]).sum(axis=1).astype(np.int64)
        demand[rows] = ((ph == 2) | (ph == 14)).any(axis=1)
        if nib is not None:
            for q in range(len(d.branches)):
                c0, B = int(d.child_first[q]), int(d.branches[q])
                if c0 + B > L.child_nibbles:
                    continue
                sel = ((reg[rows] >> np.uint64(q)) & np.uint64(1)).astype(bool)
                cnt[sel] += (nib[rows[sel], c0:c0 + B] == 2).sum(axis=1)
        running[rows] = cnt
    return running, demand


# ------------------------------------------------------------------------------------------ vectorised schedule_packed
def popcount(masks: np.ndarray) -> np.ndarray:
    """set bits per row of a [n, W] uint32 mask array"""
    return np.bitwise_count(masks).sum(axis=1, dtype=np.int64)


def truncate_rows(masks: np.ndarray, keep: np.ndarray) -> np.ndarray:
    """row r keeps its first keep[r] set bits (LSB first, word 0 first): LM.truncate_mask on every row"""
    n, W = masks.shape
    if n == 0:
        return masks.copy()
    c = np.bitwise_count(masks).astype(np.int64)
    incl = np.cumsum(c, axis=1)
    excl = incl - c
    k = np.asarray(keep, np.int64)[:, None]
    out = np.where(incl <= k, masks, np.uint32(0)).astype(np.uint32)
    r, w = np.nonzero((excl < k) & (incl > k))          # at most one split word per row
    if r.size:
        need = (k[r, 0] - excl[r, w])[:, None]
        bits = (masks[r, w][:, None] >> np.arange(32, dtype=np.uint32)) & np.uint32(1)
        kept = bits * (np.cumsum(bits, axis=1) <= need)
        out[r, w] = (kept.astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
    return out


def effective_priority_rows(priority, elapsed, aging) -> np.ndarray:
    """LM.effective_priority_packed per run, as int32"""
    el = np.asarray(elapsed, np.uint32).astype(np.int64)
    ag = np.asarray(aging, np.int64)
    base = np.asarray(priority, np.int64)
    live = (el != LM.NONE_U32) & (ag > 0) & (el != 0)
    steps = np.where(live, np.minimum(el, INT32_MAX) // np.where(ag > 0, ag, 1), 0)
    return ((np.where(steps > 0, base + steps, base) + (1 << 31)) % (1 << 32) - (1 << 31)).astype(np.int32)


def schedule_fast(run_running, run_demand, sched, ready_masks, story_limit, story_base, queue_limit, queue_aging, queue_base,
                  global_limit, global_base, queue_maxprio_base=None):
    """LM.schedule_packed with numpy: same arguments, same results"""
    n, W = ready_masks.shape
    ns, nq = len(story_limit), len(queue_limit)
    sk, qk = sched["story_key"].astype(np.int64), sched["queue_key"].astype(np.int64)
    ks, kq = sk < ns, qk < nq
    rr = np.asarray(run_running, np.int64)
    story_running = np.asarray(story_base, np.int64).copy()
    queue_running = np.asarray(queue_base, np.int64).copy()
    np.add.at(story_running, sk[ks], rr[ks])
    np.add.at(queue_running, qk[kq], rr[kq])
    global_running = int(global_base) + int(rr.sum())
    qa = np.asarray(queue_aging, np.int64)
    eff = effective_priority_rows(sched["priority"], sched["queued_elapsed_s"], np.where(kq, qa[np.minimum(qk, max(nq - 1, 0))] if nq else 0, 0))
    phase = sched["run_phase"] & 0xF
    demand = ~np.isin(phase, LM.TERMINAL_PHASES) & (np.isin(phase, [1, 2]) | (np.asarray(run_demand) != 0))
    maxprio = (np.full(nq, INT32_MIN, np.int32) if queue_maxprio_base is None
               else np.asarray(queue_maxprio_base, np.int32).copy())
    sel = demand & kq
    np.maximum.at(maxprio, qk[sel], eff[sel])

    cur = ready_masks.copy()
    cnt = popcount(cur)
    q_story = np.zeros_like(cur)
    q_sched = np.zeros_like(cur)
    sl = np.asarray(story_limit, np.int64)
    lim = np.where(ks, sl[np.minimum(sk, max(ns - 1, 0))] if ns else 0, 0)
    srun = np.where(ks, story_running[np.minimum(sk, max(ns - 1, 0))] if ns else 0, 0)
    slots = np.maximum(lim - srun, 0)
    cut = (cnt > 0) & (lim > 0) & (slots < cnt)
    if cut.any():
        kept = truncate_rows(cur[cut], slots[cut])
        q_story[cut] = cur[cut] & ~kept
        cur[cut] = kept
        cnt[cut] = slots[cut]

    reason = np.zeros(n, np.uint32)
    mp = np.where(kq, maxprio[np.minimum(qk, max(nq - 1, 0))] if nq else INT32_MIN, INT32_MIN).astype(np.int64)
    prio = (cnt > 0) & kq & (mp > eff)
    q_sched[prio] = cur[prio]
    cur[prio] = 0
    reason[prio] = LM.REASON_PRIORITY
    gl = int(global_limit)
    ql = np.where(kq, np.asarray(queue_limit, np.int64)[np.minimum(qk, max(nq - 1, 0))] if nq else 0, 0)
    qrun = np.where(kq, queue_running[np.minimum(qk, max(nq - 1, 0))] if nq else 0, 0)
    gslots = np.full(n, max(gl - global_running, 0), np.int64) if gl > 0 else cnt
    qslots = np.where(ql > 0, np.maximum(ql - qrun, 0), cnt)
    slots = np.minimum(cnt, np.minimum(gslots, qslots))
    cut = (cnt > 0) & ~prio & (slots < cnt)
    if cut.any():
        kept = truncate_rows(cur[cut], slots[cut])
        q_sched[cut] = cur[cut] & ~kept
        cur[cut] = kept
        why = np.where((gl > 0) & ((ql <= 0) | (gslots <= qslots)), LM.REASON_GLOBAL,
                       np.where(ql > 0, LM.REASON_QUEUE, LM.REASON_OTHER))
        reason[cut] = why[cut]
    info = np.stack([popcount(cur), popcount(q_story), popcount(q_sched), reason], axis=1).astype(np.uint32)
    return cur, q_story, q_sched, info, story_running, queue_running, global_running, maxprio


# ------------------------------------------------------------------------------------------ expected bf_schedule output
def ready_of(L, result: np.ndarray) -> np.ndarray:
    n, W = result.shape[0], L.words
    return np.ascontiguousarray(result[:, L.off_ready:L.off_ready + 4 * W]).view("<u4").reshape(n, W)


def expected(L, state: np.ndarray, result: np.ndarray, descs: Dict[int, SlotDesc], sched: np.ndarray, tables: dict,
             loop: bool = False) -> dict:
    """what bf_schedule returns for the batch (state, result) with these sched runs and tables (Frontier.schedule's
    keyword arguments).  loop: use the definition (LM.schedule_packed) instead of schedule_fast"""
    n, W = state.shape[0], L.words
    rr, rd = running_and_demand(L, state, descs)
    sl = np.asarray(tables["story_limit"], np.int32)
    ql = np.asarray(tables["queue_limit"], np.int32)
    sb = tables.get("story_running_base")
    qb = tables.get("queue_running_base")
    fn = LM.schedule_packed if loop else schedule_fast
    launch, q_story, q_sched, info, sr, qr, gr, mp = fn(
        rr, rd, sched, ready_of(L, result).copy(), sl, np.zeros(sl.size, np.uint32) if sb is None else np.asarray(sb, np.uint32),
        ql, np.asarray(tables["queue_aging_s"], np.int32), np.zeros(ql.size, np.uint32) if qb is None else np.asarray(qb, np.uint32),
        int(tables.get("global_limit", 0)), int(tables.get("global_running_base", 0)), tables.get("queue_max_priority_base"))
    rec = np.zeros((n, A.sched_stride(W)), np.uint8)
    rec[:, 0:16] = info.astype("<u4").view(np.uint8).reshape(n, 16)
    rec[:, 16:16 + 12 * W] = np.concatenate([launch, q_story, q_sched], axis=1).astype("<u4").view(np.uint8).reshape(n, 12 * W)
    return {"records": rec, "story_running": (sr % (1 << 32)).astype(np.uint32), "queue_running": (qr % (1 << 32)).astype(np.uint32),
            "queue_max_priority": mp.astype(np.int32), "global_running": gr % (1 << 32)}


def assert_schedule(got: dict, want: dict, what: str = ""):
    """bit for bit: every record including its zeroed tail, and every total"""
    for k in ("story_running", "queue_running", "queue_max_priority"):
        assert np.array_equal(got[k], want[k]), "%s %s differ at %s" % (what, k, np.nonzero(got[k] != want[k])[0][:10].tolist())
    assert got["global_running"] == want["global_running"], "%s global_running %d, want %d" % (what, got["global_running"],
                                                                                             want["global_running"])
    bad = np.nonzero((got["records"] != want["records"]).any(axis=1))[0]
    assert bad.size == 0, "%s schedule records differ in %d runs, first %s: got %s want %s" % (
        what, bad.size, bad[:8].tolist(), got["records"][bad[0], :32].tolist(), want["records"][bad[0], :32].tolist())


# ------------------------------------------------------------------------------------------ the device path
def to_device(a, dev):
    """a torch device copy of a numpy array, 4-byte elements as int32 and everything else as bytes"""
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int32) if a.dtype.itemsize == 4 else a.view(np.uint8)).to(dev)


def schedule_device(fr, L, n, d_state, d_result, sched, tables, stream, garbage=0xA5):
    """Frontier.schedule_device over device copies of the sched runs and tables (the state and result records are torch device
    tensors already), into output buffers pre-filled with garbage; synchronises `stream` -> dict as Frontier.schedule returns"""
    import torch
    dev = d_state.device if d_state is not None else torch.device("cuda", 0)
    ns, nq = len(tables["story_limit"]), len(tables["queue_limit"])
    t = {k: to_device(v, dev) for k, v in tables.items() if isinstance(v, np.ndarray) and v.size}
    d_runs = to_device(sched.view(np.uint8), dev) if n else None
    rec = torch.full((max(n, 1), A.sched_stride(L.words)), garbage, dtype=torch.uint8, device=dev)
    sr, qr, mp, gr = (torch.full((max(m, 1),), 0x77, dtype=torch.int32, device=dev) for m in (ns, nq, nq, 1))
    ptr = lambda x: 0 if x is None else x.data_ptr()  # noqa: E731
    torch.cuda.synchronize()
    fr.schedule_device(L, n, ptr(d_state) if n else 0, ptr(d_result) if n else 0, ptr(d_runs), rec.data_ptr() if n else 0,
                       sr.data_ptr(), qr.data_ptr(), mp.data_ptr(), gr.data_ptr(), ns, nq, ptr(t.get("story_limit")),
                       ptr(t.get("queue_limit")), ptr(t.get("queue_aging_s")), global_limit=int(tables.get("global_limit", 0)),
                       global_running_base=int(tables.get("global_running_base", 0)),
                       story_running_base_ptr=ptr(t.get("story_running_base")), queue_running_base_ptr=ptr(t.get("queue_running_base")),
                       queue_max_priority_base_ptr=ptr(t.get("queue_max_priority_base")), stream=stream.cuda_stream)
    stream.synchronize()
    return {"records": rec.cpu().numpy()[:n], "story_running": sr.cpu().numpy().view(np.uint32)[:ns],
            "queue_running": qr.cpu().numpy().view(np.uint32)[:nq], "queue_max_priority": mp.cpu().numpy()[:nq],
            "global_running": int(gr.cpu().numpy().view(np.uint32)[0])}


# ------------------------------------------------------------------------------------------ generators
PRIORITY_EDGES = (INT32_MIN, INT32_MIN + 1, -1, 0, 1, INT32_MAX - 2, INT32_MAX - 1, INT32_MAX)
ELAPSED_EDGES = (0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, LM.NONE_U32)
AGING_EDGES = (-5, 0, 1, INT32_MAX)
LIMIT_EDGES = (INT32_MIN, -1, 0, 1, INT32_MAX)


def random_sched(rng, n: int, n_stories: int, n_queues: int, edges: bool = True, out_of_range: float = 0.0) -> np.ndarray:
    """sched runs: keys in range (a fraction out_of_range of them past the tables, up to UINT32_MAX), run_phase over every
    code 0..15 and values past 15, priorities and elapsed times at their extremes when edges"""
    s = np.zeros(n, LM.SCHED_RUN_DTYPE)
    s["story_key"] = rng.integers(0, max(n_stories, 1), size=n) if n_stories else rng.integers(0, 4, size=n)
    s["queue_key"] = rng.integers(0, max(n_queues, 1), size=n) if n_queues else rng.integers(0, 4, size=n)
    for f, top in (("story_key", n_stories), ("queue_key", n_queues)):
        oor = rng.random(n) < out_of_range
        s[f][oor] = rng.choice([top, top + 1, top + 1000, 0x7FFFFFFF, 0xFFFFFFFE, 0xFFFFFFFF], size=int(oor.sum()))
    s["priority"] = rng.integers(-3, 8, size=n)
    el = rng.integers(0, 4000, size=n).astype(np.uint32)
    el[rng.random(n) < 0.3] = LM.NONE_U32
    ph = rng.integers(0, 16, size=n).astype(np.uint32)
    if edges:
        e = rng.random(n) < 0.3
        s["priority"][e] = rng.choice(PRIORITY_EDGES, size=int(e.sum()))
        e = rng.random(n) < 0.3
        el[e] = rng.choice(np.array(ELAPSED_EDGES, np.uint32), size=int(e.sum()))
        e = rng.random(n) < 0.1
        ph[e] = rng.choice(np.array([16, 17, 18, 30, 0x12, 0xFFFFFFF2, 0xFFFFFFFF], np.uint32), size=int(e.sum()))
    s["queued_elapsed_s"] = el
    s["run_phase"] = ph
    s["reserved"] = rng.integers(0, 2**32, size=(n, 3), dtype=np.uint64).astype(np.uint32)   # never read
    return s


def random_tables(rng, n_stories: int, n_queues: int, n_runs: int, edges: bool = True, maxprio_base: bool = False) -> dict:
    """limits that leave no slots, some slots and no limit; bases; aging at its extremes when edges"""
    story_limit = rng.choice([0, 0, 1, 3, 40, 200, 1000], size=n_stories).astype(np.int32)
    queue_limit = rng.choice([0, 50, 2000, 20000], size=n_queues).astype(np.int32)
    queue_aging = rng.choice([0, 30, 60, 600], size=n_queues).astype(np.int32)
    global_limit = int(rng.choice([0, 100, 5000, 100000, max(n_runs, 1)]))
    story_base = rng.integers(0, 5, size=n_stories).astype(np.uint32)
    queue_base = rng.integers(0, 50, size=n_queues).astype(np.uint32)
    if edges:
        story_limit[rng.random(n_stories) < 0.2] = rng.choice(LIMIT_EDGES)
        queue_limit[rng.random(n_queues) < 0.2] = rng.choice(LIMIT_EDGES)
        queue_aging[rng.random(n_queues) < 0.4] = rng.choice(AGING_EDGES)
        global_limit = int(rng.choice([global_limit, INT32_MIN, -1, INT32_MAX]))
    t = dict(story_limit=story_limit, queue_limit=queue_limit, queue_aging_s=queue_aging, global_limit=global_limit,
             story_running_base=story_base, queue_running_base=queue_base, global_running_base=int(queue_base.sum()))
    if maxprio_base:
        mb = rng.choice([INT32_MIN, INT32_MIN + 1, -1, 0, 3, INT32_MAX], size=n_queues).astype(np.int32)
        t["queue_max_priority_base"] = mb
    return t
