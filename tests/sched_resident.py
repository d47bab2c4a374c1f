"""Host model of the limiter inputs of resident batches and of bf_resident_schedule (include/bobrafrontier.h, "resident
limiters"), written from the contract and built on tests/schedref.py.

Batch holds one batch's inputs area (SCHED_PUT_DTYPE records without their run field), the schedule records of its last
schedule (None where a run has no baseline) and base_runs, the previous schedule's n_runs.  The lifecycle methods restate
what each resident call does to them.  schedule() limits several batches against one set of totals with schedref.schedule_fast
and returns, per batch, what the device lists."""
from __future__ import annotations

import numpy as np

from bobrapet_b200 import _abi as A
from oracle import limiters as LM
from tests import schedref as SR

NONE = A.SCHED_NONE
PUT_DTYPE = np.dtype([("run", "<u4"), ("story_key", "<u4"), ("queue_key", "<u4"), ("priority", "<i4"), ("queued_since", "<u4"),
                      ("run_phase", "<u4"), ("reserved", "<u4", (2,))])


def defaults(n: int) -> np.ndarray:
    a = np.zeros(n, PUT_DTYPE)
    a["story_key"] = a["queue_key"] = a["queued_since"] = NONE
    return a


def elapsed(since, now: int) -> np.ndarray:
    """queued_elapsed_s from the stored origin: NONE stays NONE, an origin at or past now is 0, else now - since"""
    s = np.asarray(since, np.uint32).astype(np.int64)
    out = np.where(s == NONE, NONE, np.where(now > s, now - s, 0))
    return out.astype(np.uint32)


def sched_runs(inputs: np.ndarray, now: int) -> np.ndarray:
    """the bf_sched_run records bf_schedule would take for these inputs at `now`"""
    s = np.zeros(inputs.shape[0], LM.SCHED_RUN_DTYPE)
    for f in ("story_key", "queue_key", "priority", "run_phase"):
        s[f] = inputs[f]
    s["queued_elapsed_s"] = elapsed(inputs["queued_since"], now)
    return s


class PutRefused(ValueError):
    pass


class Batch:
    def __init__(self, L, capacity: int):
        self.L, self.cap = L, capacity
        self.inputs = defaults(capacity)
        self.rec = [None] * capacity
        self.base_runs = 0

    # -- the calls of the area
    def put(self, req: np.ndarray):
        req = np.asarray(req, PUT_DTYPE)
        if req.shape[0]:
            if (req["run"] >= self.cap).any():
                raise PutRefused("run outside the batch")
            if req["reserved"].any():
                raise PutRefused("reserved fields")
            if np.unique(req["run"]).size != req.shape[0]:
                raise PutRefused("two requests name the same run")
        for q in req:
            self.inputs[int(q["run"])] = q
            self.inputs[int(q["run"])]["run"] = 0

    def download(self, first: int, n: int) -> np.ndarray:
        out = self.inputs[first:first + n].copy()
        out["run"] = np.arange(first, first + n)
        return out

    # -- what the lifecycle calls do
    def lose_baseline(self, runs):
        for r in runs:
            self.rec[int(r)] = None

    def upload(self, first: int, n: int):
        self.lose_baseline(range(first, first + n))

    def retire(self, N: int, gone) -> list:
        """bf_resident_retire's move rule -> [(from, to)]; inputs move with their runs, vacated indices get the defaults"""
        gone = set(int(g) for g in gone)
        m = N - len(gone)
        holes = sorted(g for g in gone if g < m)
        movers = [i for i in range(m, N) if i not in gone]
        moves = list(zip(movers, holes))
        for f, t in moves:
            self.inputs[t] = self.inputs[f]
            self.rec[t] = None
        for i in range(m, N):
            self.inputs[i] = defaults(1)[0]
        self.base_runs = min(self.base_runs, m)
        return moves

    def resize(self, cap: int):
        """a retire to a smaller capacity, or a reshape to a larger one"""
        if cap < self.cap:
            self.inputs, self.rec = self.inputs[:cap].copy(), self.rec[:cap]
        else:
            self.inputs = np.concatenate([self.inputs, defaults(cap - self.cap)])
            self.rec = self.rec + [None] * (cap - self.cap)
        self.cap = cap

    def relayout(self, L):
        """reshape or narrow to layout L: a change of words leaves no baseline"""
        if L.words != self.L.words:
            self.base_runs = 0
        self.L = L

    def receive(self, first: int, inputs: np.ndarray):
        """transfer arrivals at [first, first + len(inputs))"""
        self.inputs[first:first + inputs.shape[0]] = inputs
        self.lose_baseline(range(first, first + inputs.shape[0]))


def schedule(parts, tables: dict, now: int) -> dict:
    """parts: list of (Batch, n_runs, state [n, L.state_stride], result [n, L.result_stride], descs).  The totals and every run's
    record, limited together (masks padded to the widest batch), then each batch's listing against its baselines; the
    baselines become the new records.  -> dict(parts=[dict(records, listed, heads, events, n_events, full)], totals...)"""
    Wmax = max([b.L.words for b, *_ in parts] + [1])
    rr, rd, sc, ready = [], [], [], []
    for b, n, state, result, descs in parts:
        r_, d_ = SR.running_and_demand(b.L, state[:n], descs)
        rr.append(r_); rd.append(d_); sc.append(sched_runs(b.inputs[:n], now))
        m = np.zeros((n, Wmax), np.uint32)
        m[:, :b.L.words] = SR.ready_of(b.L, result[:n])
        ready.append(m)
    sl = np.asarray(tables["story_limit"], np.int32)
    ql = np.asarray(tables["queue_limit"], np.int32)
    sb, qb = tables.get("story_running_base"), tables.get("queue_running_base")
    launch, q_story, q_sched, info, srun, qrun, grun, mp = SR.schedule_fast(
        np.concatenate(rr) if rr else np.zeros(0, np.uint32), np.concatenate(rd) if rd else np.zeros(0, np.uint32),
        np.concatenate(sc) if sc else np.zeros(0, LM.SCHED_RUN_DTYPE), np.concatenate(ready) if ready else np.zeros((0, Wmax), np.uint32),
        sl, np.zeros(sl.size, np.uint32) if sb is None else np.asarray(sb, np.uint32), ql, np.asarray(tables["queue_aging_s"], np.int32),
        np.zeros(ql.size, np.uint32) if qb is None else np.asarray(qb, np.uint32), int(tables.get("global_limit", 0)),
        int(tables.get("global_running_base", 0)), tables.get("queue_max_priority_base"))
    out, at = [], 0
    for b, n, *_ in parts:
        W = b.L.words
        rec = np.zeros((n, A.sched_stride(W)), np.uint8)
        rec[:, 0:16] = info[at:at + n].astype("<u4").view(np.uint8).reshape(n, 16)
        masks = np.concatenate([launch[at:at + n, :W], q_story[at:at + n, :W], q_sched[at:at + n, :W]], axis=1)
        rec[:, 16:16 + 12 * W] = masks.astype("<u4").view(np.uint8).reshape(n, 12 * W)
        listed = [r for r in range(n) if r >= b.base_runs or b.rec[r] is None or not np.array_equal(b.rec[r], rec[r])]
        for r in range(n):
            b.rec[r] = rec[r].copy()
        b.base_runs = n
        heads = info[at:at + n][listed].astype(np.uint32)
        events = [events_of(W, rec[r]) for r in listed]
        ev = np.concatenate(events) if events else np.zeros(0, np.uint16)
        out.append({"records": rec, "listed": np.asarray(listed, np.uint32), "heads": heads, "events": ev, "n_events": int(ev.size),
                    "full": int(len(listed) == n)})
        at += n
    return {"parts": out, "story_running": (srun % (1 << 32)).astype(np.uint32), "queue_running": (qrun % (1 << 32)).astype(np.uint32),
            "queue_max_priority": mp.astype(np.int32), "global_running": grun % (1 << 32)}


def events_of(W: int, rec: np.ndarray) -> np.ndarray:
    """the events of one schedule record: step | kind << 10, step-ascending"""
    m = np.ascontiguousarray(rec[16:16 + 12 * W]).view("<u4").reshape(3, W)
    out = []
    for w in range(W):
        for b in range(32):
            for k, kind in enumerate((A.SEVT_LAUNCH, A.SEVT_QUEUED_STORY, A.SEVT_QUEUED_SCHED)):
                if (int(m[k, w]) >> b) & 1:
                    out.append((32 * w + b) | kind << 10)
    return np.asarray(out, np.uint16)


def decode(W: int, n: int, runs, heads, events) -> np.ndarray:
    """schedule records of runs [0, n) rebuilt from a listing that names every run (full = 1)"""
    rec = np.zeros((n, A.sched_stride(W)), np.uint8)
    h = np.asarray(heads)
    hv = np.stack([h[f] for f in h.dtype.names], axis=1) if h.dtype.names else h
    rec[np.asarray(runs, np.int64), 0:16] = hv.astype("<u4").view(np.uint8).reshape(-1, 16)
    masks = np.zeros((n, 3, W), np.uint32)
    at = 0
    for i, r in enumerate(np.asarray(runs, np.int64)):
        k = int(hv[i, 0] + hv[i, 1] + hv[i, 2])
        for e in np.asarray(events[at:at + k], np.uint32):
            step, kind = int(e & 0x3FF), int(e >> 10)
            masks[r, {1: 0, 2: 1, 4: 2}[kind], step >> 5] |= np.uint32(1 << (step & 31))
        at += k
    rec[:, 16:16 + 12 * W] = masks.reshape(n, 3 * W).astype("<u4").view(np.uint8)
    return rec
