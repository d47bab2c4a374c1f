"""Frontier — thin Python handle over the C ABI (include/bobrafrontier.h).

This is the call a user of the Python binding makes; it is the same call path the
cgo shim uses (go/frontier/frontier.go): bf_create -> bf_topology_put_many ->
bf_eval / bf_eval_device.  There is no CPU path here: without the CUDA library or
without an H100 the constructor raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _abi as A
from .records import EXP_DTYPE, PAR_DTYPE, TOPO_DTYPE


class TopologySet:
    """`count` topologies held as concatenated numpy arrays (keeps them alive for the C call).

    S, E, P : [count] uint32; row_ptr: concatenation of (S[i]+1) uint32 each; col_idx uint16;
    step_flags uint8; parallel PAR_DTYPE; allow_bits uint8 (bit arrays, one shared pool)."""

    def __init__(self, S, E, row_ptr, col_idx, step_flags, P=None, parallel=None, allow_bits=None):
        self.S = np.ascontiguousarray(S, dtype=np.uint32)
        self.E = np.ascontiguousarray(E, dtype=np.uint32)
        self.count = int(self.S.shape[0])
        self.row_ptr = np.ascontiguousarray(row_ptr, dtype=np.uint32)
        self.col_idx = np.ascontiguousarray(col_idx, dtype=np.uint16)
        self.step_flags = np.ascontiguousarray(step_flags, dtype=np.uint8)
        self.P = np.zeros(self.count, dtype=np.uint32) if P is None else np.ascontiguousarray(P, dtype=np.uint32)
        self.parallel = np.zeros(0, dtype=PAR_DTYPE) if parallel is None else np.ascontiguousarray(parallel, dtype=PAR_DTYPE)
        self.allow_bits = np.zeros(0, dtype=np.uint8) if allow_bits is None else np.ascontiguousarray(allow_bits, dtype=np.uint8)
        assert self.row_ptr.shape[0] == int(self.S.sum()) + self.count
        assert self.col_idx.shape[0] == int(self.E.sum())
        assert self.step_flags.shape[0] == int(self.S.sum())
        assert self.parallel.shape[0] == int(self.P.sum())

    def descriptors(self) -> np.ndarray:
        """Array of bf_topology structs pointing into the concatenated arrays."""
        t = np.zeros(self.count, dtype=TOPO_DTYPE)
        S64, E64, P64 = self.S.astype(np.uint64), self.E.astype(np.uint64), self.P.astype(np.uint64)
        rp_off = np.concatenate(([0], np.cumsum(S64 + 1)[:-1])).astype(np.uint64)
        ci_off = np.concatenate(([0], np.cumsum(E64)[:-1])).astype(np.uint64)
        sf_off = np.concatenate(([0], np.cumsum(S64)[:-1])).astype(np.uint64)
        pd_off = np.concatenate(([0], np.cumsum(P64)[:-1])).astype(np.uint64)
        t["n_steps"], t["n_edges"], t["n_parallel"] = self.S, self.E, self.P
        t["row_ptr"] = np.uint64(self.row_ptr.ctypes.data) + rp_off * np.uint64(4)
        t["col_idx"] = np.uint64(self.col_idx.ctypes.data if self.col_idx.size else 0) + ci_off * np.uint64(2)
        t["step_flags"] = np.uint64(self.step_flags.ctypes.data) + sf_off
        if self.parallel.size:
            t["parallel"] = np.uint64(self.parallel.ctypes.data) + pd_off * np.uint64(PAR_DTYPE.itemsize)
        if self.allow_bits.size:
            t["branch_allow_bits"] = np.uint64(self.allow_bits.ctypes.data)
            t["n_branch_allow_bits"] = np.uint32(self.allow_bits.size * 8)
        return t

    def algorithmic_bytes(self) -> int:
        """Canonical topology bytes, SURVEY.md 8(d): 2(S+1) + 2E + S per topology."""
        return int((2 * (self.S.astype(np.int64) + 1) + 2 * self.E.astype(np.int64) + self.S.astype(np.int64)).sum())


class Frontier:
    def __init__(self, device: int = 0, arena_bytes: int = 0, _borrowed_ctx=None, reserve_sms: int = 0):
        self._lib = A.load()
        self._owned = _borrowed_ctx is None
        self._steps_max: Dict[int, int] = {}   # steps_max of each resident batch's layout
        self._child_nibbles: Dict[int, int] = {}   # and its child_nibbles
        self._timer_k: Dict[int, int] = {}   # slots per run of each resident batch's timer area (resident_timers)
        if _borrowed_ctx is not None:       # a shard's ctx owned by a FrontierGroup
            self._ctx = C.c_void_p(_borrowed_ctx)
            return
        self._ctx = C.c_void_p()
        cfg = A.Config(struct_size=C.sizeof(A.Config), device=device, arena_bytes=arena_bytes, max_topologies=0,
                       flags=(reserve_sms & 0xFF))   # BF_CFG_RESERVE_SMS: SMs left to other streams' kernels (the count all-gather)
        rc = self._lib.bf_create(C.byref(self._ctx), C.byref(cfg))
        if rc != A.BF_OK:
            self._ctx = None
            raise A.FrontierError(rc, "bf_create(device=%d): no CUDA fallback exists for this path" % device)

    # -- lifecycle
    def close(self):
        if getattr(self, "_ctx", None):
            if self._owned:
                self._lib.bf_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc != A.BF_OK:
            raise A.FrontierError(rc, "%s: %s" % (what, self._lib.bf_last_error(self._ctx).decode()))

    # -- topologies
    def put_topologies(self, ts: TopologySet) -> np.ndarray:
        desc = ts.descriptors()
        slots = np.zeros(ts.count, dtype=np.uint32)
        rc = self._lib.bf_topology_put_many(self._ctx, desc.ctypes.data_as(C.POINTER(A.Topology)), ts.count,
                                            slots.ctypes.data_as(C.POINTER(C.c_uint32)))
        self._check(rc, "bf_topology_put_many")
        return slots

    def put_topologies_checked_on_device(self, ts: TopologySet):
        """Bulk upload with acyclicity checked by the device kernel -> (slots, status words)."""
        desc = ts.descriptors()
        slots = np.zeros(ts.count, dtype=np.uint32)
        status = np.zeros(ts.count, dtype=np.uint32)
        rc = self._lib.bf_topology_put_many_checked_on_device(
            self._ctx, desc.ctypes.data_as(C.POINTER(A.Topology)), ts.count, slots.ctypes.data_as(C.POINTER(C.c_uint32)),
            status.ctypes.data_as(C.POINTER(C.c_uint32)))
        self._check(rc, "bf_topology_put_many_checked_on_device")
        return slots, status

    def check_topologies(self, slots) -> np.ndarray:
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        status = np.zeros(slots.shape[0], dtype=np.uint32)
        self._check(self._lib.bf_topology_check(self._ctx, slots.ctypes.data_as(C.POINTER(C.c_uint32)), slots.shape[0],
                                                status.ctypes.data_as(C.POINTER(C.c_uint32))), "bf_topology_check")
        return status

    def drop_topology(self, slot: int):
        self._check(self._lib.bf_topology_drop(self._ctx, int(slot)), "bf_topology_drop")

    TIMING_DTYPE = np.dtype([("step", "<u2"), ("code", "u1"), ("reserved", "u1"), ("delay", "<u4")])   # bf_step_timing, 8 B

    def put_timings(self, slot: int, entries=None):
        """bf_topology_timings: replace the step timings of a live slot (TIMING_DTYPE or (step, code, delay) tuples; none clears
        them).  A timed resident_commit arms the launched sleep, gate and wait steps that have one."""
        ents = np.zeros(0, dtype=self.TIMING_DTYPE) if entries is None else entries
        if not isinstance(ents, np.ndarray):
            ents = np.array([(int(s), int(c), 0, int(d)) for s, c, d in ents], dtype=self.TIMING_DTYPE)
        ents = np.ascontiguousarray(ents, dtype=self.TIMING_DTYPE)
        self._check(self._lib.bf_topology_timings(self._ctx, int(slot), ents.ctypes.data if ents.shape[0] else None, ents.shape[0]),
                    "bf_topology_timings")

    def child_first(self, slot: int) -> np.ndarray:
        out = np.zeros(A.MAX_PARALLEL, dtype=np.uint32)
        n = self._lib.bf_topology_child_first(self._ctx, int(slot), out.ctypes.data_as(C.POINTER(C.c_uint32)), A.MAX_PARALLEL)
        if n < 0:
            raise A.FrontierError(n, "bf_topology_child_first")
        return out[:n]

    def topology_record(self, slot: int):
        addr, nbytes = C.c_uint64(), C.c_uint32()
        self._check(self._lib.bf_topology_record(self._ctx, int(slot), C.byref(addr), C.byref(nbytes)), "bf_topology_record")
        return addr.value, nbytes.value

    # -- evaluation over HOST buffers (H2D + kernels + D2H inside the call)
    def eval(self, L: A.Layout, state: np.ndarray, result: Optional[np.ndarray] = None, flags: int = 0,
             max_iterations: int = 0, expansion_cap: int = 0):
        n = int(state.shape[0])
        assert state.dtype == np.uint8 and state.flags["C_CONTIGUOUS"] and state.shape[1] == L.state_stride
        if result is None:
            result = np.zeros((n, L.result_stride), dtype=np.uint8)
        counts = A.Counts()
        exp = np.zeros(max(expansion_cap, 1), dtype=EXP_DTYPE) if (flags & A.EVAL_EXPANSION) else None
        b = A.Batch(struct_size=C.sizeof(A.Batch), n_runs=n, flags=flags, max_iterations=max_iterations, layout=L,
                    state=state.ctypes.data, result=result.ctypes.data,
                    expansion=(exp.ctypes.data if exp is not None else None),
                    expansion_cap=(expansion_cap if exp is not None else 0),
                    counts=C.addressof(counts))
        self._check(self._lib.bf_eval(self._ctx, C.byref(b)), "bf_eval")
        cdict = {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}
        if exp is not None:
            return result, cdict, exp[:min(int(counts.expansion), expansion_cap)]
        return result, cdict




    # -- compact results: one head word per run + 16-bit (step | kind << 10) events instead of mask records
    def _compact_out(self, n_runs: int, events_cap: int, head, events):
        if head is None:
            head = np.zeros(max(n_runs, 1), dtype=np.uint32)
        if events is None:
            events = np.zeros(max(events_cap, 1), dtype=np.uint16)
        assert head.dtype == np.uint32 and head.flags["C_CONTIGUOUS"] and head.shape[0] >= n_runs
        assert events.dtype == np.uint16 and events.flags["C_CONTIGUOUS"] and events.shape[0] >= events_cap
        co = A.CompactOut(struct_size=C.sizeof(A.CompactOut), head=head.ctypes.data, events=events.ctypes.data,
                          events_cap=events_cap, n_events=0)
        return co, head, events

    def eval_compact(self, L: A.Layout, state: np.ndarray, events_cap: int, flags: int = 0, max_iterations: int = 0,
                     head: Optional[np.ndarray] = None, events: Optional[np.ndarray] = None):
        """bf_eval_compact -> (head [n] uint32, events[:min(n_events, cap)] uint16, n_events, counts)"""
        n = int(state.shape[0])
        assert state.dtype == np.uint8 and state.flags["C_CONTIGUOUS"] and state.shape[1] == L.state_stride
        co, head, events = self._compact_out(n, events_cap, head, events)
        counts = A.Counts()
        b = A.Batch(struct_size=C.sizeof(A.Batch), n_runs=n, flags=flags, max_iterations=max_iterations, layout=L,
                    state=state.ctypes.data, result=None, expansion=None, expansion_cap=0, counts=C.addressof(counts))
        self._check(self._lib.bf_eval_compact(self._ctx, C.byref(b), C.byref(co)), "bf_eval_compact")
        cdict = {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}
        return head[:n], events[:min(int(co.n_events), events_cap)], int(co.n_events), cdict

    def resident_tick_compact(self, handle: int, n_runs: int, deltas: np.ndarray, events_cap: int, flags: int = 0,
                              max_iterations: int = 0, head: Optional[np.ndarray] = None, events: Optional[np.ndarray] = None):
        """bf_resident_tick_compact -> (head, events, n_events, counts, n_listed); flags may carry A.EVAL_CHANGED_ONLY"""
        assert deltas.dtype == self.DELTA_DTYPE and deltas.flags["C_CONTIGUOUS"]
        co, head, events = self._compact_out(n_runs, events_cap, head, events)
        counts = A.Counts()
        self._check(self._lib.bf_resident_tick_compact(self._ctx, handle, deltas.ctypes.data, deltas.shape[0], n_runs, flags,
                                                       max_iterations, C.byref(co), C.byref(counts)), "bf_resident_tick_compact")
        cdict = {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}
        return head[:n_runs], events[:min(int(co.n_events), events_cap)], int(co.n_events), cdict, int(co.n_listed)

    def resident_tick_touched(self, handle: int, n_runs: int, deltas: np.ndarray, runs_cap: int, events_cap: int, flags: int = 0,
                              max_iterations: int = 0, runs: Optional[np.ndarray] = None, head: Optional[np.ndarray] = None,
                              events: Optional[np.ndarray] = None):
        """bf_resident_tick_touched: evaluate and list only the runs touched since they were last evaluated.
        -> dict(full, runs, head, events, n_listed, n_evaluated, n_events, counts); runs / head hold the first
        min(n_listed, runs_cap) entries, events the first min(n_events, events_cap)."""
        assert deltas.dtype == self.DELTA_DTYPE and deltas.flags["C_CONTIGUOUS"]
        if runs is None:
            runs = np.zeros(max(runs_cap, 1), dtype=np.uint32)
        if head is None:
            head = np.zeros(max(runs_cap, 1), dtype=np.uint32)
        if events is None:
            events = np.zeros(max(events_cap, 1), dtype=np.uint16)
        for a, dt, n in ((runs, np.uint32, runs_cap), (head, np.uint32, runs_cap), (events, np.uint16, events_cap)):
            assert a.dtype == dt and a.flags["C_CONTIGUOUS"] and a.shape[0] >= n
        to = A.TouchedOut(struct_size=C.sizeof(A.TouchedOut), runs=runs.ctypes.data, head=head.ctypes.data, runs_cap=runs_cap,
                          events=events.ctypes.data, events_cap=events_cap)
        counts = A.Counts()
        self._check(self._lib.bf_resident_tick_touched(self._ctx, handle, deltas.ctypes.data, deltas.shape[0], n_runs, flags,
                                                       max_iterations, C.byref(to), C.byref(counts)), "bf_resident_tick_touched")
        nl = min(int(to.n_listed), runs_cap)
        return {"full": int(to.full), "runs": runs[:nl], "head": head[:nl], "events": events[:min(int(to.n_events), events_cap)],
                "n_listed": int(to.n_listed), "n_evaluated": int(to.n_evaluated), "n_events": int(to.n_events),
                "counts": {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}}

    def resident_tick_touched_many(self, parts, flags: int = 0, max_iterations: int = 0):
        """bf_resident_tick_touched_many: the touched ticks of several resident batches of this ctx in one call and one
        synchronisation.  Each part is a dict with handle, n_runs, deltas, runs_cap and events_cap, and optionally runs / head /
        events buffers (as resident_tick_touched takes them) and counts=False (pass no counts block).  -> one dict per part,
        shaped as resident_tick_touched returns it (counts None without a counts block).  A refusal or failure raises
        FrontierError with .bad_part set: the part it names, or A.COMMIT_NONE."""
        n = len(parts)
        cparts = (A.TickPart * max(n, 1))()
        keep = []
        for k, p in enumerate(parts):
            deltas = p["deltas"]
            assert deltas.dtype == self.DELTA_DTYPE and deltas.flags["C_CONTIGUOUS"]
            runs_cap, events_cap = p["runs_cap"], p["events_cap"]
            runs, head, events = p.get("runs"), p.get("head"), p.get("events")
            if runs is None:
                runs = np.zeros(max(runs_cap, 1), dtype=np.uint32)
            if head is None:
                head = np.zeros(max(runs_cap, 1), dtype=np.uint32)
            if events is None:
                events = np.zeros(max(events_cap, 1), dtype=np.uint16)
            for a, dt, m in ((runs, np.uint32, runs_cap), (head, np.uint32, runs_cap), (events, np.uint16, events_cap)):
                assert a.dtype == dt and a.flags["C_CONTIGUOUS"] and a.shape[0] >= m
            to = A.TouchedOut(struct_size=C.sizeof(A.TouchedOut), runs=runs.ctypes.data, head=head.ctypes.data, runs_cap=runs_cap,
                              events=events.ctypes.data, events_cap=events_cap)
            counts = A.Counts() if p.get("counts", True) else None
            cparts[k] = A.TickPart(struct_size=C.sizeof(A.TickPart), handle=p["handle"], deltas=deltas.ctypes.data,
                                   n_deltas=deltas.shape[0], n_runs=p["n_runs"], out=C.addressof(to),
                                   counts=(C.addressof(counts) if counts is not None else None))
            keep.append((to, counts, runs, head, events, runs_cap, events_cap))
        bad = C.c_uint32(0)
        rc = self._lib.bf_resident_tick_touched_many(self._ctx, flags, max_iterations, cparts, n, C.byref(bad))
        if rc != A.BF_OK:
            err = A.FrontierError(rc, "bf_resident_tick_touched_many: %s" % self._lib.bf_last_error(self._ctx).decode())
            err.bad_part = bad.value
            raise err
        res = []
        for to, counts, runs, head, events, runs_cap, events_cap in keep:
            nl = min(int(to.n_listed), runs_cap)
            res.append({"full": int(to.full), "runs": runs[:nl], "head": head[:nl], "events": events[:min(int(to.n_events), events_cap)],
                        "n_listed": int(to.n_listed), "n_evaluated": int(to.n_evaluated), "n_events": int(to.n_events),
                        "counts": None if counts is None else
                        {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}})
        return res

    def resident_migrate(self, handle: int, old_slot: int, new_slot: int, step_map, n_runs: int) -> int:
        """bf_resident_migrate: move the runs in [0, n_runs) on old_slot to new_slot (an edited Story), re-indexing their step
        state in place.  step_map[i] = new index of old step i, or A.MIGRATE_GONE.  -> number of runs migrated."""
        sm = np.ascontiguousarray(step_map, dtype=np.uint16)
        m = A.Migration(struct_size=C.sizeof(A.Migration), old_slot=int(old_slot), new_slot=int(new_slot), n_runs=int(n_runs),
                        step_map=sm.ctypes.data, n_old_steps=sm.shape[0])
        self._check(self._lib.bf_resident_migrate(self._ctx, handle, C.byref(m)), "bf_resident_migrate")
        return int(m.migrated)

    REDRIVE_DTYPE = np.dtype([("run", "<u4"), ("slot", "<u4"), ("step", "<u4"), ("reserved", "<u4")])

    def resident_redrive(self, handle: int, requests: np.ndarray):
        """bf_resident_redrive: reset, in place, the step set of each request (run, slot, step or A.REDRIVE_ALL) in the records of
        the runs that hold the request's slot.  -> (status [n] uint8: 1 = applied, 0 = the run holds another slot; applied)"""
        rq = np.ascontiguousarray(requests, dtype=self.REDRIVE_DTYPE)
        status = np.zeros(max(rq.shape[0], 1), dtype=np.uint8)
        applied = C.c_uint32()
        self._check(self._lib.bf_resident_redrive(self._ctx, handle, rq.ctypes.data, rq.shape[0], status.ctypes.data,
                                                  C.byref(applied)), "bf_resident_redrive")
        return status[:rq.shape[0]], int(applied.value)

    def resident_reshape(self, handle: int, L: A.Layout, capacity: int):
        """bf_resident_reshape: grow the batch to layout L (from make_layout) and `capacity` runs in place, keeping every run's
        state, the current result records and the touch marks"""
        self._check(self._lib.bf_resident_reshape(self._ctx, handle, C.byref(L), capacity), "bf_resident_reshape")
        self._steps_max[handle] = int(L.steps_max)
        self._child_nibbles[handle] = int(L.child_nibbles)

    def resident_retire(self, handle: int, n_runs: int, runs, capacity: int = 0):
        """bf_resident_retire: take `runs` (distinct indices below n_runs) out of the batch; the last live runs move into the
        freed indices.  capacity 0 keeps the capacity, else it becomes `capacity` (n_runs - len(runs) <= capacity <= current).
        -> (new n_runs, moves_from, moves_to): run moves_from[i] now lives at moves_to[i], ascending by target"""
        rs = np.ascontiguousarray(runs, dtype=np.uint32)
        n = rs.shape[0]
        mf = np.zeros(max(n, 1), dtype=np.uint32)
        mt = np.zeros(max(n, 1), dtype=np.uint32)
        rt = A.Retire(struct_size=C.sizeof(A.Retire), n_runs=int(n_runs), runs=rs.ctypes.data if n else None, n=n,
                      capacity=int(capacity), moves_from=mf.ctypes.data, moves_to=mt.ctypes.data)
        self._check(self._lib.bf_resident_retire(self._ctx, handle, C.byref(rt)), "bf_resident_retire")
        return int(rt.n_runs), mf[:rt.n_moves].copy(), mt[:rt.n_moves].copy()

    def resident_extent(self, handle: int, n_runs: int) -> dict:
        """bf_resident_extent: the smallest layout the batch's runs [0, n_runs) and records allow -> dict(steps_max, child_nibbles,
        fields, widest_run)"""
        e = A.Extent(struct_size=C.sizeof(A.Extent), n_runs=int(n_runs))
        self._check(self._lib.bf_resident_extent(self._ctx, handle, C.byref(e)), "bf_resident_extent")
        return e.as_dict()

    def resident_narrow(self, handle: int, L: A.Layout, n_runs: int) -> dict:
        """bf_resident_narrow: re-lay the batch at the smaller layout L (from make_layout) in place when its runs [0, n_runs) and
        records allow it -> the extent (dict as resident_extent).  A rejection raises FrontierError with the extent as .extent"""
        e = A.Extent(struct_size=C.sizeof(A.Extent), n_runs=int(n_runs))
        rc = self._lib.bf_resident_narrow(self._ctx, handle, C.byref(L), C.byref(e))
        if rc != A.BF_OK:
            err = A.FrontierError(rc, "bf_resident_narrow: %s" % self._lib.bf_last_error(self._ctx).decode())
            err.extent = e.as_dict()
            raise err
        self._steps_max[handle] = int(L.steps_max)
        self._child_nibbles[handle] = int(L.child_nibbles)
        return e.as_dict()

    def resident_transfer(self, src: int, dst: int, src_n: int, dst_n: int, runs) -> dict:
        """bf_resident_transfer: move `runs` (distinct indices below src_n) of batch src to the end of batch dst's runs [0, dst_n),
        re-laid at dst's layout; src compacts as after resident_retire.  -> dict(src_n_runs, dst_n_runs, moves_from, moves_to).
        A refusal raises FrontierError with .unfit (position in runs of the first run dst cannot hold, or A.EXTENT_NO_RUN) and
        .why (that run's extent, as resident_extent's dict)"""
        rs = np.ascontiguousarray(runs, dtype=np.uint32)
        n = rs.shape[0]
        mf = np.zeros(max(n, 1), dtype=np.uint32)
        mt = np.zeros(max(n, 1), dtype=np.uint32)
        t = A.Transfer(struct_size=C.sizeof(A.Transfer), src_n_runs=int(src_n), dst_n_runs=int(dst_n), runs=rs.ctypes.data if n else None,
                       n=n, moves_from=mf.ctypes.data, moves_to=mt.ctypes.data)
        rc = self._lib.bf_resident_transfer(self._ctx, src, dst, C.byref(t))
        if rc != A.BF_OK:
            err = A.FrontierError(rc, "bf_resident_transfer: %s" % self._lib.bf_last_error(self._ctx).decode())
            err.unfit = int(t.unfit)
            err.why = t.why.as_dict()
            raise err
        return {"src_n_runs": int(t.src_n_runs), "dst_n_runs": int(t.dst_n_runs), "moves_from": mf[:t.n_moves].copy(),
                "moves_to": mt[:t.n_moves].copy()}

    def resident_transfer_ctx(self, dst_frontier: "Frontier", src: int, dst: int, src_n: int, dst_n: int, runs, slot_map) -> dict:
        """bf_resident_transfer_ctx: resident_transfer from batch src of this ctx to batch dst of dst_frontier's ctx (another
        device, or another ctx of the same one).  slot_map[s] is the destination slot of this ctx's slot s, or A.SLOT_NONE.
        -> dict(src_n_runs, dst_n_runs, moves_from, moves_to).  A refusal raises FrontierError with .unfit, .unfit_reason
        (A.UNFIT_*) and .why"""
        rs = np.ascontiguousarray(runs, dtype=np.uint32)
        sm = np.ascontiguousarray(slot_map, dtype=np.uint32)
        n = rs.shape[0]
        mf = np.zeros(max(n, 1), dtype=np.uint32)
        mt = np.zeros(max(n, 1), dtype=np.uint32)
        t = A.CtxTransfer(struct_size=C.sizeof(A.CtxTransfer), src_n_runs=int(src_n), dst_n_runs=int(dst_n),
                          runs=rs.ctypes.data if n else None, n=n, slot_map=sm.ctypes.data if sm.size else None, n_slot_map=sm.size,
                          moves_from=mf.ctypes.data, moves_to=mt.ctypes.data)
        rc = self._lib.bf_resident_transfer_ctx(self._ctx, src, dst_frontier._ctx, dst, C.byref(t))
        if rc != A.BF_OK:
            err = A.FrontierError(rc, "bf_resident_transfer_ctx: %s" % self._lib.bf_last_error(self._ctx).decode())
            err.unfit = int(t.unfit)
            err.unfit_reason = int(t.unfit_reason)
            err.why = t.why.as_dict()
            raise err
        return {"src_n_runs": int(t.src_n_runs), "dst_n_runs": int(t.dst_n_runs), "moves_from": mf[:t.n_moves].copy(),
                "moves_to": mt[:t.n_moves].copy()}

    # -- step timers of a resident batch (bf_resident_timers*, bf_resident_fire)
    TIMER_DTYPE = np.dtype([("run", "<u4"), ("step", "<u2"), ("code", "u1"), ("reserved", "u1"), ("deadline", "<u4"),
                            ("reserved2", "<u4")])                                             # bf_timer, 16 B
    SLOT_DTYPE = np.dtype([("deadline", "<u4"), ("step", "<u2"), ("code", "u1"), ("reserved", "u1")])   # bf_timer_slot, 8 B
    FIRED_DTYPE = np.dtype([("run", "<u4"), ("step", "<u2"), ("code", "u1"), ("written", "u1")])         # bf_fired, 8 B

    def resident_timers(self, handle: int, slots_per_run: int):
        """bf_resident_timers: create the batch's timer area with K = slots_per_run slots per run, or grow K keeping every slot"""
        self._check(self._lib.bf_resident_timers(self._ctx, handle, int(slots_per_run)), "bf_resident_timers")
        self._timer_k[handle] = int(slots_per_run)   # the row width resident_resync_areas checks its timers against

    def resident_timers_arm(self, handle: int, requests: np.ndarray):
        """bf_resident_timers_arm: arm (or replace) the timer of each (run, step); deadline A.TIMER_NONE cancels it.
        requests: TIMER_DTYPE, at most one per (run, step)"""
        rq = np.ascontiguousarray(requests, dtype=self.TIMER_DTYPE)
        self._check(self._lib.bf_resident_timers_arm(self._ctx, handle, rq.ctypes.data if rq.shape[0] else None, rq.shape[0]),
                    "bf_resident_timers_arm")

    def resident_fire(self, handle: int, n_runs: int, now: int, fired_cap: Optional[int] = None,
                      fired: Optional[np.ndarray] = None) -> dict:
        """bf_resident_fire: fire the due timers of runs [0, n_runs) at `now` -> dict(n_fired, n_written, n_pruned,
        next_deadline, fired); fired (FIRED_DTYPE) holds the first min(n_fired, fired_cap) entries, ascending by run and step"""
        if fired is None:
            fired = np.zeros(max(fired_cap if fired_cap is not None else 4096, 1), dtype=self.FIRED_DTYPE)
        cap = fired.shape[0] if fired_cap is None else fired_cap
        assert fired.dtype == self.FIRED_DTYPE and fired.flags["C_CONTIGUOUS"] and fired.shape[0] >= cap
        fo = A.FireOut(struct_size=C.sizeof(A.FireOut), n_runs=int(n_runs), fired=fired.ctypes.data, fired_cap=cap)
        self._check(self._lib.bf_resident_fire(self._ctx, handle, int(now), C.byref(fo)), "bf_resident_fire")
        return {"n_fired": int(fo.n_fired), "n_written": int(fo.n_written), "n_pruned": int(fo.n_pruned),
                "next_deadline": int(fo.next_deadline), "fired": fired[:min(int(fo.n_fired), cap)].copy()}

    def resident_timers_download(self, handle: int, first_run: int, n_runs: int, slots_per_run: int) -> np.ndarray:
        """bf_resident_timers_download -> the raw slots, SLOT_DTYPE array of shape (n_runs, slots_per_run)"""
        out = np.zeros((n_runs, slots_per_run), dtype=self.SLOT_DTYPE)
        self._check(self._lib.bf_resident_timers_download(self._ctx, handle, first_run, n_runs, out.ctypes.data),
                    "bf_resident_timers_download")
        return out

    # -- StoryRun stops and deadlines of a resident batch (bf_resident_runctl*; bf_resident_fire reports the deadlines)
    RUNCTL_DTYPE = np.dtype([("story_deadline", "<u4"), ("drain_deadline", "<u4"), ("stop", "u1"), ("saved_flags", "u1"),
                             ("reserved", "u1", (6,))])                                        # bf_run_ctl, 16 B
    RUNCTL_PUT_DTYPE = np.dtype([("run", "<u4"), ("story_deadline", "<u4"), ("drain_deadline", "<u4"), ("stop", "u1"),
                                 ("reserved", "u1", (3,))])                                    # bf_run_ctl_put, 16 B

    def resident_runctl(self, handle: int):
        """bf_resident_runctl: create the batch's run-control area, every run at the default (no deadline, not stopped)"""
        self._check(self._lib.bf_resident_runctl(self._ctx, handle), "bf_resident_runctl")

    def resident_runctl_put(self, handle: int, requests: np.ndarray):
        """bf_resident_runctl_put: write both deadlines of each requests[i].run and stop it when stop != A.STOP_NONE
        (RUNCTL_PUT_DTYPE, at most one per run)"""
        rq = np.ascontiguousarray(requests, dtype=self.RUNCTL_PUT_DTYPE)
        self._check(self._lib.bf_resident_runctl_put(self._ctx, handle, rq.ctypes.data if rq.shape[0] else None, rq.shape[0]),
                    "bf_resident_runctl_put")

    def resident_runctl_download(self, handle: int, first_run: int, n_runs: int) -> np.ndarray:
        """bf_resident_runctl_download -> the records of runs [first_run, first_run + n_runs), RUNCTL_DTYPE"""
        out = np.zeros(n_runs, dtype=self.RUNCTL_DTYPE)
        self._check(self._lib.bf_resident_runctl_download(self._ctx, handle, first_run, n_runs, out.ctypes.data),
                    "bf_resident_runctl_download")
        return out

    # -- tick commits of a resident batch (bf_resident_commit)
    COMMIT_DTYPE = np.dtype([("run", "<u4"), ("step", "<u2"), ("kind", "u1"), ("code", "u1")])   # bf_commit_entry, 8 B

    COMMIT_WRITE_DTYPE = np.dtype([("run", "<u4"), ("index", "<u2"), ("field", "u1"), ("code", "u1"), ("before", "<u4"),
                                   ("after", "<u4")])   # bf_commit_write, 16 B

    def resident_commit_marks(self, handle: int) -> None:
        """bf_resident_commit_marks: enable the batch's commit-due bits (every run due), which resident_commit(touched=True)
        needs"""
        self._check(self._lib.bf_resident_commit_marks(self._ctx, handle), "bf_resident_commit_marks")

    def resident_commit(self, handle: int, n_runs: int, entries=None, now: Optional[int] = None,
                        journal_cap: Optional[int] = None, rewrites: bool = False, touched: bool = False) -> dict:
        """bf_resident_commit: write the skips, launches and queue marks of the last tick (and schedule) of runs [0, n_runs)
        into the state records.  entries: COMMIT_DTYPE (or (run, step, kind, code) tuples), at most one per (run, step).
        With `now` (bf_resident_commit_timed) the launched sleep, gate and wait steps with a timing (put_timings) are armed too.
        With journal_cap (bf_resident_commit_journal) the call also lists what it wrote, up to journal_cap items.
        With rewrites (bf_resident_commit_rewrites; needs journal_cap) the writes start from the codes after a single pass's
        stages G, H and I, so that the sleeps, gates, waits, joins and fail-fast skips that pass rewrote are stored and listed
        (PHASE items with code A.COMMIT_WRITE_REWRITE), and the result also holds n_rewritten.
        -> dict(n_runs_written, n_skipped, n_launched, n_queued, n_failed), with `now` also n_armed and next_deadline, with
        journal_cap also items (COMMIT_WRITE_DTYPE[min(n_items, journal_cap)]), n_items, runs (u32, the runs whose record
        changed) and n_runs_listed.  A refusal raises FrontierError with .bad_run and .bad_step (A.COMMIT_NONE for a refusal
        of the whole call).  With touched (bf_resident_commit_touched; needs resident_commit_marks) the same form considers only
        the runs whose writes may not be in place, with the same results, and the dict also holds full and n_considered"""
        ents = np.zeros(0, dtype=self.COMMIT_DTYPE) if entries is None else entries
        if not isinstance(ents, np.ndarray):
            ents = np.array([tuple(e) for e in ents], dtype=self.COMMIT_DTYPE)
        ents = np.ascontiguousarray(ents, dtype=self.COMMIT_DTYPE)
        if rewrites and journal_cap is None:
            raise ValueError("resident_commit(rewrites=True) needs journal_cap: the rewrites are persisted from the journal")
        out = A.CommitOut(struct_size=C.sizeof(A.CommitOut))
        n_rw = C.c_uint32(0)
        ep = ents.ctypes.data if ents.shape[0] else None
        arm = None if now is None else A.CommitArm(struct_size=C.sizeof(A.CommitArm), now=int(now))
        scope = A.CommitScope(struct_size=C.sizeof(A.CommitScope), flags=A.COMMIT_SCOPE_REWRITES if rewrites else 0)
        j = None
        if journal_cap is not None:
            items = np.zeros(max(int(journal_cap), 1), dtype=self.COMMIT_WRITE_DTYPE)
            runs = np.zeros(max(int(n_runs), 1), dtype=np.uint32)
            j = A.CommitJournal(struct_size=C.sizeof(A.CommitJournal), items=items.ctypes.data if journal_cap else None,
                                items_cap=int(journal_cap), runs=runs.ctypes.data if n_runs else None, runs_cap=int(n_runs))
        a = None if arm is None else C.byref(arm)
        if touched:
            rc = self._lib.bf_resident_commit_touched(self._ctx, handle, int(n_runs), ep, ents.shape[0], C.byref(out), a,
                                                      None if j is None else C.byref(j), C.byref(n_rw) if rewrites else None,
                                                      C.byref(scope))
        elif rewrites:
            rc = self._lib.bf_resident_commit_rewrites(self._ctx, handle, int(n_runs), ep, ents.shape[0], C.byref(out), a,
                                                       C.byref(j), C.byref(n_rw))
        elif j is not None:
            rc = self._lib.bf_resident_commit_journal(self._ctx, handle, int(n_runs), ep, ents.shape[0], C.byref(out), a,
                                                      C.byref(j))
        elif arm is None:
            rc = self._lib.bf_resident_commit(self._ctx, handle, int(n_runs), ep, ents.shape[0], C.byref(out))
        else:
            rc = self._lib.bf_resident_commit_timed(self._ctx, handle, int(n_runs), ep, ents.shape[0], C.byref(out), a)
        if rc != A.BF_OK:
            err = A.FrontierError(rc, "bf_resident_commit: %s" % self._lib.bf_last_error(self._ctx).decode())
            err.bad_run, err.bad_step = int(out.bad_run), int(out.bad_step)
            raise err
        got = {k: int(getattr(out, k)) for k in ("n_runs_written", "n_skipped", "n_launched", "n_queued", "n_failed")}
        if arm is not None:
            got.update(n_armed=int(arm.n_armed), next_deadline=int(arm.next_deadline))
        if journal_cap is not None:
            got.update(items=items[:min(int(j.n_items), int(journal_cap))].copy(), n_items=int(j.n_items),
                       runs=runs[:int(j.n_runs_listed)].copy(), n_runs_listed=int(j.n_runs_listed))
        if rewrites:
            got["n_rewritten"] = int(n_rw.value)
        if touched:
            got.update(full=int(scope.full), n_considered=int(scope.n_considered))
        return got

    # -- run status of resident batches (bf_resident_status)
    STATUS_DTYPE = np.dtype([("run", "<u4"), ("first_event", "<u4"), ("n_events", "<u2"), ("first_failed", "<u2"),
                             ("summary", "<u2"), ("group", "u1"), ("outcome", "u1"), ("story_phase", "u1"),
                             ("reserved", "u1", (7,)), ("active", "<u2"), ("completed", "<u2"), ("failed", "<u2"),
                             ("skipped", "<u2")])   # bf_status_rec, 32 B

    def resident_status(self, handle: int, n_runs: int, runs=None, events_cap: Optional[int] = None):
        """bf_resident_status: the status of the listed runs (runs: strictly ascending, below n_runs; None: every run of
        [0, n_runs)) after the stage G / H / I rewrites of a single pass, without changing anything.  events_cap: events to
        fetch (default: every one the runs can have, 32 * words of the batch's layout per run).  -> (records STATUS_DTYPE[len(runs)], events u16[min(n_events, events_cap)],
        n_events)"""
        rl = None if runs is None else np.ascontiguousarray(runs, dtype=np.uint32)
        n = int(n_runs) if rl is None else rl.shape[0]
        recs = np.zeros(n, dtype=self.STATUS_DTYPE)
        if events_cap is None:
            events_cap = n * 32 * ((self._steps_max[handle] + 31) // 32)
        events = np.zeros(max(int(events_cap), 1), dtype=np.uint16)
        out = A.StatusOut(struct_size=C.sizeof(A.StatusOut), records=recs.ctypes.data if n else None,
                          events=events.ctypes.data if events_cap else None, events_cap=int(events_cap))
        self._check(self._lib.bf_resident_status(self._ctx, handle, int(n_runs), None if rl is None else rl.ctypes.data, n,
                                                 C.byref(out)), "bf_resident_status")
        return recs, events[:min(int(out.n_events), int(events_cap))].copy(), int(out.n_events)

    # -- resyncs of resident batches (bf_resident_resync)
    DRIFT_DTYPE = np.dtype([("run", "<u4"), ("index", "<u2"), ("field", "u1"), ("reserved", "u1"), ("device", "<u4"),
                            ("record", "<u4")])   # bf_drift, 16 B

    def resident_resync(self, handle: int, n_runs: int, records, runs=None, fields: int = A.RESYNC_ALL_FIELDS,
                        check: bool = False, drifted_cap: Optional[int] = None, items_cap: Optional[int] = None) -> dict:
        """bf_resident_resync: compare the device's records of the listed runs (runs: strictly ascending, below n_runs; None:
        every run of [0, n_runs)) with `records` (one packed state record per listed run, list order) after a single pass's
        stages, list every difference and, unless check, repair the runs that drifted.  drifted_cap defaults to every listed
        run, items_cap to 65 536 items (1 MiB; n_items is the true count, so a check with a larger cap lists the rest).  -> {drifted u32[min(n_drifted, cap)], items DRIFT_DTYPE[min(n_items, cap)], n_drifted,
        n_written, n_items}.  A refusal raises FrontierError with .bad_run set."""
        rl = None if runs is None else np.ascontiguousarray(runs, dtype=np.uint32)
        n = int(n_runs) if rl is None else rl.shape[0]
        recs = np.ascontiguousarray(records, dtype=np.uint8)
        if drifted_cap is None:
            drifted_cap = n
        if items_cap is None:   # a buffer not in pinned memory is staged in the ctx's device scratch, which keeps its largest size
            items_cap = min(n * (3 * 32 * ((self._steps_max[handle] + 31) // 32) + self._child_nibbles[handle] + 65), 1 << 16)
        drifted = np.zeros(max(int(drifted_cap), 1), dtype=np.uint32)
        items = np.zeros(max(int(items_cap), 1), dtype=self.DRIFT_DTYPE)
        q = A.Resync(struct_size=C.sizeof(A.Resync), n_runs=int(n_runs), runs=None if rl is None else rl.ctypes.data, n=n,
                     fields=int(fields), records=recs.ctypes.data if recs.size else None, flags=A.RESYNC_CHECK if check else 0,
                     drifted_cap=int(drifted_cap), drifted=drifted.ctypes.data if drifted_cap else None,
                     items=items.ctypes.data if items_cap else None, items_cap=int(items_cap))
        rc = self._lib.bf_resident_resync(self._ctx, handle, C.byref(q))
        if rc != 0:
            err = A.FrontierError(rc, "bf_resident_resync: %s" % self._lib.bf_last_error(self._ctx).decode())
            err.bad_run = int(q.bad_run)
            raise err
        return {"drifted": drifted[:min(int(q.n_drifted), int(drifted_cap))].copy(),
                "items": items[:min(int(q.n_items), int(items_cap))].copy(), "n_drifted": int(q.n_drifted),
                "n_written": int(q.n_written), "n_items": int(q.n_items)}

    def resident_resync_areas(self, handle: int, n_runs: int, runs=None, timers=None, sched=None, runctl=None,
                              fired_now: int = A.TIMER_NONE, check: bool = False, drifted_cap: Optional[int] = None,
                              items_cap: Optional[int] = None) -> dict:
        """bf_resident_resync_areas: compare the device's step timers, limiter inputs and run control of the listed runs (runs:
        strictly ascending, below n_runs; None: every run of [0, n_runs)) with the caller's, list every difference and, unless
        check, repair the runs that drifted.  Each area given is selected: timers SLOT_DTYPE of shape (n, K) with K the batch's
        slots per run (resident_timers; any other shape is a ValueError, as the library reads n * K slots), sched
        SCHED_PUT_DTYPE[n] (.run = the listed run), runctl RUNCTL_DTYPE[n] (saved_flags 0).  fired_now: `now` of the last
        resident_fire on the batch (A.TIMER_NONE: none).  drifted_cap defaults to every listed run, items_cap to 65 536 items.
        -> {drifted u32[min(n_drifted, cap)], items DRIFT_DTYPE[min(n_items, cap)], n_drifted, n_written, n_items}.  A refusal
        raises FrontierError with .bad_run set."""
        rl = None if runs is None else np.ascontiguousarray(runs, dtype=np.uint32)
        n = int(n_runs) if rl is None else rl.shape[0]
        areas = 0
        arrays = []
        for bit, arr, dt in ((A.RESYNC_AREA_TIMERS, timers, self.SLOT_DTYPE), (A.RESYNC_AREA_SCHED, sched, self.SCHED_PUT_DTYPE),
                             (A.RESYNC_AREA_RUNCTL, runctl, self.RUNCTL_DTYPE)):
            if arr is not None:
                areas |= bit
                arr = np.ascontiguousarray(arr, dtype=dt)
                if arr.shape[0] != n:
                    raise ValueError("one row per listed run: %d rows for %d runs" % (arr.shape[0], n))
                K = self._timer_k.get(handle)
                if bit == A.RESYNC_AREA_TIMERS and K is not None and arr.shape != (n, K):
                    raise ValueError("timers must have shape (%d, %d), the batch's slots per run: got %s" % (n, K, arr.shape))
            arrays.append(arr)
        ptr = lambda a: a.ctypes.data if a is not None and a.size else None  # noqa: E731
        if drifted_cap is None:
            drifted_cap = n
        if items_cap is None:   # a buffer not in pinned memory is staged in the ctx's device scratch, which keeps its largest size
            items_cap = 1 << 16
        drifted = np.zeros(max(int(drifted_cap), 1), dtype=np.uint32)
        items = np.zeros(max(int(items_cap), 1), dtype=self.DRIFT_DTYPE)
        q = A.ResyncAreas(struct_size=C.sizeof(A.ResyncAreas), n_runs=int(n_runs), runs=None if rl is None else rl.ctypes.data,
                          n=n, areas=areas, flags=A.RESYNC_CHECK if check else 0, fired_now=int(fired_now),
                          timers=ptr(arrays[0]), sched=ptr(arrays[1]), runctl=ptr(arrays[2]), drifted_cap=int(drifted_cap),
                          drifted=drifted.ctypes.data if drifted_cap else None, items=items.ctypes.data if items_cap else None,
                          items_cap=int(items_cap))
        rc = self._lib.bf_resident_resync_areas(self._ctx, handle, C.byref(q))
        if rc != 0:
            err = A.FrontierError(rc, "bf_resident_resync_areas: %s" % self._lib.bf_last_error(self._ctx).decode())
            err.bad_run = int(q.bad_run)
            raise err
        return {"drifted": drifted[:min(int(q.n_drifted), int(drifted_cap))].copy(),
                "items": items[:min(int(q.n_items), int(items_cap))].copy(), "n_drifted": int(q.n_drifted),
                "n_written": int(q.n_written), "n_items": int(q.n_items)}

    # -- limiter inputs and schedules of resident batches (bf_resident_sched*, bf_resident_schedule)
    SCHED_PUT_DTYPE = np.dtype([("run", "<u4"), ("story_key", "<u4"), ("queue_key", "<u4"), ("priority", "<i4"),
                                ("queued_since", "<u4"), ("run_phase", "<u4"), ("reserved", "<u4", (2,))])   # bf_sched_put, 32 B
    SCHED_HEAD_DTYPE = np.dtype([("n_launch", "<u4"), ("n_queued_story", "<u4"), ("n_queued_sched", "<u4"),
                                 ("reason", "<u4")])                                                         # bf_sched_header

    def resident_sched(self, handle: int):
        """bf_resident_sched: create the batch's limiter-inputs area, every run at the defaults"""
        self._check(self._lib.bf_resident_sched(self._ctx, handle), "bf_resident_sched")

    def resident_sched_put(self, handle: int, requests: np.ndarray):
        """bf_resident_sched_put: write the limiter inputs of each requests[i].run (SCHED_PUT_DTYPE, at most one per run)"""
        rq = np.ascontiguousarray(requests, dtype=self.SCHED_PUT_DTYPE)
        self._check(self._lib.bf_resident_sched_put(self._ctx, handle, rq.ctypes.data if rq.shape[0] else None, rq.shape[0]),
                    "bf_resident_sched_put")

    def resident_sched_download(self, handle: int, first_run: int, n_runs: int) -> np.ndarray:
        """bf_resident_sched_download -> the stored inputs of runs [first_run, first_run + n_runs), SCHED_PUT_DTYPE"""
        out = np.zeros(n_runs, dtype=self.SCHED_PUT_DTYPE)
        self._check(self._lib.bf_resident_sched_download(self._ctx, handle, first_run, n_runs, out.ctypes.data),
                    "bf_resident_sched_download")
        return out

    def resident_schedule(self, parts, tables: dict, now: int) -> dict:
        """bf_resident_schedule over several resident batches against one set of totals.  parts: list of dicts with handle,
        n_runs and optionally runs_cap / events_cap (default: n_runs and n_runs * 1024) and pinned buffers runs / heads / events.
        tables: Frontier.schedule's keyword arguments.  -> dict(parts=[dict(runs, heads, events, n_listed, full, n_events)],
        story_running, queue_running, queue_max_priority, global_running)"""
        call = _SchedCall(tables, parts)
        self._check(self._lib.bf_resident_schedule(self._ctx, C.byref(call.t), int(now), call.ps, len(parts), C.byref(call.out)),
                    "bf_resident_schedule")
        return call.result()

    # -- resident batches: device-side state, delta uploads (row f2)
    DELTA_DTYPE = np.dtype([("run", "<u4"), ("index", "<u2"), ("field", "u1"), ("code", "u1")])

    def resident_create(self, L: A.Layout, capacity: int) -> int:
        h = C.c_uint32()
        self._check(self._lib.bf_resident_create(self._ctx, C.byref(L), capacity, C.byref(h)), "bf_resident_create")
        self._steps_max[h.value] = int(L.steps_max)   # its words size resident_status's default event buffer
        self._child_nibbles[h.value] = int(L.child_nibbles)   # and, with it, resident_resync's default item buffer
        self._timer_k.pop(h.value, None)
        return h.value

    def resident_destroy(self, handle: int):
        self._check(self._lib.bf_resident_destroy(self._ctx, handle), "bf_resident_destroy")

    def resident_upload(self, handle: int, first_run: int, state: np.ndarray):
        assert state.dtype == np.uint8 and state.flags["C_CONTIGUOUS"]
        self._check(self._lib.bf_resident_upload(self._ctx, handle, first_run, state.shape[0], state.ctypes.data), "bf_resident_upload")

    def resident_download(self, handle: int, first_run: int, n_runs: int, state_stride: int) -> np.ndarray:
        out = np.zeros((n_runs, state_stride), dtype=np.uint8)
        self._check(self._lib.bf_resident_download(self._ctx, handle, first_run, n_runs, out.ctypes.data), "bf_resident_download")
        return out

    def resident_apply(self, handle: int, deltas: np.ndarray):
        """deltas: structured array of DELTA_DTYPE (8 bytes each), at most one per (run, field, index)"""
        d = np.ascontiguousarray(deltas, dtype=self.DELTA_DTYPE)
        self._check(self._lib.bf_resident_apply(self._ctx, handle, d.ctypes.data, d.shape[0]), "bf_resident_apply")

    def resident_eval(self, handle: int, L: A.Layout, n_runs: int, result: Optional[np.ndarray] = None, flags: int = 0,
                      max_iterations: int = 0):
        if result is None:
            result = np.zeros((n_runs, L.result_stride), dtype=np.uint8)
        counts = A.Counts()
        self._check(self._lib.bf_resident_eval(self._ctx, handle, n_runs, flags, max_iterations, result.ctypes.data, C.byref(counts)),
                    "bf_resident_eval")
        return result, {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}

    def resident_tick(self, handle: int, L: A.Layout, n_runs: int, deltas: np.ndarray, result: Optional[np.ndarray] = None,
                      flags: int = 0, max_iterations: int = 0):
        """bf_resident_tick: deltas + pass + results in one call.  `deltas` must be a C-contiguous DELTA_DTYPE array
        (pinned memory from alloc_pinned makes its upload asynchronous)."""
        assert deltas.dtype == self.DELTA_DTYPE and deltas.flags["C_CONTIGUOUS"]
        if result is None:
            result = np.zeros((n_runs, L.result_stride), dtype=np.uint8)
        counts = A.Counts()
        self._check(self._lib.bf_resident_tick(self._ctx, handle, deltas.ctypes.data, deltas.shape[0], n_runs, flags, max_iterations,
                                               result.ctypes.data, C.byref(counts)), "bf_resident_tick")
        return result, {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}

    # -- redrive closure (row f3; storyrun_controller.go:535-558)
    def closure(self, slots, steps, words: int) -> np.ndarray:
        """bf_topology_closure: [count, words] uint32 masks of the steps a redrive from (slot, step) resets."""
        sl = np.ascontiguousarray(slots, dtype=np.uint32)
        st = np.ascontiguousarray(steps, dtype=np.uint32)
        assert sl.shape == st.shape
        out = np.zeros((sl.size, words), dtype=np.uint32)
        u32p = C.POINTER(C.c_uint32)
        self._check(self._lib.bf_topology_closure(self._ctx, sl.ctypes.data_as(u32p), st.ctypes.data_as(u32p), sl.size, words,
                                                  out.ctypes.data_as(u32p)), "bf_topology_closure")
        return out

    # -- limiters over the ready sets of the batch just evaluated (rows a9 / f4; dag.go:1780-1961)
    def schedule(self, L: A.Layout, n_runs: int, sched_runs: np.ndarray, story_limit, queue_limit, queue_aging_s,
                 global_limit: int = 0, story_running_base=None, queue_running_base=None, global_running_base: int = 0,
                 queue_max_priority_base=None):
        """bf_schedule: must follow eval() of the same batch.  sched_runs: [n_runs] records of 32 bytes (bf_sched_run).
        Returns dict(records [n, stride] uint8, story_running, queue_running, queue_max_priority, global_running)."""
        assert sched_runs.nbytes == 32 * n_runs and sched_runs.flags["C_CONTIGUOUS"]
        sl = np.ascontiguousarray(story_limit, dtype=np.int32)
        ql = np.ascontiguousarray(queue_limit, dtype=np.int32)
        qa = np.ascontiguousarray(queue_aging_s, dtype=np.int32)
        sb = None if story_running_base is None else np.ascontiguousarray(story_running_base, dtype=np.uint32)
        qb = None if queue_running_base is None else np.ascontiguousarray(queue_running_base, dtype=np.uint32)
        pb = None if queue_max_priority_base is None else np.ascontiguousarray(queue_max_priority_base, dtype=np.int32)
        assert ql.shape == qa.shape
        t = A.SchedTables(struct_size=C.sizeof(A.SchedTables), n_stories=sl.size, n_queues=ql.size, global_limit=global_limit,
                          global_running_base=global_running_base, story_limit=sl.ctypes.data,
                          story_running_base=(sb.ctypes.data if sb is not None else None), queue_limit=ql.ctypes.data,
                          queue_aging_s=qa.ctypes.data, queue_running_base=(qb.ctypes.data if qb is not None else None),
                          queue_max_priority_base=(pb.ctypes.data if pb is not None else None))
        stride = A.sched_stride(L.words)
        rec = np.zeros((n_runs, stride), dtype=np.uint8)
        sr = np.zeros(max(sl.size, 1), dtype=np.uint32)
        qr = np.zeros(max(ql.size, 1), dtype=np.uint32)
        mp = np.zeros(max(ql.size, 1), dtype=np.int32)
        gr = np.zeros(1, dtype=np.uint32)
        out = A.SchedOut(struct_size=C.sizeof(A.SchedOut), records=rec.ctypes.data, story_running=sr.ctypes.data,
                         queue_running=qr.ctypes.data, queue_max_priority=mp.ctypes.data, global_running=gr.ctypes.data)
        b = A.Batch(struct_size=C.sizeof(A.Batch), n_runs=n_runs, layout=L)
        self._check(self._lib.bf_schedule(self._ctx, C.byref(b), C.c_void_p(sched_runs.ctypes.data), C.byref(t), C.byref(out)),
                    "bf_schedule")
        return {"records": rec, "story_running": sr[:sl.size], "queue_running": qr[:ql.size], "queue_max_priority": mp[:ql.size],
                "global_running": int(gr[0])}

    def schedule_device(self, L: A.Layout, n_runs: int, state_ptr: int, result_ptr: int, runs_ptr: int, records_ptr: int,
                        story_running_ptr: int, queue_running_ptr: int, queue_max_priority_ptr: int, global_running_ptr: int,
                        n_stories: int, n_queues: int, story_limit_ptr: int, queue_limit_ptr: int, queue_aging_ptr: int,
                        global_limit: int = 0, global_running_base: int = 0, story_running_base_ptr: int = 0,
                        queue_running_base_ptr: int = 0, queue_max_priority_base_ptr: int = 0, stream: int = 0):
        """bf_schedule_device: every pointer is a device address (0 = NULL); the batch is the (state, result) pair of a
        preceding eval_device.  The totals arrays are the reduction scratch and must be given.  Asynchronous on `stream`."""
        t = A.SchedTables(struct_size=C.sizeof(A.SchedTables), n_stories=n_stories, n_queues=n_queues, global_limit=global_limit,
                          global_running_base=global_running_base, story_limit=(story_limit_ptr or None),
                          story_running_base=(story_running_base_ptr or None), queue_limit=(queue_limit_ptr or None),
                          queue_aging_s=(queue_aging_ptr or None), queue_running_base=(queue_running_base_ptr or None),
                          queue_max_priority_base=(queue_max_priority_base_ptr or None))
        out = A.SchedOut(struct_size=C.sizeof(A.SchedOut), records=(records_ptr or None), story_running=(story_running_ptr or None),
                         queue_running=(queue_running_ptr or None), queue_max_priority=(queue_max_priority_ptr or None),
                         global_running=(global_running_ptr or None))
        b = A.Batch(struct_size=C.sizeof(A.Batch), n_runs=n_runs, layout=L, state=(state_ptr or None), result=(result_ptr or None))
        self._check(self._lib.bf_schedule_device(self._ctx, C.byref(b), C.c_void_p(runs_ptr or None), C.byref(t), C.byref(out),
                                                 C.c_void_p(stream)), "bf_schedule_device")

    # -- evaluation over DEVICE buffers (async on `stream`)
    def eval_device(self, L: A.Layout, n_runs: int, state_ptr: int, result_ptr: int, counts_ptr: int = 0,
                    stream: int = 0, flags: int = 0, max_iterations: int = 0, expansion_ptr: int = 0,
                    expansion_cap: int = 0):
        b = A.Batch(struct_size=C.sizeof(A.Batch), n_runs=n_runs, flags=flags, max_iterations=max_iterations, layout=L,
                    state=state_ptr, result=result_ptr, expansion=(expansion_ptr or None), expansion_cap=expansion_cap,
                    counts=(counts_ptr or None))
        self._check(self._lib.bf_eval_device(self._ctx, C.byref(b), C.c_void_p(stream)), "bf_eval_device")

    def alloc_pinned(self, nbytes: int) -> np.ndarray:
        p = C.c_void_p()
        self._check(self._lib.bf_alloc_pinned(self._ctx, nbytes, C.byref(p)), "bf_alloc_pinned")
        buf = (C.c_uint8 * nbytes).from_address(p.value)
        arr = np.frombuffer(buf, dtype=np.uint8)
        self._pinned = getattr(self, "_pinned", {})
        self._pinned[arr.ctypes.data] = p.value
        return arr

    def free_pinned(self, arr: np.ndarray):
        ptr = getattr(self, "_pinned", {}).pop(arr.ctypes.data, None)
        if ptr is not None:
            self._check(self._lib.bf_free_pinned(self._ctx, C.c_void_p(ptr)), "bf_free_pinned")

    def stats(self) -> Dict[str, int]:
        s = A.Stats()
        self._check(self._lib.bf_get_stats(self._ctx, C.byref(s)), "bf_get_stats")
        return {n: getattr(s, n) for n, _ in s._fields_}


class _SchedCall:
    """The arguments of one bf_resident_schedule / bf_resident_schedule_ctxs call (tables, parts with their output buffers,
    totals), kept alive together, and the result dict they hold afterwards."""

    def __init__(self, tables: dict, parts):
        self.sl = np.ascontiguousarray(tables["story_limit"], dtype=np.int32)
        ql = self.ql = np.ascontiguousarray(tables["queue_limit"], dtype=np.int32)
        self.qa = np.ascontiguousarray(tables["queue_aging_s"], dtype=np.int32)
        arr = lambda k, dt: None if tables.get(k) is None else np.ascontiguousarray(tables[k], dtype=dt)  # noqa: E731
        self.bases = sb, qb, pb = (arr("story_running_base", np.uint32), arr("queue_running_base", np.uint32),
                                   arr("queue_max_priority_base", np.int32))
        self.t = A.SchedTables(struct_size=C.sizeof(A.SchedTables), n_stories=self.sl.size, n_queues=ql.size,
                               global_limit=int(tables.get("global_limit", 0)),
                               global_running_base=int(tables.get("global_running_base", 0)),
                               story_limit=self.sl.ctypes.data, story_running_base=(sb.ctypes.data if sb is not None else None),
                               queue_limit=ql.ctypes.data, queue_aging_s=self.qa.ctypes.data,
                               queue_running_base=(qb.ctypes.data if qb is not None else None),
                               queue_max_priority_base=(pb.ctypes.data if pb is not None else None))
        self.ps = (A.ResidentSchedPart * max(len(parts), 1))()
        self.bufs = []
        for i, p in enumerate(parts):
            n = int(p["n_runs"])
            rcap = int(p.get("runs_cap", n))
            ecap = int(p.get("events_cap", n * 1024))
            runs = p.get("runs", np.zeros(max(rcap, 1), np.uint32))
            heads = p.get("heads", np.zeros(max(rcap, 1), Frontier.SCHED_HEAD_DTYPE))
            events = p.get("events", np.zeros(max(ecap, 1), np.uint16))
            self.bufs.append((runs, heads, events, rcap, ecap))
            self.ps[i] = A.ResidentSchedPart(struct_size=C.sizeof(A.ResidentSchedPart), handle=int(p["handle"]), n_runs=n,
                                             runs_cap=rcap, runs=runs.ctypes.data, heads=heads.ctypes.data, events=events.ctypes.data,
                                             events_cap=ecap)
        self.sr = np.zeros(max(self.sl.size, 1), dtype=np.uint32)
        self.qr = np.zeros(max(ql.size, 1), dtype=np.uint32)
        self.mp = np.zeros(max(ql.size, 1), dtype=np.int32)
        self.gr = np.zeros(1, dtype=np.uint32)
        self.out = A.SchedOut(struct_size=C.sizeof(A.SchedOut), records=None, story_running=self.sr.ctypes.data,
                              queue_running=self.qr.ctypes.data, queue_max_priority=self.mp.ctypes.data,
                              global_running=self.gr.ctypes.data)

    def result(self) -> dict:
        res = []
        for i, (runs, heads, events, rcap, ecap) in enumerate(self.bufs):
            q = self.ps[i]
            nl = min(int(q.n_listed), rcap)
            res.append({"runs": runs[:nl].copy(), "heads": heads[:nl].copy(), "events": events[:min(int(q.n_events), ecap)].copy(),
                        "n_listed": int(q.n_listed), "full": int(q.full), "n_events": int(q.n_events)})
        ns, nq = self.sl.size, self.ql.size
        return {"parts": res, "story_running": self.sr[:ns], "queue_running": self.qr[:nq], "queue_max_priority": self.mp[:nq],
                "global_running": int(self.gr[0])}


def resident_schedule_ctxs(parts, tables: dict, now: int) -> dict:
    """bf_resident_schedule_ctxs: one schedule over resident batches of several ctxs.  parts: list of (frontier, part), each part
    a dict as Frontier.resident_schedule takes.  -> Frontier.resident_schedule's dict, its parts in the order given"""
    if not parts:
        raise ValueError("resident_schedule_ctxs needs at least one part")
    call = _SchedCall(tables, [p for _, p in parts])
    cps = (A.CtxSchedPart * len(parts))()
    for i, (fr, _) in enumerate(parts):
        cps[i] = A.CtxSchedPart(struct_size=C.sizeof(A.CtxSchedPart), ctx=fr._ctx, part=C.pointer(call.ps[i]))
    lib = parts[0][0]._lib
    rc = lib.bf_resident_schedule_ctxs(C.byref(call.t), int(now), cps, len(parts), C.byref(call.out))
    if rc != A.BF_OK:
        fr = parts[0][0]
        raise A.FrontierError(rc, "bf_resident_schedule_ctxs: %s" % fr._lib.bf_last_error(fr._ctx).decode())
    return call.result()


class FrontierGroup:
    """One process, several GPUs: bf_group_* (a ctx per device + an NCCL communicator over them).  Runs shard into
    contiguous blocks; the only exchange of a pass is the all-gather of the per-shard counts."""

    def __init__(self, devices: Sequence[int]):
        self._lib = A.load()
        self._g = C.c_void_p()
        dev = (C.c_int32 * len(devices))(*devices)
        rc = self._lib.bf_group_create(C.byref(self._g), dev, len(devices), None)
        if rc != A.BF_OK:
            self._g = None
            raise A.FrontierError(rc, "bf_group_create(devices=%s)" % list(devices))
        self.size = int(self._lib.bf_group_size(self._g))
        self.shards = [Frontier(_borrowed_ctx=self._lib.bf_group_ctx(self._g, k)) for k in range(self.size)]

    def close(self):
        if getattr(self, "_g", None):
            for s in self.shards:
                s.close()
            self._lib.bf_group_destroy(self._g)
            self._g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc != A.BF_OK:
            raise A.FrontierError(rc, "%s: %s" % (what, self._lib.bf_group_last_error(self._g).decode()))

    def shard_range(self, n_runs: int, shard: int):
        first, count = C.c_uint32(), C.c_uint32()
        self._check(self._lib.bf_group_shard_range(self._g, n_runs, shard, C.byref(first), C.byref(count)), "bf_group_shard_range")
        return first.value, count.value

    def put_topologies_replicated(self, ts: TopologySet) -> np.ndarray:
        desc = ts.descriptors()
        slots = np.zeros(ts.count, dtype=np.uint32)
        self._check(self._lib.bf_group_topology_put_many(self._g, desc.ctypes.data_as(C.POINTER(A.Topology)), ts.count,
                                                         slots.ctypes.data_as(C.POINTER(C.c_uint32))), "bf_group_topology_put_many")
        return slots

    def eval(self, L: A.Layout, state: np.ndarray, result: Optional[np.ndarray] = None, flags: int = 0, max_iterations: int = 0):
        """bf_group_eval -> (result, global counts, per-shard counts)"""
        n = int(state.shape[0])
        assert state.dtype == np.uint8 and state.flags["C_CONTIGUOUS"] and state.shape[1] == L.state_stride
        if result is None:
            result = np.zeros((n, L.result_stride), dtype=np.uint8)
        counts = A.Counts()
        per = (A.Counts * self.size)()
        b = A.Batch(struct_size=C.sizeof(A.Batch), n_runs=n, flags=flags, max_iterations=max_iterations, layout=L,
                    state=state.ctypes.data, result=result.ctypes.data, expansion=None, expansion_cap=0, counts=C.addressof(counts))
        self._check(self._lib.bf_group_eval(self._g, C.byref(b), per), "bf_group_eval")
        as_dict = lambda c: {"ready": c.ready, "skip": c.skip, "expansion": c.expansion, "evals": c.evals}
        return result, as_dict(counts), [as_dict(c) for c in per]

    def schedule(self, L: A.Layout, n_runs: int, sched_runs: np.ndarray, story_limit, queue_limit, queue_aging_s,
                 global_limit: int = 0, story_running_base=None, queue_running_base=None, global_running_base: int = 0,
                 queue_max_priority_base=None):
        """bf_group_schedule: must follow eval() of the same batch; limits and priority ordering hold across all shards."""
        assert sched_runs.nbytes == 32 * n_runs and sched_runs.flags["C_CONTIGUOUS"]
        sl = np.ascontiguousarray(story_limit, dtype=np.int32)
        ql = np.ascontiguousarray(queue_limit, dtype=np.int32)
        qa = np.ascontiguousarray(queue_aging_s, dtype=np.int32)
        sb = None if story_running_base is None else np.ascontiguousarray(story_running_base, dtype=np.uint32)
        qb = None if queue_running_base is None else np.ascontiguousarray(queue_running_base, dtype=np.uint32)
        pb = None if queue_max_priority_base is None else np.ascontiguousarray(queue_max_priority_base, dtype=np.int32)
        t = A.SchedTables(struct_size=C.sizeof(A.SchedTables), n_stories=sl.size, n_queues=ql.size, global_limit=global_limit,
                          global_running_base=global_running_base, story_limit=sl.ctypes.data,
                          story_running_base=(sb.ctypes.data if sb is not None else None), queue_limit=ql.ctypes.data,
                          queue_aging_s=qa.ctypes.data, queue_running_base=(qb.ctypes.data if qb is not None else None),
                          queue_max_priority_base=(pb.ctypes.data if pb is not None else None))
        rec = np.zeros((n_runs, A.sched_stride(L.words)), dtype=np.uint8)
        sr, qr = np.zeros(max(sl.size, 1), dtype=np.uint32), np.zeros(max(ql.size, 1), dtype=np.uint32)
        mp, gr = np.zeros(max(ql.size, 1), dtype=np.int32), np.zeros(1, dtype=np.uint32)
        out = A.SchedOut(struct_size=C.sizeof(A.SchedOut), records=rec.ctypes.data, story_running=sr.ctypes.data,
                         queue_running=qr.ctypes.data, queue_max_priority=mp.ctypes.data, global_running=gr.ctypes.data)
        b = A.Batch(struct_size=C.sizeof(A.Batch), n_runs=n_runs, layout=L)
        self._check(self._lib.bf_group_schedule(self._g, C.byref(b), C.c_void_p(sched_runs.ctypes.data), C.byref(t), C.byref(out)),
                    "bf_group_schedule")
        return {"records": rec, "story_running": sr[:sl.size], "queue_running": qr[:ql.size], "queue_max_priority": mp[:ql.size],
                "global_running": int(gr[0])}
