"""ctypes binding of include/bobrafrontier_host.h — the C++ host-side mirror (Story / StoryRun packer)."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import numpy as np

from . import _abi as A

_SYMS = [
    ("bfh_story_new", C.c_void_p, []),
    ("bfh_story_free", None, [C.c_void_p]),
    ("bfh_story_error", C.c_char_p, [C.c_void_p]),
    ("bfh_story_add_step", C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_char_p]),
    ("bfh_step_add_need", C.c_int, [C.c_void_p, C.c_int, C.c_char_p]),
    ("bfh_step_add_branch", C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_int]),
    ("bfh_story_set_policy", C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    ("bfh_story_finalize", C.c_int, [C.c_void_p]),
    ("bfh_story_dims", C.c_int, [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    ("bfh_story_csr", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("bfh_story_upload", C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]),
    ("bfh_story_step_index", C.c_int, [C.c_void_p, C.c_char_p]),
    ("bfh_story_step_name", C.c_char_p, [C.c_void_p, C.c_uint32]),
    ("bfh_story_run_flags", C.c_uint32, [C.c_void_p]),
    ("bfh_scan_step_refs", C.c_int, [C.c_char_p, C.c_char_p, C.c_size_t]),
    ("bfh_batch_new", C.c_void_p, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
    ("bfh_batch_free", None, [C.c_void_p]),
    ("bfh_batch_error", C.c_char_p, [C.c_void_p]),
    ("bfh_batch_layout", C.POINTER(A.Layout), [C.c_void_p]),
    ("bfh_batch_size", C.c_uint32, [C.c_void_p]),
    ("bfh_batch_state", C.c_void_p, [C.c_void_p]),
    ("bfh_batch_result", C.c_void_p, [C.c_void_p]),
    ("bfh_batch_add_run", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32]),
    ("bfh_batch_remove_last_run", C.c_int, [C.c_void_p]),
    ("bfh_run_set_phase", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_char_p, C.c_char_p]),
    ("bfh_run_set_phase_code", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]),
    ("bfh_run_set_cond", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]),
    ("bfh_run_set_decision", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]),
    ("bfh_run_set_gate", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_char_p, C.c_int]),
    ("bfh_run_set_run_flags", C.c_int, [C.c_void_p, C.c_uint32, C.c_int, C.c_int]),
    ("bfh_run_register_children", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]),
    ("bfh_run_set_child_phase", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p]),
    ("bfh_story_migration_map", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]),
    ("bfh_batch_migrate", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]),
    ("bfh_batch_redrive", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]),
    ("bfh_batch_reshape", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
    ("bfh_batch_retire", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]),
    ("bfh_batch_narrow", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]),
    ("bfh_batch_transfer", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    ("bfh_batch_eval", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(A.Counts)]),
    ("bfh_batch_commit", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(A.CommitOut)]),
    ("bfh_batch_commit_rewrites", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(A.CommitOut), C.POINTER(C.c_uint32)]),
    ("bfh_batch_set_resident", C.c_int, [C.c_void_p, C.c_int]),
    ("bfh_batch_traffic", C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]),
    ("bfh_run_summary", C.c_uint32, [C.c_void_p, C.c_uint32]),
    ("bfh_run_ready", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bfh_run_skipped", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bfh_run_failed", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bfh_run_needs_cond", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bfh_run_phase_out", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    ("bfh_run_skip_reason", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]),
    ("bfh_sched_new", C.c_void_p, [C.c_void_p]),
    ("bfh_sched_free", None, [C.c_void_p]),
    ("bfh_sched_error", C.c_char_p, [C.c_void_p]),
    ("bfh_sched_set_global", C.c_int, [C.c_void_p, C.c_int32, C.c_uint32]),
    ("bfh_sched_set_queue", C.c_int, [C.c_void_p, C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.c_uint32]),
    ("bfh_sched_set_story_base", C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_uint32]),
    ("bfh_sched_set_run", C.c_int, [C.c_void_p, C.c_uint32, C.c_char_p, C.c_char_p, C.c_int32, C.c_char_p, C.c_int, C.c_int32,
                                    C.c_char_p, C.c_int64, C.c_int64]),
    ("bfh_sched_runs", C.c_void_p, [C.c_void_p]),
    ("bfh_sched_tables", C.c_int, [C.c_void_p, C.POINTER(A.SchedTables)]),
    ("bfh_sched_queue_name", C.c_char_p, [C.c_void_p, C.c_uint32]),
    ("bfh_sched_apply", C.c_int, [C.c_void_p]),
    ("bfh_sched_steps", C.c_int, [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_uint32]),
    ("bfh_sched_message", C.c_int, [C.c_void_p, C.c_uint32, C.c_int, C.c_char_p, C.c_size_t]),
    ("bfh_sched_format_message", C.c_int, [C.c_int, C.c_uint32, C.c_int32, C.c_char_p, C.c_size_t]),
]
HOST_SYMBOLS = [n for n, _, _ in _SYMS]
_bound = False


def lib():
    global _bound
    L = A.load()
    if not _bound:
        for name, res, args in _SYMS:
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _bound = True
    return L


def _b(s: Optional[str]):
    return None if s is None else s.encode()


class HostStory:
    """bfh_story: a Story generation packed by the C++ host mirror."""

    def __init__(self):
        self._l = lib()
        self._p = C.c_void_p(self._l.bfh_story_new())

    def close(self):
        if self._p:
            self._l.bfh_story_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def error(self) -> str:
        return self._l.bfh_story_error(self._p).decode()

    def add_step(self, name, group=0, type_=0, allow_failure=False, on_timeout_skip=False, if_expr=None, with_raw=None,
                 needs=(), branches=()) -> int:
        h = self._l.bfh_story_add_step(self._p, _b(name), group, type_, int(bool(allow_failure)), int(bool(on_timeout_skip)),
                                       _b(if_expr), _b(with_raw))
        if h < 0:
            raise A.FrontierError(h, "bfh_story_add_step")
        for d in needs:
            self._l.bfh_step_add_need(self._p, h, _b(d))
        for bn, al in branches:
            self._l.bfh_step_add_branch(self._p, h, _b(bn), int(bool(al)))
        return h

    def set_policy(self, continue_on_step_failure=None, realtime=False):
        c = -1 if continue_on_step_failure is None else int(bool(continue_on_step_failure))
        self._l.bfh_story_set_policy(self._p, c, int(bool(realtime)))

    def finalize(self) -> int:
        return self._l.bfh_story_finalize(self._p)

    def csr(self):
        S, E, P = C.c_uint32(), C.c_uint32(), C.c_uint32()
        rc = self._l.bfh_story_dims(self._p, C.byref(S), C.byref(E), C.byref(P))
        if rc != 0:
            raise A.FrontierError(rc, "bfh_story_dims: " + self.error())
        rp = np.zeros(S.value + 1, np.uint32)
        ci = np.zeros(max(E.value, 1), np.uint16)
        fl = np.zeros(S.value, np.uint8)
        self._l.bfh_story_csr(self._p, rp.ctypes.data, ci.ctypes.data, fl.ctypes.data)
        return rp, ci[:E.value], fl, P.value

    def upload(self, frontier) -> int:
        slot = C.c_uint32()
        rc = self._l.bfh_story_upload(self._p, frontier._ctx, C.byref(slot))
        if rc != 0:
            raise A.FrontierError(rc, "bfh_story_upload: " + self.error())
        return slot.value

    def index(self, name: str) -> int:
        return self._l.bfh_story_step_index(self._p, _b(name))

    def name(self, idx: int) -> str:
        return self._l.bfh_story_step_name(self._p, idx).decode()

    def run_flags(self) -> int:
        return self._l.bfh_story_run_flags(self._p)

    def migration_map(self, new: "HostStory") -> np.ndarray:
        """bfh_story_migration_map: [S] uint16, the index in `new` of each step of this story by name, or A.MIGRATE_GONE"""
        n = self._l.bfh_story_migration_map(self._p, new._p, None, 0)
        if n < 0:
            raise A.FrontierError(n, "bfh_story_migration_map")
        out = np.zeros(max(n, 1), np.uint16)
        self._l.bfh_story_migration_map(self._p, new._p, out.ctypes.data, n)
        return out[:n]


def scan_step_refs(expr: str) -> List[str]:
    buf = C.create_string_buffer(65536)
    n = lib().bfh_scan_step_refs(expr.encode(), buf, len(buf))
    out = buf.value.decode().split("\n")[:-1]
    assert len(out) == n
    return out


class HostBatch:
    """bfh_batch: live StoryRuns packed in place (pinned when a device ctx is given)."""

    def __init__(self, frontier, steps_max, child_nibbles=0, fields=0, capacity=1024):
        self._l = lib()
        self._fr = frontier
        ctx = frontier._ctx if frontier is not None else None
        self._p = C.c_void_p(self._l.bfh_batch_new(ctx, steps_max, child_nibbles, fields, capacity))
        if not self._p:
            raise RuntimeError("bfh_batch_new failed")
        self.L = self._l.bfh_batch_layout(self._p).contents

    def close(self):
        if self._p:
            self._l.bfh_batch_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc, what):
        if rc < 0:
            raise A.FrontierError(rc, "%s: %s" % (what, self._l.bfh_batch_error(self._p).decode()))
        return rc

    def add_run(self, story: HostStory, slot: int) -> int:
        return self._chk(self._l.bfh_batch_add_run(self._p, story._p, slot), "bfh_batch_add_run")

    def set_phase(self, run, step, phase, message=""):
        self._chk(self._l.bfh_run_set_phase(self._p, run, step, _b(phase), _b(message)), "bfh_run_set_phase")

    def set_resident(self, on=True):
        self._chk(self._l.bfh_batch_set_resident(self._p, int(bool(on))), "bfh_batch_set_resident")

    def traffic(self):
        """(bytes sent as full records, bytes sent as deltas, deltas pending)"""
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint32()
        self._chk(self._l.bfh_batch_traffic(self._p, C.byref(a), C.byref(b), C.byref(c)), "bfh_batch_traffic")
        return a.value, b.value, c.value

    def set_phase_code(self, run, step, code):
        self._chk(self._l.bfh_run_set_phase_code(self._p, run, step, code), "bfh_run_set_phase_code")

    def set_cond(self, run, step, code):
        self._chk(self._l.bfh_run_set_cond(self._p, run, step, code), "bfh_run_set_cond")

    def set_decision(self, run, step, code):
        self._chk(self._l.bfh_run_set_decision(self._p, run, step, code), "bfh_run_set_decision")

    def set_gate(self, run, step, state, timed_out=False):
        self._chk(self._l.bfh_run_set_gate(self._p, run, step, _b(state), int(timed_out)), "bfh_run_set_gate")

    def set_run_flags(self, run, topology_terminated=False, host_group=-1):
        self._chk(self._l.bfh_run_set_run_flags(self._p, run, int(topology_terminated), host_group), "bfh_run_set_run_flags")

    def register_children(self, run, q, on=True):
        self._chk(self._l.bfh_run_register_children(self._p, run, q, int(on)), "bfh_run_register_children")

    def set_child_phase(self, run, q, branch, phase):
        self._chk(self._l.bfh_run_set_child_phase(self._p, run, q, branch, _b(phase)), "bfh_run_set_child_phase")

    def migrate(self, old: HostStory, new: HostStory, old_slot: int, new_slot: int) -> int:
        """bfh_batch_migrate: move the runs on old_slot to `new` / new_slot (in resident mode on the device too) -> runs moved"""
        return self._chk(self._l.bfh_batch_migrate(self._p, old._p, new._p, old_slot, new_slot), "bfh_batch_migrate")

    def redrive(self, runs, steps) -> None:
        """bfh_batch_redrive: reset runs[i] from step steps[i] (an index of its story) or, for -1, the whole run (in resident
        mode on the device too)"""
        r = np.ascontiguousarray(runs, dtype=np.uint32)
        s = np.ascontiguousarray(steps, dtype=np.int32)
        assert r.shape == s.shape
        self._chk(self._l.bfh_batch_redrive(self._p, r.ctypes.data, s.ctypes.data, r.shape[0]), "bfh_batch_redrive")

    def reshape(self, steps_max, child_nibbles, fields, capacity) -> None:
        """bfh_batch_reshape: grow the layout to bf_layout_init(steps_max, child_nibbles, fields) and the capacity, keeping every
        run's records and the pending deltas (in resident mode on the device too)"""
        self._chk(self._l.bfh_batch_reshape(self._p, steps_max, child_nibbles, fields, capacity), "bfh_batch_reshape")

    def narrow(self, steps_max, child_nibbles, fields) -> None:
        """bfh_batch_narrow: shrink the layout to bf_layout_init(steps_max, child_nibbles, fields) when the records, the runs'
        stories and the pending deltas allow it, keeping every run's records and the pending deltas (in resident mode on the
        device too)"""
        self._chk(self._l.bfh_batch_narrow(self._p, steps_max, child_nibbles, fields), "bfh_batch_narrow")

    def retire(self, runs, capacity=0):
        """bfh_batch_retire: take `runs` out of the batch; the last live runs move into the freed indices (in resident mode on the
        device too), and pending deltas follow them.  -> (moves_from, moves_to), ascending by target"""
        rs = np.ascontiguousarray(runs, dtype=np.uint32)
        mf = np.zeros(max(rs.shape[0], 1), np.uint32)
        mt = np.zeros(max(rs.shape[0], 1), np.uint32)
        k = self._chk(self._l.bfh_batch_retire(self._p, rs.ctypes.data if rs.shape[0] else None, rs.shape[0], capacity,
                                               mf.ctypes.data, mt.ctypes.data), "bfh_batch_retire")
        return mf[:k].copy(), mt[:k].copy()

    def transfer(self, dst: "HostBatch", runs):
        """bfh_batch_transfer: move `runs` to the end of `dst`, re-laid at its layout, with their Stories and pending deltas (in
        resident mode on the device too); this batch compacts as after retire.  -> (moves_from, moves_to), ascending by target"""
        rs = np.ascontiguousarray(runs, dtype=np.uint32)
        mf = np.zeros(max(rs.shape[0], 1), np.uint32)
        mt = np.zeros(max(rs.shape[0], 1), np.uint32)
        k = self._chk(self._l.bfh_batch_transfer(self._p, dst._p, rs.ctypes.data if rs.shape[0] else None, rs.shape[0],
                                                 mf.ctypes.data, mt.ctypes.data), "bfh_batch_transfer")
        return mf[:k].copy(), mt[:k].copy()

    def size(self) -> int:
        return self._l.bfh_batch_size(self._p)

    def state(self) -> np.ndarray:
        n = self.size()
        buf = (C.c_uint8 * (n * self.L.state_stride)).from_address(self._l.bfh_batch_state(self._p))
        return np.frombuffer(buf, np.uint8).reshape(n, self.L.state_stride)

    def result(self) -> np.ndarray:
        n = self.size()
        buf = (C.c_uint8 * (n * self.L.result_stride)).from_address(self._l.bfh_batch_result(self._p))
        return np.frombuffer(buf, np.uint8).reshape(n, self.L.result_stride)

    def eval(self, flags=0):
        c = A.Counts()
        self._chk(self._l.bfh_batch_eval(self._p, flags, C.byref(c)), "bfh_batch_eval")
        return {"ready": c.ready, "skip": c.skip, "expansion": c.expansion, "evals": c.evals}

    def commit(self, entries=None, rewrites: bool = False) -> dict:
        """bfh_batch_commit: the tick commit of the last eval's runs on the device (resident mode), its writes applied to the
        mirror's records except where a delta logged since the eval covers them.  entries: Frontier.COMMIT_DTYPE rows (or
        tuples).  With rewrites (bfh_batch_commit_rewrites) the commit also stores the phases a single pass's stages G, H and I
        rewrote, and the result holds n_rewritten.  -> dict(n_runs_written, n_skipped, n_launched, n_queued, n_failed); a refusal
        raises FrontierError with .bad_run and .bad_step"""
        from .frontier import Frontier
        ents = np.zeros(0, Frontier.COMMIT_DTYPE) if entries is None else entries
        if not isinstance(ents, np.ndarray):
            ents = np.array([tuple(e) for e in ents], dtype=Frontier.COMMIT_DTYPE)
        ents = np.ascontiguousarray(ents, dtype=Frontier.COMMIT_DTYPE)
        out = A.CommitOut(struct_size=C.sizeof(A.CommitOut))
        ep = ents.ctypes.data if ents.shape[0] else None
        nrw = C.c_uint32(0)
        if rewrites:
            rc = self._l.bfh_batch_commit_rewrites(self._p, ep, ents.shape[0], C.byref(out), C.byref(nrw))
        else:
            rc = self._l.bfh_batch_commit(self._p, ep, ents.shape[0], C.byref(out))
        if rc < 0:
            err = A.FrontierError(rc, "bfh_batch_commit: %s" % self._l.bfh_batch_error(self._p).decode())
            err.bad_run, err.bad_step = int(out.bad_run), int(out.bad_step)
            raise err
        got = {k: int(getattr(out, k)) for k in ("n_runs_written", "n_skipped", "n_launched", "n_queued", "n_failed")}
        if rewrites:
            got["n_rewritten"] = int(nrw.value)
        return got

    def _list(self, fn, run, cap=1024):
        out = np.zeros(cap, np.uint32)
        n = fn(self._p, run, out.ctypes.data, cap)
        if n < 0:
            raise A.FrontierError(n, "result list")
        return out[:n].tolist()

    def ready(self, run):
        return self._list(self._l.bfh_run_ready, run)

    def skipped(self, run):
        return self._list(self._l.bfh_run_skipped, run)

    def failed(self, run):
        return self._list(self._l.bfh_run_failed, run)

    def needs_cond(self, run):
        return self._list(self._l.bfh_run_needs_cond, run)

    def summary(self, run):
        return self._l.bfh_run_summary(self._p, run)

    def phase_out(self, run, step):
        return self._l.bfh_run_phase_out(self._p, run, step)

    def skip_reason(self, run, step) -> str:
        buf = C.create_string_buffer(512)
        self._chk(self._l.bfh_run_skip_reason(self._p, run, step, buf, len(buf)), "bfh_run_skip_reason")
        return buf.value.decode()


class HostSched:
    """bfh_sched: host side of the limiters (rows a9 / f4) for one HostBatch — scheduling decisions, keys, elapsed
    seconds in; launch / queued step lists and the reference's queue messages out."""

    def __init__(self, batch: "HostBatch"):
        self._l = lib()
        self._batch = batch
        self._p = C.c_void_p(self._l.bfh_sched_new(batch._p))
        if not self._p:
            raise RuntimeError("bfh_sched_new failed")

    def close(self):
        if self._p:
            self._l.bfh_sched_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc, what):
        if rc < 0:
            raise A.FrontierError(rc, "%s: %s" % (what, self._l.bfh_sched_error(self._p).decode()))
        return rc

    def set_global(self, limit: int, running_base: int = 0):
        self._chk(self._l.bfh_sched_set_global(self._p, limit, running_base), "bfh_sched_set_global")

    def set_queue(self, name, concurrency=0, default_priority=0, aging_s=0, running_base=0) -> int:
        return self._chk(self._l.bfh_sched_set_queue(self._p, _b(name), concurrency, default_priority, aging_s, running_base),
                         "bfh_sched_set_queue")

    def set_story_base(self, namespace, name, running_base) -> int:
        return self._chk(self._l.bfh_sched_set_story_base(self._p, _b(namespace), _b(name), running_base), "bfh_sched_set_story_base")

    def set_run(self, run, namespace, story, story_concurrency=0, queue=None, priority=None, run_phase="", queued_since=None, now=0.0):
        """queued_since / now: Unix seconds (float); passed to the library in nanoseconds"""
        self._chk(self._l.bfh_sched_set_run(self._p, run, _b(namespace), _b(story), story_concurrency, _b(queue),
                                            int(priority is not None), int(priority or 0), _b(run_phase),
                                            -1 if queued_since is None else int(round(queued_since * 1e9)), int(round(now * 1e9))), "bfh_sched_set_run")

    def packed(self):
        """(runs [n] structured array copy, SchedTables with pointers into the C++ object, table arrays as numpy copies)"""
        n = self._l.bfh_batch_size(self._batch._p)
        dt = np.dtype([("story_key", "<u4"), ("queue_key", "<u4"), ("priority", "<i4"), ("queued_elapsed_s", "<u4"),
                       ("run_phase", "<u4"), ("reserved", "<u4", (3,))])
        ptr = self._l.bfh_sched_runs(self._p)
        runs = np.frombuffer((C.c_uint8 * (32 * n)).from_address(ptr), dtype=dt).copy() if ptr and n else np.zeros(0, dt)
        t = A.SchedTables()
        self._chk(self._l.bfh_sched_tables(self._p, C.byref(t)), "bfh_sched_tables")

        def arr(p, cnt, ctype, npdt):
            return np.frombuffer((ctype * cnt).from_address(p), dtype=npdt).copy() if p and cnt else np.zeros(0, npdt)
        tabs = {"story_limit": arr(t.story_limit, t.n_stories, C.c_int32, np.int32),
                "story_base": arr(t.story_running_base, t.n_stories, C.c_uint32, np.uint32),
                "queue_limit": arr(t.queue_limit, t.n_queues, C.c_int32, np.int32),
                "queue_aging": arr(t.queue_aging_s, t.n_queues, C.c_int32, np.int32),
                "queue_base": arr(t.queue_running_base, t.n_queues, C.c_uint32, np.uint32),
                "global_limit": t.global_limit, "global_base": t.global_running_base}
        return runs, tabs

    def queue_name(self, key: int) -> str:
        return self._l.bfh_sched_queue_name(self._p, key).decode()

    def apply(self):
        self._chk(self._l.bfh_sched_apply(self._p), "bfh_sched_apply")

    def steps(self, run: int, which: int) -> List[int]:
        buf = np.zeros(1024, np.uint32)
        n = self._chk(self._l.bfh_sched_steps(self._p, run, which, buf.ctypes.data, 1024), "bfh_sched_steps")
        return buf[:n].tolist()

    def message(self, run: int, which: int) -> str:
        buf = C.create_string_buffer(256)
        self._chk(self._l.bfh_sched_message(self._p, run, which, buf, len(buf)), "bfh_sched_message")
        return buf.value.decode()


def format_queue_message(reason: int, running: int, limit: int) -> str:
    buf = C.create_string_buffer(256)
    lib().bfh_sched_format_message(reason, running, limit, buf, len(buf))
    return buf.value.decode()
