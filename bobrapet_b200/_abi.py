"""ctypes mirror of include/bobrafrontier.h and loader of lib/libbobrafrontier.so.

The product path has NO CPU fallback: if the CUDA library is missing or cannot
be loaded this module raises, loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BF_LIB") or os.path.join(_HERE, "lib", "libbobrafrontier.so")  # BF_LIB: A/B builds

BF_ABI_VERSION = 3
BF_OK, BF_EINVAL, BF_ENOMEM, BF_ECUDA, BF_ENCCL, BF_ETOPO, BF_ENODEV = 0, -1, -2, -3, -4, -5, -6

# phase codes (pkg/enums/enums.go:44-97 order; 14 = Pending + "Queued due to ..." message)
PHASE_NONE, PHASE_PENDING, PHASE_RUNNING, PHASE_SUCCEEDED, PHASE_FAILED = 0, 1, 2, 3, 4
PHASE_FINISHED, PHASE_CANCELED, PHASE_COMPENSATED, PHASE_PAUSED, PHASE_BLOCKED = 5, 6, 7, 8, 9
PHASE_SCHEDULING, PHASE_TIMEOUT, PHASE_ABORTED, PHASE_SKIPPED, PHASE_PENDING_QUEUED = 10, 11, 12, 13, 14
PHASE_NAMES = ["", "Pending", "Running", "Succeeded", "Failed", "Finished", "Canceled", "Compensated",
               "Paused", "Blocked", "Scheduling", "Timeout", "Aborted", "Skipped", "Pending"]

QUEUED_NONE, QUEUED_PRIORITY, QUEUED_GLOBAL, QUEUED_QUEUE, QUEUED_OTHER = range(5)  # BF_QUEUED_*
SCHED_NONE = 0xFFFFFFFF
DELTA_PHASE, DELTA_COND, DELTA_DECISION, DELTA_CHILD, DELTA_RUN_FLAGS, DELTA_REGISTERED, DELTA_TOPO_SLOT = range(7)  # BF_DELTA_*
STEP_ENGRAM, STEP_CONDITION, STEP_PARALLEL, STEP_SLEEP, STEP_STOP, STEP_WAIT, STEP_EXECUTE_STORY, STEP_GATE = range(8)
STEP_TYPE_CODE = {"": STEP_ENGRAM, "condition": STEP_CONDITION, "parallel": STEP_PARALLEL, "sleep": STEP_SLEEP,
                  "stop": STEP_STOP, "wait": STEP_WAIT, "executeStory": STEP_EXECUTE_STORY, "gate": STEP_GATE}
SF_TYPE_MASK, SF_ALLOW_FAILURE, SF_ON_TIMEOUT_SKIP, SF_HAS_IF, SF_GROUP_SHIFT = 0x07, 0x08, 0x10, 0x20, 6
GROUP_MAIN, GROUP_COMPENSATION, GROUP_FINALLY, GROUP_DONE = 0, 1, 2, 3
RF_FAIL_FAST, RF_REALTIME, RF_TOPOLOGY_TERMINATED, RF_HOST_GROUP, RF_HOST_GROUP_SHIFT = 0x01, 0x02, 0x04, 0x08, 4
COND_PASS, COND_SKIP, COND_HOLD, COND_FAIL = 0, 1, 2, 3
DEC_PENDING, DEC_SUCCEED, DEC_FAIL, DEC_TIMED_OUT = 0, 1, 2, 3
MAX_STEPS, MAX_EDGES, MAX_PARALLEL, OFF_NONE = 1024, 65535, 64, 0xFFFFFFFF

F_COND, F_DECISION, F_CHILD = 0x1, 0x2, 0x4
F_OUT_FAIL, F_OUT_NEEDS_COND, F_OUT_SKIP_DEP, F_OUT_PHASE = 0x10, 0x20, 0x40, 0x80
F_ALL_OUT = F_OUT_FAIL | F_OUT_NEEDS_COND | F_OUT_SKIP_DEP | F_OUT_PHASE
EVAL_VALIDATE, EVAL_FIXPOINT, EVAL_EXPANSION, EVAL_NO_COUNTS = 0x1, 0x2, 0x4, 0x8

SUM_GROUP_MASK, SUM_MAIN_DONE, SUM_MAIN_FAILED, SUM_COMP_DONE, SUM_FINAL_DONE = 0x3, 0x4, 0x8, 0x10, 0x20
SUM_COMP_FAILED, SUM_FINAL_FAILED, SUM_PHASE_CHANGED, SUM_ITER_SHIFT = 0x40, 0x80, 0x100, 16


class ParallelDesc(C.Structure):
    _fields_ = [("step", C.c_uint16), ("branches", C.c_uint16), ("allow_first", C.c_uint32)]


class Topology(C.Structure):
    _fields_ = [
        ("n_steps", C.c_uint32), ("n_edges", C.c_uint32),
        ("row_ptr", C.c_void_p), ("col_idx", C.c_void_p), ("step_flags", C.c_void_p),
        ("parallel", C.c_void_p), ("n_parallel", C.c_uint32),
        ("branch_allow_bits", C.c_void_p), ("n_branch_allow_bits", C.c_uint32),
    ]


class Layout(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "steps_max", "words", "fields", "child_nibbles", "state_stride",
        "off_phase", "off_cond", "off_decision", "off_child", "result_stride",
        "off_ready", "off_skip", "off_fail", "off_needs_cond", "off_skip_dep", "off_phase_out")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class Expansion(C.Structure):
    _fields_ = [("run", C.c_uint32), ("step", C.c_uint16), ("branch", C.c_uint16)]


class Counts(C.Structure):
    _fields_ = [("ready", C.c_uint64), ("skip", C.c_uint64), ("expansion", C.c_uint64), ("evals", C.c_uint64)]


class Batch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("n_runs", C.c_uint32), ("flags", C.c_uint32), ("max_iterations", C.c_uint32),
        ("layout", Layout),
        ("state", C.c_void_p), ("result", C.c_void_p),
        ("expansion", C.c_void_p), ("expansion_cap", C.c_uint64),
        ("counts", C.c_void_p),
    ]


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("arena_bytes", C.c_uint64),
                ("max_topologies", C.c_uint32), ("flags", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("arena_used_bytes", C.c_uint64), ("arena_cap_bytes", C.c_uint64),
                ("n_topologies", C.c_uint32), ("sm_count", C.c_uint32), ("last_grid", C.c_uint32),
                ("last_block", C.c_uint32), ("last_smem_bytes", C.c_uint32), ("last_stages", C.c_uint32),
                ("last_kernel", C.c_uint32), ("last_runs_per_trip", C.c_uint32),
                ("last_eval_chunks", C.c_uint32), ("arena_compactions", C.c_uint32)]


EVT_READY, EVT_SKIP, EVT_FAIL, EVT_NEEDS_COND, EVT_SKIP_DEP = 0x1, 0x2, 0x4, 0x8, 0x10  # BF_EVT_*


HEAD_SUMMARY_MASK, HEAD_DEAD, HEAD_LISTED, HEAD_COUNT_SHIFT = 0x7FFF, 0x7FFF, 0x8000, 16  # BF_HEAD_*
EVAL_CHANGED_ONLY = 0x10
EVAL_COUNTS_SET, EVAL_PIPELINED = 0x20, 0x40


class CompactOut(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_listed", C.c_uint32), ("head", C.c_void_p), ("events", C.c_void_p),
                ("events_cap", C.c_uint64), ("n_events", C.c_uint64)]


class TouchedOut(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("full", C.c_uint32), ("runs", C.c_void_p), ("head", C.c_void_p),
                ("runs_cap", C.c_uint32), ("n_listed", C.c_uint32), ("n_evaluated", C.c_uint32), ("reserved", C.c_uint32),
                ("events", C.c_void_p), ("events_cap", C.c_uint64), ("n_events", C.c_uint64)]


class TickPart(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("handle", C.c_uint32), ("deltas", C.c_void_p), ("n_deltas", C.c_uint32),
                ("n_runs", C.c_uint32), ("out", C.c_void_p), ("counts", C.c_void_p)]


MIGRATE_GONE = 0xFFFF   # BF_MIGRATE_GONE: the old step has no step of the new generation


class Migration(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("old_slot", C.c_uint32), ("new_slot", C.c_uint32), ("n_runs", C.c_uint32),
                ("step_map", C.c_void_p), ("n_old_steps", C.c_uint32), ("migrated", C.c_uint32)]


REDRIVE_ALL = 0xFFFFFFFF   # BF_REDRIVE_ALL: bf_redrive.step for a redrive of the whole run


class Redrive(C.Structure):
    _fields_ = [("run", C.c_uint32), ("slot", C.c_uint32), ("step", C.c_uint32), ("reserved", C.c_uint32)]


class Retire(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_runs", C.c_uint32), ("runs", C.c_void_p), ("n", C.c_uint32),
                ("capacity", C.c_uint32), ("moves_from", C.c_void_p), ("moves_to", C.c_void_p), ("n_moves", C.c_uint32)]


EXTENT_NO_RUN = 0xFFFFFFFF   # BF_EXTENT_NO_RUN: bf_extent.widest_run when no run needs any step


class Extent(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_runs", C.c_uint32), ("steps_max", C.c_uint32), ("child_nibbles", C.c_uint32),
                ("fields", C.c_uint32), ("widest_run", C.c_uint32), ("reserved", C.c_uint32 * 2)]

    def as_dict(self):
        return {n: getattr(self, n) for n in ("steps_max", "child_nibbles", "fields", "widest_run")}


class Transfer(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("src_n_runs", C.c_uint32), ("dst_n_runs", C.c_uint32), ("runs", C.c_void_p),
                ("n", C.c_uint32), ("moves_from", C.c_void_p), ("moves_to", C.c_void_p), ("n_moves", C.c_uint32),
                ("unfit", C.c_uint32), ("why", Extent)]


SLOT_NONE = 0xFFFFFFFF   # BF_SLOT_NONE: a slot_map entry of bf_resident_transfer_ctx that maps no slot
UNFIT_NONE, UNFIT_LAYOUT, UNFIT_SLOT_UNMAPPED, UNFIT_SLOT_PAST_MAP, UNFIT_SLOT_DEAD = 0, 1, 2, 3, 4   # BF_UNFIT_*


class CtxTransfer(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("src_n_runs", C.c_uint32), ("dst_n_runs", C.c_uint32), ("runs", C.c_void_p),
                ("n", C.c_uint32), ("slot_map", C.c_void_p), ("n_slot_map", C.c_uint32), ("moves_from", C.c_void_p),
                ("moves_to", C.c_void_p), ("n_moves", C.c_uint32), ("unfit", C.c_uint32), ("unfit_reason", C.c_uint32),
                ("why", Extent)]


TIMER_NONE = 0xFFFFFFFF   # BF_TIMER_NONE: an empty slot's deadline; as a request's deadline it cancels
TIMER_MAX_SLOTS = 64      # BF_TIMER_MAX_SLOTS


class FireOut(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_runs", C.c_uint32), ("n_fired", C.c_uint32), ("n_written", C.c_uint32),
                ("n_pruned", C.c_uint32), ("next_deadline", C.c_uint32), ("fired", C.c_void_p), ("fired_cap", C.c_uint32),
                ("reserved", C.c_uint32)]


class SchedTables(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_stories", C.c_uint32), ("n_queues", C.c_uint32), ("global_limit", C.c_int32),
                ("global_running_base", C.c_uint32), ("story_limit", C.c_void_p), ("story_running_base", C.c_void_p),
                ("queue_limit", C.c_void_p), ("queue_aging_s", C.c_void_p), ("queue_running_base", C.c_void_p),
                ("queue_max_priority_base", C.c_void_p)]


class SchedOut(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("records", C.c_void_p), ("story_running", C.c_void_p),
                ("queue_running", C.c_void_p), ("queue_max_priority", C.c_void_p), ("global_running", C.c_void_p)]


SEVT_LAUNCH, SEVT_QUEUED_STORY, SEVT_QUEUED_SCHED = 0x1, 0x2, 0x4   # BF_SEVT_*: event kinds of bf_resident_schedule


class ResidentSchedPart(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("handle", C.c_uint32), ("n_runs", C.c_uint32), ("runs_cap", C.c_uint32),
                ("runs", C.c_void_p), ("heads", C.c_void_p), ("events", C.c_void_p), ("events_cap", C.c_uint64),
                ("n_listed", C.c_uint32), ("full", C.c_uint32), ("n_events", C.c_uint64)]


class CtxSchedPart(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("ctx", C.c_void_p), ("part", C.POINTER(ResidentSchedPart))]


STOP_NONE, STOP_TIMEOUT, STOP_CANCEL, STOP_HOST = 0, 1, 2, 3   # BF_STOP_*: why a run of a resident batch is stopped
FIRED_DRAIN, FIRED_STORY = 0xFFFE, 0xFFFF                       # bf_fired.step of a drain deadline / a story timeout


COMMIT_HOLD, COMMIT_ERROR, COMMIT_PHASE = 1, 2, 3   # BF_COMMIT_*: bf_commit_entry.kind
COMMIT_NONE = 0xFFFFFFFF                           # BF_COMMIT_NONE: bad_run / bad_step of a refusal of the whole call


class CommitOut(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("struct_size", "n_runs_written", "n_skipped", "n_launched", "n_queued", "n_failed",
                                          "bad_run", "bad_step")]


class CommitArm(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("struct_size", "now", "n_armed", "next_deadline")]


COMMIT_WRITE_TIMER = 0x10   # BF_COMMIT_WRITE_TIMER: bf_commit_write.field of a timer-arm item (else DELTA_PHASE / DELTA_REGISTERED)
COMMIT_WRITE_REWRITE = 0x1   # BF_COMMIT_WRITE_REWRITE: bf_commit_write.code of a PHASE item whose code comes from stages G / H / I


class CommitJournal(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("items", C.c_void_p), ("items_cap", C.c_uint64),
                ("n_items", C.c_uint64), ("runs", C.c_void_p), ("runs_cap", C.c_uint32), ("n_runs_listed", C.c_uint32)]


COMMIT_SCOPE_REWRITES = 0x1   # BF_COMMIT_SCOPE_REWRITES: bf_commit_scope.flags of a touched commit matching bf_resident_commit_rewrites


class CommitScope(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("struct_size", "flags", "full", "n_considered")]


OUTCOME_NONE, OUTCOME_SUCCEEDED, OUTCOME_DEPENDENCY_FAILED, OUTCOME_COMPENSATED = 0, 1, 2, 3   # BF_OUTCOME_*: bf_status_rec.outcome
OUTCOME_COMPENSATION_FAILED, OUTCOME_CLEANUP_FAILED, OUTCOME_TIMED_OUT = 4, 5, 6
OUTCOME_CANCELED, OUTCOME_STOPPED, OUTCOME_DEAD = 7, 8, 9
STATUS_EVT_FAILED, STATUS_EVT_ALLOWED = 0x1, 0x2   # BF_STATUS_EVT_*: kind of a status event (bits 14-15)
STATUS_NO_STEP = 0xFFFF                            # BF_STATUS_NO_STEP: first_failed of a run without a listed failed set


class StatusOut(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("records", C.c_void_p), ("events", C.c_void_p),
                ("events_cap", C.c_uint64), ("n_events", C.c_uint64)]


RESYNC_CHECK = 0x1          # BF_RESYNC_CHECK: compare and list only
RESYNC_ALL_FIELDS = 0x3F    # BF_RESYNC_FIELD(BF_DELTA_PHASE) | ... | BF_RESYNC_FIELD(BF_DELTA_REGISTERED)
RESYNC_NONE = 0xFFFFFFFF    # BF_RESYNC_NONE: bf_resync.bad_run of a refusal that names no run


def resync_field(f: int) -> int:
    """BF_RESYNC_FIELD(f) for a BF_DELTA_* field"""
    return 1 << f


class Resync(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_runs", C.c_uint32), ("runs", C.c_void_p), ("n", C.c_uint32),
                ("fields", C.c_uint32), ("records", C.c_void_p), ("flags", C.c_uint32), ("drifted_cap", C.c_uint32),
                ("drifted", C.c_void_p), ("n_drifted", C.c_uint32), ("n_written", C.c_uint32), ("items", C.c_void_p),
                ("items_cap", C.c_uint64), ("n_items", C.c_uint64), ("bad_run", C.c_uint32), ("reserved", C.c_uint32)]


RESYNC_AREA_TIMERS, RESYNC_AREA_SCHED, RESYNC_AREA_RUNCTL = 0x1, 0x2, 0x4   # BF_RESYNC_AREA_*: areas of bf_resident_resync_areas
RESYNC_ALL_AREAS = 0x7
DRIFT_TIMER, DRIFT_TIMER_CODE = 8, 9                   # BF_DRIFT_*: bf_drift.field of bf_resident_resync_areas
DRIFT_SCHED_STORY_KEY, DRIFT_SCHED_QUEUE_KEY, DRIFT_SCHED_PRIORITY, DRIFT_SCHED_QUEUED_SINCE, DRIFT_SCHED_RUN_PHASE = 10, 11, 12, 13, 14
DRIFT_STORY_DEADLINE, DRIFT_DRAIN_DEADLINE, DRIFT_STOP = 15, 16, 17


class ResyncAreas(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_runs", C.c_uint32), ("runs", C.c_void_p), ("n", C.c_uint32),
                ("areas", C.c_uint32), ("flags", C.c_uint32), ("fired_now", C.c_uint32), ("timers", C.c_void_p),
                ("sched", C.c_void_p), ("runctl", C.c_void_p), ("drifted_cap", C.c_uint32), ("n_drifted", C.c_uint32),
                ("drifted", C.c_void_p), ("n_written", C.c_uint32), ("bad_run", C.c_uint32), ("items", C.c_void_p),
                ("items_cap", C.c_uint64), ("n_items", C.c_uint64)]


def sched_stride(words: int) -> int:
    return (16 + 12 * words + 15) & ~15


# every symbol include/bobrafrontier.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("bf_abi_version", C.c_uint32, []),
    ("bf_strerror", C.c_char_p, [C.c_int]),
    ("bf_last_error", C.c_char_p, [C.c_void_p]),
    ("bf_create", C.c_int, [C.POINTER(C.c_void_p), C.POINTER(Config)]),
    ("bf_destroy", None, [C.c_void_p]),
    ("bf_topology_put", C.c_int, [C.c_void_p, C.POINTER(Topology), C.POINTER(C.c_uint32)]),
    ("bf_topology_put_many", C.c_int, [C.c_void_p, C.POINTER(Topology), C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bf_topology_put_many_checked_on_device", C.c_int, [C.c_void_p, C.POINTER(Topology), C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    ("bf_topology_check", C.c_int, [C.c_void_p, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bf_topology_closure", C.c_int, [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bf_topology_drop", C.c_int, [C.c_void_p, C.c_uint32]),
    ("bf_topology_timings", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bf_topology_child_first", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32]),
    ("bf_layout_init", C.c_int, [C.POINTER(Layout), C.c_uint32, C.c_uint32, C.c_uint32]),
    ("bf_eval", C.c_int, [C.c_void_p, C.POINTER(Batch)]),
    ("bf_eval_device", C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p]),
    ("bf_schedule", C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.POINTER(SchedTables), C.POINTER(SchedOut)]),
    ("bf_schedule_device", C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.POINTER(SchedTables), C.POINTER(SchedOut), C.c_void_p]),
    ("bf_resident_create", C.c_int, [C.c_void_p, C.POINTER(Layout), C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bf_resident_destroy", C.c_int, [C.c_void_p, C.c_uint32]),
    ("bf_resident_upload", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]),
    ("bf_resident_apply", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bf_resident_eval", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(Counts)]),
    ("bf_resident_tick", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(Counts)]),
    ("bf_resident_download", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]),
    ("bf_eval_compact", C.c_int, [C.c_void_p, C.POINTER(Batch), C.POINTER(CompactOut)]),
    ("bf_resident_tick_compact", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(CompactOut), C.POINTER(Counts)]),
    ("bf_resident_tick_touched", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(TouchedOut), C.POINTER(Counts)]),
    ("bf_resident_tick_touched_many", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(TickPart), C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bf_resident_migrate", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(Migration)]),
    ("bf_resident_redrive", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]),
    ("bf_resident_reshape", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(Layout), C.c_uint32]),
    ("bf_resident_retire", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(Retire)]),
    ("bf_resident_extent", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(Extent)]),
    ("bf_resident_narrow", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(Layout), C.POINTER(Extent)]),
    ("bf_resident_transfer", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(Transfer)]),
    ("bf_resident_transfer_ctx", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(CtxTransfer)]),
    ("bf_resident_timers", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    ("bf_resident_timers_arm", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bf_resident_fire", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(FireOut)]),
    ("bf_resident_timers_download", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]),
    ("bf_resident_sched", C.c_int, [C.c_void_p, C.c_uint32]),
    ("bf_resident_sched_put", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bf_resident_sched_download", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]),
    ("bf_resident_schedule", C.c_int, [C.c_void_p, C.POINTER(SchedTables), C.c_uint32, C.POINTER(ResidentSchedPart), C.c_uint32,
                                       C.POINTER(SchedOut)]),
    ("bf_resident_schedule_ctxs", C.c_int, [C.POINTER(SchedTables), C.c_uint32, C.POINTER(CtxSchedPart), C.c_uint32,
                                            C.POINTER(SchedOut)]),
    ("bf_resident_runctl", C.c_int, [C.c_void_p, C.c_uint32]),
    ("bf_resident_runctl_put", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]),
    ("bf_resident_runctl_download", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]),
    ("bf_resident_commit", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(CommitOut)]),
    ("bf_resident_commit_timed", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(CommitOut),
                                           C.POINTER(CommitArm)]),
    ("bf_resident_commit_journal", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(CommitOut),
                                             C.POINTER(CommitArm), C.POINTER(CommitJournal)]),
    ("bf_resident_commit_rewrites", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(CommitOut),
                                              C.POINTER(CommitArm), C.POINTER(CommitJournal), C.POINTER(C.c_uint32)]),
    ("bf_resident_commit_marks", C.c_int, [C.c_void_p, C.c_uint32]),
    ("bf_resident_commit_touched", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(CommitOut),
                                             C.POINTER(CommitArm), C.POINTER(CommitJournal), C.POINTER(C.c_uint32),
                                             C.POINTER(CommitScope)]),
    ("bf_resident_status", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(StatusOut)]),
    ("bf_resident_resync", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(Resync)]),
    ("bf_resident_resync_areas", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(ResyncAreas)]),
    ("bf_group_create", C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_uint32, C.POINTER(Config)]),
    ("bf_group_destroy", None, [C.c_void_p]),
    ("bf_group_size", C.c_uint32, [C.c_void_p]),
    ("bf_group_ctx", C.c_void_p, [C.c_void_p, C.c_uint32]),
    ("bf_group_last_error", C.c_char_p, [C.c_void_p]),
    ("bf_group_shard_range", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    ("bf_group_topology_put_many", C.c_int, [C.c_void_p, C.POINTER(Topology), C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bf_group_eval", C.c_int, [C.c_void_p, C.POINTER(Batch), C.POINTER(Counts)]),
    ("bf_group_schedule", C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.POINTER(SchedTables), C.POINTER(SchedOut)]),
    ("bf_alloc_pinned", C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]),
    ("bf_free_pinned", C.c_int, [C.c_void_p, C.c_void_p]),
    ("bf_get_stats", C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    ("bf_topology_record", C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]),
    ("bf_topology_record_build", C.c_int, [C.POINTER(Topology), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]),
]

_lib = None


class FrontierError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__("bobrafrontier: %s (%d): %s" % (_strerror(status), status, message))
        self.status = status


def _strerror(status: int) -> str:
    try:
        return load().bf_strerror(status).decode()
    except Exception:
        return "status"


def load() -> C.CDLL:
    """Load the CUDA extension.  Raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "bobrapet_b200: %s is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the frontier path)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    ab_build = bool(os.environ.get("BF_LIB"))  # an older build loaded for a same-box A/B timing: newer entry points may be absent
    for name, res, args in SYMBOLS:
        try:
            fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        except AttributeError:
            if ab_build:
                continue
            raise
        fn.restype = res
        fn.argtypes = args
    if lib.bf_abi_version() != BF_ABI_VERSION and not ab_build:
        raise RuntimeError("bobrapet_b200: ABI version mismatch")
    _lib = lib
    return lib
