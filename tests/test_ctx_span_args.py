"""bf_resident_transfer_ctx and bf_resident_schedule_ctxs without a GPU: the symbols and their argument types, the layouts of
bf_ctx_transfer and bf_ctx_sched_part against the header, the constants, and the refusals that need no ctx."""
import ctypes as C
import os
import re

from bobrapet_b200 import _abi as A
from bobrapet_b200 import frontier as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "bobrafrontier.h")).read()


def _fields(struct):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), HEADER, re.S).group(1)
    return re.findall(r"\b(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))


def test_ctx_transfer_layout():
    assert C.sizeof(A.CtxTransfer) == 112
    assert [(n, getattr(A.CtxTransfer, n).offset) for n, _ in A.CtxTransfer._fields_] == [
        ("struct_size", 0), ("src_n_runs", 4), ("dst_n_runs", 8), ("runs", 16), ("n", 24), ("slot_map", 32), ("n_slot_map", 40),
        ("moves_from", 48), ("moves_to", 56), ("n_moves", 64), ("unfit", 68), ("unfit_reason", 72), ("why", 76)]
    assert _fields("bf_ctx_transfer") == [n for n, _ in A.CtxTransfer._fields_]


def test_ctx_sched_part_layout():
    assert C.sizeof(A.CtxSchedPart) == 24
    assert [(n, getattr(A.CtxSchedPart, n).offset) for n, _ in A.CtxSchedPart._fields_] == [
        ("struct_size", 0), ("reserved", 4), ("ctx", 8), ("part", 16)]
    assert _fields("bf_ctx_sched_part") == [n for n, _ in A.CtxSchedPart._fields_]


def test_constants_match_the_header():
    assert re.search(r"#define BF_SLOT_NONE 0xFFFFFFFFu", HEADER) and A.SLOT_NONE == 0xFFFFFFFF
    enum = dict((n, int(v)) for n, v in re.findall(r"\b(BF_UNFIT_[A-Z_]+) = (\d+)", HEADER))
    assert enum == {"BF_UNFIT_NONE": A.UNFIT_NONE, "BF_UNFIT_LAYOUT": A.UNFIT_LAYOUT, "BF_UNFIT_SLOT_UNMAPPED": A.UNFIT_SLOT_UNMAPPED,
                    "BF_UNFIT_SLOT_PAST_MAP": A.UNFIT_SLOT_PAST_MAP, "BF_UNFIT_SLOT_DEAD": A.UNFIT_SLOT_DEAD}


def test_symbols_and_argument_types():
    lib = A.load()
    fn = lib.bf_resident_transfer_ctx
    assert fn.restype == C.c_int
    assert fn.argtypes == [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(A.CtxTransfer)]
    fn = lib.bf_resident_schedule_ctxs
    assert fn.restype == C.c_int
    assert fn.argtypes == [C.POINTER(A.SchedTables), C.c_uint32, C.POINTER(A.CtxSchedPart), C.c_uint32, C.POINTER(A.SchedOut)]
    assert callable(F.resident_schedule_ctxs) and callable(F.Frontier.resident_transfer_ctx)


def test_null_ctxs_and_empty_calls_are_refused():
    lib = A.load()
    t = A.CtxTransfer(struct_size=C.sizeof(A.CtxTransfer))
    assert lib.bf_resident_transfer_ctx(None, 0, None, 0, C.byref(t)) == A.BF_EINVAL
    tables = A.SchedTables(struct_size=C.sizeof(A.SchedTables))
    out = A.SchedOut(struct_size=C.sizeof(A.SchedOut))
    assert lib.bf_resident_schedule_ctxs(C.byref(tables), 0, None, 0, C.byref(out)) == A.BF_EINVAL
    parts = (A.CtxSchedPart * 1)()
    parts[0] = A.CtxSchedPart(struct_size=C.sizeof(A.CtxSchedPart))   # no ctx, no part
    assert lib.bf_resident_schedule_ctxs(C.byref(tables), 0, parts, 1, C.byref(out)) == A.BF_EINVAL
