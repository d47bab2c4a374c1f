"""bf_resident_tick_touched_many without a GPU: the symbol and its argument types, and the bf_tick_part layout the header gives."""
import ctypes as C
import os
import re

from bobrapet_b200 import _abi as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tick_part_layout():
    assert C.sizeof(A.TickPart) == 40
    assert [(n, getattr(A.TickPart, n).offset) for n, _ in A.TickPart._fields_] == [
        ("struct_size", 0), ("handle", 4), ("deltas", 8), ("n_deltas", 16), ("n_runs", 20), ("out", 24), ("counts", 32)]
    text = open(os.path.join(ROOT, "include", "bobrafrontier.h")).read()
    body = re.search(r"typedef struct bf_tick_part \{(.*?)\} bf_tick_part;", text, re.S).group(1)
    names = re.findall(r"\b(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [n for n, _ in A.TickPart._fields_]


def test_symbol_and_argument_types():
    lib = A.load()
    fn = lib.bf_resident_tick_touched_many
    assert fn.restype == C.c_int
    assert fn.argtypes == [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(A.TickPart), C.c_uint32, C.POINTER(C.c_uint32)]


def test_null_ctx_is_refused_and_names_no_part():
    lib = A.load()
    bad = C.c_uint32(5)
    parts = (A.TickPart * 1)()
    assert lib.bf_resident_tick_touched_many(None, 0, 0, parts, 1, C.byref(bad)) == A.BF_EINVAL
    assert bad.value == A.COMMIT_NONE
    assert lib.bf_resident_tick_touched_many(None, 0, 0, None, 0, None) == A.BF_EINVAL
