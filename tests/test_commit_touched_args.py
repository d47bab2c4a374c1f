"""bf_resident_commit_touched and bf_resident_commit_marks without a GPU: the symbols and their argument types, the bf_commit_scope
layout the header gives, and the refusals that need no batch."""
import ctypes as C
import os
import re

from bobrapet_b200 import _abi as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_commit_scope_layout():
    assert C.sizeof(A.CommitScope) == 16
    assert [(n, getattr(A.CommitScope, n).offset) for n, _ in A.CommitScope._fields_] == [
        ("struct_size", 0), ("flags", 4), ("full", 8), ("n_considered", 12)]
    text = open(os.path.join(ROOT, "include", "bobrafrontier.h")).read()
    body = re.search(r"typedef struct bf_commit_scope \{(.*?)\} bf_commit_scope;", text, re.S).group(1)
    names = re.findall(r"\b(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [n for n, _ in A.CommitScope._fields_]
    assert re.search(r"#define BF_COMMIT_SCOPE_REWRITES 0x1u", text) and A.COMMIT_SCOPE_REWRITES == 1


def test_symbols_and_argument_types():
    lib = A.load()
    fn = lib.bf_resident_commit_touched
    assert fn.restype == C.c_int
    assert fn.argtypes == [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(A.CommitOut), C.POINTER(A.CommitArm),
                           C.POINTER(A.CommitJournal), C.POINTER(C.c_uint32), C.POINTER(A.CommitScope)]
    assert lib.bf_resident_commit_marks.restype == C.c_int
    assert lib.bf_resident_commit_marks.argtypes == [C.c_void_p, C.c_uint32]


def test_null_ctx_is_refused():
    lib = A.load()
    out = A.CommitOut(struct_size=C.sizeof(A.CommitOut))
    scope = A.CommitScope(struct_size=C.sizeof(A.CommitScope), full=7, n_considered=7)
    assert lib.bf_resident_commit_touched(None, 0, 0, None, 0, C.byref(out), None, None, None, C.byref(scope)) == A.BF_EINVAL
    assert lib.bf_resident_commit_touched(None, 0, 0, None, 0, C.byref(out), None, None, None, None) == A.BF_EINVAL
    assert lib.bf_resident_commit_marks(None, 0) == A.BF_EINVAL
