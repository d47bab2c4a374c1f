"""ctypes wrapper of oracle/packed_ref.c (TEST INFRASTRUCTURE — see oracle/README.md).

Evaluates the same packed records the CUDA kernel sees, on the CPU, bit for bit.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libpacked_ref.so")
_LIB = None

ORC_TOPO_DTYPE = np.dtype([
    ("n_steps", "<u4"), ("n_edges", "<u4"), ("row_ptr", "<u8"), ("col_idx", "<u8"), ("step_flags", "<u8"),
    ("parallel", "<u8"), ("n_parallel", "<u4"), ("_pad", "<u4"), ("branch_allow_bits", "<u8"), ("child_first", "<u8"),
])


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "packed_ref.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-pthread", "-I" + os.path.join(_HERE, "..", "include"),
                               src, "-o", _SO])
    return _SO


def _lib():
    global _LIB
    if _LIB is None:
        lib = C.CDLL(build())
        lib.orc_packed_eval.restype = C.c_int
        lib.orc_packed_eval.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                        C.c_uint32, C.c_uint32, C.c_void_p, C.c_int]
        lib.orc_packed_expand.restype = C.c_int
        lib.orc_packed_expand.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_uint64, C.c_void_p]
        _LIB = lib
    return _LIB


def child_first_of(branches) -> np.ndarray:
    """Nibble offsets of parallel descs in the child area: each desc starts 8-nibble aligned
    (the rule bf_topology_put applies, bobrapet_b200/csrc/topology.cu plan_record)."""
    out, nib = [], 0
    for b in branches:
        nib = (nib + 7) // 8 * 8
        out.append(nib)
        nib += int(b)
    return np.asarray(out, dtype=np.uint32)


class PackedTopologies:
    """orc_topology[] indexed by slot, built from a bobrapet_b200.TopologySet-shaped object."""

    def __init__(self, ts, slots=None):
        self.ts = ts
        n = ts.count
        slots = np.arange(n, dtype=np.uint32) if slots is None else np.asarray(slots, dtype=np.uint32)
        self.n_slots = int(slots.max()) + 1 if n else 0
        S64, E64, P64 = ts.S.astype(np.uint64), ts.E.astype(np.uint64), ts.P.astype(np.uint64)
        rp_off = np.concatenate(([0], np.cumsum(S64 + 1)[:-1])).astype(np.uint64)
        ci_off = np.concatenate(([0], np.cumsum(E64)[:-1])).astype(np.uint64)
        sf_off = np.concatenate(([0], np.cumsum(S64)[:-1])).astype(np.uint64)
        pd_off = np.concatenate(([0], np.cumsum(P64)[:-1])).astype(np.uint64)
        # child_first pool: one entry per desc
        cf = np.zeros(int(ts.P.sum()), dtype=np.uint32)
        if cf.size:
            br = ts.parallel["branches"].astype(np.int64)
            pos = 0
            for i in range(n):  # only taken when parallel steps exist
                p = int(ts.P[i])
                cf[pos:pos + p] = child_first_of(br[pos:pos + p])
                pos += p
        self.child_first = cf
        t = np.zeros(self.n_slots, dtype=ORC_TOPO_DTYPE)
        t["n_steps"][slots], t["n_edges"][slots], t["n_parallel"][slots] = ts.S, ts.E, ts.P
        t["row_ptr"][slots] = np.uint64(ts.row_ptr.ctypes.data) + rp_off * np.uint64(4)
        t["col_idx"][slots] = np.uint64(ts.col_idx.ctypes.data if ts.col_idx.size else 0) + ci_off * np.uint64(2)
        t["step_flags"][slots] = np.uint64(ts.step_flags.ctypes.data) + sf_off
        if ts.parallel.size:
            t["parallel"][slots] = np.uint64(ts.parallel.ctypes.data) + pd_off * np.uint64(8)
            t["child_first"][slots] = np.uint64(cf.ctypes.data) + pd_off * np.uint64(4)
        if ts.allow_bits.size:
            t["branch_allow_bits"][slots] = np.uint64(ts.allow_bits.ctypes.data)
        self.table = t

    def max_child_nibbles(self) -> int:
        if not self.child_first.size:
            return 0
        ends = self.child_first.astype(np.int64) + self.ts.parallel["branches"].astype(np.int64)
        return int((int(ends.max()) + 7) // 8 * 8)


def evaluate(pt: PackedTopologies, L, state: np.ndarray, flags: int = 0, max_iter: int = 0, threads: int = 1):
    """-> (result [N, result_stride] uint8, counts dict)."""
    from bobrapet_b200 import _abi as A  # struct definitions only (shared contract header)
    n = int(state.shape[0])
    result = np.zeros((n, L.result_stride), dtype=np.uint8)
    counts = A.Counts()
    rc = _lib().orc_packed_eval(pt.table.ctypes.data, pt.n_slots, C.addressof(L), n, state.ctypes.data,
                                result.ctypes.data, flags, max_iter, C.addressof(counts), threads)
    if rc != 0:
        raise RuntimeError("orc_packed_eval failed: %d" % rc)
    return result, {"ready": counts.ready, "skip": counts.skip, "expansion": counts.expansion, "evals": counts.evals}


def compact_events(L, result: np.ndarray, prev: np.ndarray = None):
    """The compact form of oracle result records (the checker of bf_eval_compact / bf_resident_tick_compact):
    -> (head [N] uint32, events uint16 (step | kind << 10), run-major / step-ascending, n_listed).
    head = low 15 summary bits (0x7FFF for a dead slot) | listed << 15 | event count << 16; kind bits: 1 ready, 2 skip, 4 fail,
    8 needs_cond, 16 skip_dep (BF_EVT_*).  With `prev` (the previous tick's records) only runs whose record differs are listed."""
    n = result.shape[0]
    W = L.words
    summary = np.ascontiguousarray(result[:, 0:4]).view("<u4").reshape(n).copy()
    dead = summary == 0xFFFFFFFF
    kind = np.zeros((n, W * 32), dtype=np.uint16)
    for bit, off in ((1, L.off_ready), (2, L.off_skip), (4, L.off_fail), (8, L.off_needs_cond), (16, L.off_skip_dep)):
        if off != 0xFFFFFFFF:
            m = np.unpackbits(np.ascontiguousarray(result[:, off:off + 4 * W]), axis=1, bitorder="little")
            kind |= m.astype(np.uint16) * np.uint16(bit)
    kind[dead] = 0
    listed = np.ones(n, dtype=bool) if prev is None else (result != prev).any(axis=1)
    kind[~listed] = 0
    count = (kind != 0).sum(axis=1).astype(np.uint32)
    head = np.where(dead, 0x7FFF, summary & 0x7FFF).astype(np.uint32) | (listed.astype(np.uint32) << 15) | (count << 16)
    run, step = np.nonzero(kind)
    ev = (step.astype(np.uint16) | (kind[run, step] << 10)).astype(np.uint16)
    return head, ev, int(listed.sum())


def expand(pt: PackedTopologies, L, state: np.ndarray, result: np.ndarray, cap: int):
    from bobrapet_b200.records import EXP_DTYPE
    out = np.zeros(max(cap, 1), dtype=EXP_DTYPE)
    n_out = C.c_uint64()
    rc = _lib().orc_packed_expand(pt.table.ctypes.data, pt.n_slots, C.addressof(L), int(state.shape[0]),
                                  state.ctypes.data, result.ctypes.data, out.ctypes.data, cap, C.addressof(n_out))
    if rc != 0:
        raise RuntimeError("orc_packed_expand failed: %d" % rc)
    return out[:min(cap, n_out.value)], int(n_out.value)


# ---------------------------------------------------------------------------------------------
# refshape.cc — the reference-SHAPED restatement (string-keyed maps, per-pass graph rebuild)
# ---------------------------------------------------------------------------------------------
_RS = None


def _rs():
    global _RS
    if _RS is None:
        so = os.path.join(_HERE, "_build", "librefshape.so")
        src = os.path.join(_HERE, "refshape.cc")
        if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
            os.makedirs(os.path.dirname(so), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread",
                                   "-I" + os.path.join(_HERE, "..", "include"), src, "-o", so])
        lib = C.CDLL(so)
        lib.orc_refshape_build.restype = C.c_void_p
        lib.orc_refshape_build.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
        lib.orc_refshape_run.restype = C.c_uint64
        lib.orc_refshape_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        lib.orc_refshape_free.restype = None
        lib.orc_refshape_free.argtypes = [C.c_void_p]
        _RS = lib
    return _RS


class RefShapeBatch:
    """Object-form Stories / StoryRuns rebuilt from packed records; run() = one runDagIterations iteration each."""

    def __init__(self, pt: PackedTopologies, L, state: np.ndarray):
        self.pt, self.L, self.n = pt, L, int(state.shape[0])
        self.h = _rs().orc_refshape_build(pt.table.ctypes.data, pt.n_slots, C.addressof(L), self.n, state.ctypes.data)
        if not self.h:
            raise RuntimeError("orc_refshape_build failed (bad slot)")

    def run(self, threads: int = 1):
        result = np.zeros((self.n, self.L.result_stride), dtype=np.uint8)
        evals = _rs().orc_refshape_run(self.h, result.ctypes.data, threads)
        return result, int(evals)

    def close(self):
        if self.h:
            _rs().orc_refshape_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
