"""The records a reshape must leave (bf_resident_reshape, bfh_batch_reshape), restated from the record format alone: every code of
the old records is unpacked and packed again at the new layout, and every result mask likewise."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import _pack_planes, _unpack_planes, pack_state


def _area(L):
    """bytes of the child area the layout reserves (whole u32 words)"""
    return ((L.child_nibbles + 1) // 2 + 3) // 4 * 4


def _planes(raw, off, W, nbits):
    """every code of a plane field, padding steps included: [N, 32 * W]"""
    return _unpack_planes(np.ascontiguousarray(raw[:, off:off + nbits * W * 4]), W, nbits, 32 * W)


def reshape_state(F, T, state, capacity):
    """state [n, F.state_stride] -> [capacity, T.state_stride]: codes packed again at T (zero for a field F lacks), the header and
    the child area's old bytes kept, runs from n on zero"""
    n, Wo = state.shape[0], F.words
    out = np.zeros((capacity, T.state_stride), np.uint8)
    code = lambda off, nbits: _planes(state, off, Wo, nbits) if off != A.OFF_NONE else None   # noqa: E731
    slots = np.ascontiguousarray(state[:, 0:4]).view("<u4").reshape(n)
    pack_state(T, slots, state[:, 4], _planes(state, F.off_phase, Wo, 4), code(F.off_cond, 2), code(F.off_decision, 2),
               out=out[:n])
    out[:n, 0:16] = state[:, 0:16]
    if F.off_child != A.OFF_NONE:
        nb = _area(F)
        out[:n, T.off_child:T.off_child + nb] = state[:, F.off_child:F.off_child + nb]
    return out


RESULT_FIELDS = (("off_ready", 1), ("off_skip", 1), ("off_fail", 1), ("off_needs_cond", 1), ("off_skip_dep", 1), ("off_phase_out", 4))


def reshape_result(F, T, result, capacity):
    """result records [n, F.result_stride] -> [capacity, T.result_stride]: header kept, each mask / phase_out plane packed again
    at T's width, the masks of an output field F lacks zero, runs from n on zero"""
    n = result.shape[0]
    out = np.zeros((capacity, T.result_stride), np.uint8)
    out[:n, 0:16] = result[:, 0:16]
    for name, nbits in RESULT_FIELDS:
        fo, to = getattr(F, name), getattr(T, name)
        if fo != A.OFF_NONE:
            out[:n, to:to + nbits * T.words * 4] = _pack_planes(_planes(result, fo, F.words, nbits), T.words, nbits)
    return out
