"""The journal of a tick commit (bf_resident_commit_journal), written from the contract in include/bobrafrontier.h: what the
commit wrote, read off as the byte difference of the state records and timer slots before and after it.

States are the uint8 arrays of tests/packing.py (one row per run), timer areas the (capacity, K) uint64 arrays of tests/timers.py
(None: no arming).  Items are (run, index, field, code, before, after) tuples, the fields of bf_commit_write."""
import numpy as np

from bobrapet_b200 import _abi as A
from tests import timers as T

PHASE, REGISTERED, TIMER = A.DELTA_PHASE, A.DELTA_REGISTERED, A.COMMIT_WRITE_TIMER


def _nibbles(row, L):
    """the stored phase nibble of every step of the layout (15 as stored)"""
    w = row[L.off_phase:L.off_phase + 16 * L.words].view("<u4").reshape(4, L.words)
    bits = [np.unpackbits(w[b].view(np.uint8), bitorder="little") for b in range(4)]
    return bits[0] | bits[1] << 1 | bits[2] << 2 | bits[3] << 3


def journal(L, before, after, n_runs, area_before=None, area_after=None):
    """-> (items sorted by (run, field, index), ascending runs whose record changed) of a commit over runs [0, n_runs)"""
    items, runs = [], []
    for r in range(n_runs):
        changed = not np.array_equal(before[r], after[r])
        if changed:
            runs.append(r)
            nb, na = _nibbles(before[r], L), _nibbles(after[r], L)
            items += [(r, int(s), PHASE, 0, int(nb[s]), int(na[s])) for s in np.nonzero(nb != na)[0]]
            rb, ra = int(before[r][8:16].view("<u8")[0]), int(after[r][8:16].view("<u8")[0])
            assert rb & ~ra == 0, "a commit only sets registered bits"
            items += [(r, q, REGISTERED, 0, 0, 1) for q in range(64) if (ra & ~rb) >> q & 1]
        if area_before is not None:
            old = {s for s, _d, _c in T.armed(area_before[r])}
            items += [(r, s, TIMER, c, T.NONE, d) for s, d, c in sorted(T.armed(area_after[r])) if s not in old]
    return items, runs


def as_tuples(arr):
    """COMMIT_WRITE_DTYPE rows -> item tuples"""
    return [(int(x["run"]), int(x["index"]), int(x["field"]), int(x["code"]), int(x["before"]), int(x["after"])) for x in arr]
