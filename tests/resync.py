"""A host model of bf_resident_resync, written from the contract in include/bobrafrontier.h ("resyncs").

State records are the uint8 arrays of tests/packing.py (one row per run).  The phases after stages G, H and I come the way
tests/runstatus.py gets them: the packed oracle's single pass with BF_F_OUT_PHASE | BF_F_OUT_FAIL, the steps of its fail mask
(stage D's cond-FAIL writes) set back to their input codes.  runctl is a run-control area (tests/runctl.py) or None.  Nothing here
changes its arguments."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from oracle import packed as PK
from oracle.packed import child_first_of
from tests.runstatus import IN_FIELDS, _codes, _mask

DRIFT_DTYPE = Frontier.DRIFT_DTYPE
F = A.resync_field
TERMINAL = (3, 4, 5, 6, 7, 11, 12, 13)   # BF_LUT_TERMINAL (0x38F8)


def _codes2(row, off, words, S):
    w = np.frombuffer(row[off:off + 8 * words].tobytes(), "<u4").reshape(2, words)
    bits = np.unpackbits(w.view(np.uint8).reshape(2, words * 4), axis=1, bitorder="little")[:, :S]
    return (bits[0] | bits[1] << 1).astype(np.uint8)


def _nibbles(row, off, n):
    b = row[off:off + (n + 1) // 2]
    c = np.zeros(2 * b.size, np.uint8)
    c[0::2], c[1::2] = b & 0xF, b >> 4
    c = c[:n]
    c[c == 15] = 0
    return c


def _reg(row):
    return int(row[8:16].view("<u8")[0])


class Topos:
    """S, the parallel descs (step, branches, child_first) and the slot of every topology of a TopologySet put at `slots`"""

    def __init__(self, ts, slots):
        self.ts, self.slots = ts, np.asarray(slots, dtype=np.uint32)
        self.info = {}
        pos = 0
        for i in range(ts.count):
            p = int(ts.P[i])
            par = ts.parallel[pos:pos + p] if p else None
            br = par["branches"].astype(np.int64) if p else np.zeros(0, np.int64)
            cf = child_first_of(br) if p else np.zeros(0, np.uint32)
            steps = par["step"].astype(np.int64) if p else np.zeros(0, np.int64)
            self.info[int(self.slots[i])] = (int(ts.S[i]), steps, br, cf.astype(np.int64))
            pos += p


def post_phases(L, topos, rows):
    """the phases of steps [0, S) of each row after a single pass's stages G, H and I (None for a dead slot or one wider than the
    layout), as bf_resident_status takes them"""
    # the width of the layout, not its steps_max: a slot whose S passes steps_max but not 32 * words fits it on the device (the
    # records are laid out by words alone)
    L2 = make_layout(32 * L.words, L.child_nibbles, (L.fields & IN_FIELDS) | A.F_OUT_PHASE | A.F_OUT_FAIL)
    assert L2.state_stride == L.state_stride and L2.off_phase == L.off_phase
    out = [None] * len(rows)
    slot_of = [int(r[:4].view("<u4")[0]) for r in rows]
    alive = [k for k, sl in enumerate(slot_of) if sl in topos.info and (topos.info[sl][0] + 31) // 32 <= L.words]
    if not alive:
        return out
    res = PK.evaluate(PK.PackedTopologies(topos.ts, topos.slots), L2, np.ascontiguousarray(np.asarray(rows)[alive]))[0]
    for j, k in enumerate(alive):
        S = topos.info[slot_of[k]][0]
        ph = _codes(res[j], L2.off_phase_out, L.words, S)
        fail = _mask(res[j], L2.off_fail, L.words, S)
        ph[fail] = _codes(rows[k], L.off_phase, L.words, S)[fail]
        out[k] = ph
    return out


def effective_fields(L, fields):
    if L.off_cond == A.OFF_NONE:
        fields &= ~F(A.DELTA_COND)
    if L.off_decision == A.OFF_NONE:
        fields &= ~F(A.DELTA_DECISION)
    if L.off_child == A.OFF_NONE:
        fields &= ~F(A.DELTA_CHILD)
    return fields


def _merged(L, dev, rec, fields, stopped):
    """the caller's record as the repair would leave it, without its slot: the device's record with the caller's codes in the
    selected fields, and for a stopped run the stopped flags byte"""
    m = dev.copy()
    W = L.words
    for f, off, nb in ((A.DELTA_PHASE, L.off_phase, 16), (A.DELTA_COND, L.off_cond, 8), (A.DELTA_DECISION, L.off_decision, 8)):
        if fields & F(f):
            m[off:off + nb * W] = rec[off:off + nb * W]
    if fields & F(A.DELTA_CHILD):
        nb = (L.child_nibbles + 7) // 8 * 4
        m[L.off_child:L.off_child + nb] = rec[L.off_child:L.off_child + nb]
    if fields & F(A.DELTA_REGISTERED):
        m[8:16] = rec[8:16]
    if fields & F(A.DELTA_RUN_FLAGS) and not stopped:
        m[4] = rec[4]
    return m


def compare(L, topos, dev_rows, records, runs, fields, runctl=None):
    """-> the items (DRIFT_DTYPE) of the listed runs, ordered by (run, field, index)"""
    fields = effective_fields(L, fields)
    W = L.words
    items = []
    stopped = [runctl is not None and int(runctl[r]["stop"]) != 0 for r in runs]
    merged = [_merged(L, dev_rows[k], records[k], fields, stopped[k]) for k in range(len(runs))]
    dev_post = post_phases(L, topos, [dev_rows[k] for k in range(len(runs))])
    rec_post = post_phases(L, topos, merged)
    for k, r in enumerate(runs):
        dev, rec = dev_rows[k], records[k]
        sd, sr = int(dev[:4].view("<u4")[0]), int(rec[:4].view("<u4")[0])
        if sd != sr:
            items.append((r, 0, A.DELTA_TOPO_SLOT, 0, sd, sr))
            continue
        live = dev_post[k] is not None
        if live:
            S, steps, br, cf = topos.info[sd]
            a, b = dev_post[k], rec_post[k]
            nt = ~(np.isin(a, TERMINAL) & np.isin(b, TERMINAL))
            dmask = np.zeros(64, bool)
            dmask[:steps.size] = nt[steps]
        else:
            S = 32 * W
            a, b = _codes(dev, L.off_phase, W, S), _codes(merged[k], L.off_phase, W, S)
            nt = np.ones(S, bool)
            dmask = np.ones(64, bool)
        if fields & F(A.DELTA_PHASE):
            for s in np.flatnonzero(a != b):
                items.append((r, s, A.DELTA_PHASE, 0, a[s], b[s]))
        for f, off in ((A.DELTA_COND, L.off_cond), (A.DELTA_DECISION, L.off_decision)):
            if fields & F(f):
                x, y = _codes2(dev, off, W, S), _codes2(rec, off, W, S)
                for s in np.flatnonzero((x != y) & nt):
                    items.append((r, s, f, 0, x[s], y[s]))
        if fields & F(A.DELTA_CHILD):
            x, y = _nibbles(dev, L.off_child, L.child_nibbles), _nibbles(rec, L.off_child, L.child_nibbles)
            cmp = np.zeros(L.child_nibbles, bool)
            if live:
                for q in np.flatnonzero(dmask[:steps.size]):
                    cmp[cf[q]:min(cf[q] + br[q], L.child_nibbles)] = True
            else:
                cmp[:] = True
            for c in np.flatnonzero((x != y) & cmp):
                items.append((r, c, A.DELTA_CHILD, 0, x[c], y[c]))
        if fields & F(A.DELTA_RUN_FLAGS):
            fd = int(runctl[r]["saved_flags"]) if stopped[k] else int(dev[4])
            if fd != int(rec[4]):
                items.append((r, 0, A.DELTA_RUN_FLAGS, 0, fd, int(rec[4])))
        if fields & F(A.DELTA_REGISTERED):
            x, y = _reg(dev), _reg(rec)
            for q in range(64):
                if dmask[q] and ((x ^ y) >> q) & 1:
                    items.append((r, q, A.DELTA_REGISTERED, 0, (x >> q) & 1, (y >> q) & 1))
    out = np.zeros(len(items), dtype=DRIFT_DTYPE)
    for i, (r, idx, f, _, d, v) in enumerate(items):
        out[i] = (r, idx, f, 0, d, v)
    return out


def resync(L, topos, state, records, n_runs, runs=None, fields=A.RESYNC_ALL_FIELDS, check=False, runctl=None):
    """-> (items, drifted runs, state after, runctl after) of bf_resident_resync over the device records `state` (the whole batch)
    and the caller's `records` (one per listed run)"""
    runs = np.arange(n_runs, dtype=np.uint32) if runs is None else np.asarray(runs, dtype=np.uint32)
    records = np.asarray(records, dtype=np.uint8)
    items = compare(L, topos, state[runs], records, runs, fields, runctl)
    drifted = np.unique(items["run"]).astype(np.uint32)
    st = state.copy()
    rc = None if runctl is None else runctl.copy()
    if check:
        return items, drifted, st, rc
    f = effective_fields(L, fields)
    pos = {int(r): k for k, r in enumerate(runs)}
    W = L.words
    for r in drifted:
        k = pos[int(r)]
        rec = records[k]
        stopped = rc is not None and int(rc[r]["stop"]) != 0
        if int(st[r][:4].view("<u4")[0]) != int(rec[:4].view("<u4")[0]):
            st[r] = rec
            if stopped:
                rc[r]["saved_flags"] = rec[4]
                st[r][4] = A.RF_HOST_GROUP | A.GROUP_DONE << A.RF_HOST_GROUP_SHIFT
            continue
        for fl, off, nb in ((A.DELTA_PHASE, L.off_phase, 16), (A.DELTA_COND, L.off_cond, 8), (A.DELTA_DECISION, L.off_decision, 8)):
            if f & F(fl):
                st[r][off:off + nb * W] = rec[off:off + nb * W]
        if f & F(A.DELTA_CHILD):
            nb = (L.child_nibbles + 7) // 8 * 4
            st[r][L.off_child:L.off_child + nb] = rec[L.off_child:L.off_child + nb]
        if f & F(A.DELTA_REGISTERED):
            st[r][8:16] = rec[8:16]
        if f & F(A.DELTA_RUN_FLAGS):
            if stopped:
                rc[r]["saved_flags"] = rec[4]
            else:
                st[r][4] = rec[4]
    return items, drifted, st, rc


def slot_drifted(items):
    """the runs whose only item is a slot drift"""
    return np.unique(items["run"][items["field"] == A.DELTA_TOPO_SLOT]).astype(np.uint32)
