"""The records and the extent a narrow must leave (bf_resident_extent / bf_resident_narrow), restated from the record format, and
the host model of tests/resident_model.py extended by the call: NarrowBatch and NarrowRig, for the sequences of
test_gpu_narrow_sequences.py."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import _pack_planes, pack_state
from tests import randgen
from tests import reshape as RS
from tests import resident_model as RM
from tests.seqrig import Rig

COND, DEC, CHILD = A.F_COND, A.F_DECISION, A.F_CHILD


def narrow_state(F, T, state):
    """state records at F -> the same codes packed at the narrower T: header kept, each plane its low T.words words, the child
    area its low bytes, the planes of a field T lacks gone"""
    n, w = state.shape[0], 32 * T.words
    out = np.zeros((n, T.state_stride), np.uint8)
    code = lambda off, toff, nbits: RS._planes(state, off, F.words, nbits)[:, :w] if toff != A.OFF_NONE else None  # noqa: E731
    slots = np.ascontiguousarray(state[:, 0:4]).view("<u4").reshape(n)
    pack_state(T, slots, state[:, 4], code(F.off_phase, T.off_phase, 4), code(F.off_cond, T.off_cond, 2),
               code(F.off_decision, T.off_decision, 2), out=out)
    out[:, 0:16] = state[:, 0:16]
    if T.off_child != A.OFF_NONE:
        nb = RS._area(T)
        out[:, T.off_child:T.off_child + nb] = state[:, F.off_child:F.off_child + nb]
    return out


def narrow_result(F, T, result):
    """result records at F -> what a pass at T writes for an unchanged run: header kept, kept masks truncated, dropped ones gone"""
    out = np.zeros((result.shape[0], T.result_stride), np.uint8)
    out[:, 0:16] = result[:, 0:16]
    for name, nbits in RS.RESULT_FIELDS:
        fo, to = getattr(F, name), getattr(T, name)
        if fo != A.OFF_NONE and to != A.OFF_NONE:
            out[:, to:to + nbits * T.words * 4] = _pack_planes(RS._planes(result, fo, F.words, nbits)[:, :32 * T.words], T.words, nbits)
    return out


def topo_child_nibbles(ts):
    """the child area each topology needs (bf_topology_put rounds it to 8 nibbles)"""
    cfs, _ = randgen.child_layout(ts)
    out, pos = [], 0
    for i in range(ts.count):
        p = int(ts.P[i])
        br = ts.parallel["branches"][pos:pos + p].astype(np.int64)
        out.append(int((int(cfs[i][-1]) + int(br[-1]) + 7) // 8 * 8) if p else 0)
        pos += p
    return np.asarray(out, np.int64)


def numpy_extent(L, state, result, n_runs, slot_S, slot_child, result_fields=None, counted=None):
    """bf_resident_extent restated: slot_S / slot_child map a slot id to its S / child area (alive slots only); counted: the runs
    whose result record counts (default: every run below n_runs, as after a full tick over them)"""
    cap, W = state.shape[0], L.words
    steps = np.zeros(cap, np.int64)
    child = np.zeros(cap, np.int64)
    fields = 0
    idx = np.arange(32 * W)[None, :]

    def top(codes):
        return np.where(codes.any(axis=1), np.where(codes != 0, idx + 1, 0).max(axis=1), 0)
    for off, nbits, f in ((L.off_phase, 4, 0), (L.off_cond, 2, COND), (L.off_decision, 2, DEC)):
        if off == A.OFF_NONE:
            continue
        codes = RS._planes(state, off, W, nbits)
        steps = np.maximum(steps, top(codes))
        if codes.any():
            fields |= f
    if L.off_child != A.OFF_NONE and L.child_nibbles:
        raw = state[:, L.off_child:L.off_child + (L.child_nibbles + 1) // 2]
        nib = np.stack([raw & 0xF, raw >> 4], axis=2).reshape(cap, -1)[:, :L.child_nibbles]
        child = np.where(nib.any(axis=1), np.where(nib != 0, np.arange(L.child_nibbles)[None, :] + 1, 0).max(axis=1), 0)
        if nib.any():
            fields |= CHILD
    names = [nm for nm, _ in RS.RESULT_FIELDS] if result_fields is None else result_fields
    rows = np.arange(n_runs) if counted is None else np.asarray(sorted(counted), np.int64)
    for name, nbits in RS.RESULT_FIELDS:
        off = getattr(L, name)
        if off != A.OFF_NONE and name in names and len(rows):
            steps[rows] = np.maximum(steps[rows], top(RS._planes(result[rows], off, W, nbits)))
    slots = np.ascontiguousarray(state[:n_runs, 0:4]).view("<u4").reshape(n_runs)
    for r, s in enumerate(slots.tolist()):
        if s in slot_S:
            steps[r] = max(steps[r], slot_S[s])
            child[r] = max(child[r], slot_child[s])
    smax = int(steps.max()) if cap else 0
    return {"steps_max": max(1, smax), "child_nibbles": int(child.max()) if cap else 0, "fields": fields,
            "widest_run": int(np.argmax(steps == smax)) if smax else A.EXTENT_NO_RUN}



def baseline_runs(b, n_runs):
    """the runs below n_runs whose current result record a later tick compares with (bf_resident_extent): the changed-only
    baseline, and unless the next touched tick is full the touched one (the last full tick's runs and the uploaded runs from
    there on that a touched tick evaluated), without the runs still to be listed whatever their record holds"""
    rows = set(range(min(b.prev_runs, n_runs))) if b.prev_valid else set()
    if not b.need_full:
        end = b.full_runs
        while end in b.uploaded:
            end += 1
        rows |= {r for r in range(min(end, n_runs)) if r not in b.must}
    return rows


class NarrowBatch(RM.Batch):
    """RM.Batch with bf_resident_extent and bf_resident_narrow"""

    def extent(self, n_runs, T=None):
        reg = self.reg
        S = {s: reg.stories[k].S for s, k in reg.live.items()}
        C = {s: reg.stories[k].child_nibbles() for s, k in reg.live.items()}
        names = None if T is None else [nm for nm, _ in RS.RESULT_FIELDS if getattr(T, nm) != A.OFF_NONE]
        return numpy_extent(self.L, self.state, self.cur, n_runs, S, C, names, baseline_runs(self, n_runs))

    def narrow(self, T, n_runs):
        F = self.L
        if n_runs > self.cap:
            raise RM.Refused(A.BF_EINVAL, "n_runs exceeds the resident batch")

        def refuse(why, e):
            err = RM.Refused(A.BF_EINVAL, why)
            err.extent = e
            return err
        if (T.steps_max > F.steps_max or T.fields & ~F.fields or
                (F.off_child != A.OFF_NONE and T.off_child != A.OFF_NONE and T.child_nibbles > F.child_nibbles)):
            raise refuse("narrow grows a dimension", self.extent(n_runs))
        e = self.extent(n_runs, T)
        if T.as_dict() == F.as_dict():
            return e
        placed = (COND if T.off_cond != A.OFF_NONE else 0) | (DEC if T.off_decision != A.OFF_NONE else 0) | \
                 (CHILD if T.off_child != A.OFF_NONE else 0)
        if (T.steps_max < e["steps_max"] or (T.off_child != A.OFF_NONE and T.child_nibbles < e["child_nibbles"]) or
                e["fields"] & ~placed):
            raise refuse("below the extent", e)
        self._end_snapshot()
        self.state, self.cur = narrow_state(F, T, self.state), narrow_result(F, T, self.cur)
        dropped = [n for n in ("off_decision", "off_child", "off_fail", "off_needs_cond", "off_skip_dep", "off_phase_out")
                   if getattr(F, n) != A.OFF_NONE and getattr(T, n) == A.OFF_NONE]
        self.L = T
        self.full_runs = min(self.full_runs, n_runs)
        if self.prev_runs > n_runs:
            self.prev_valid = False
        if dropped:
            self.need_full = True
        return e


class NarrowRig(Rig):
    """Rig whose batches take extents and narrows, each checked against the model"""

    def create(self, L, cap):
        b = NarrowBatch(self.reg, L, cap)
        self.handles[b] = self.fr.resident_create(L, cap)
        self.log.append("create batch %d cap %d S %d" % (self.handles[b], cap, L.steps_max))
        return b

    def extent(self, b, n_runs):
        self.log.append("extent b%d n %d" % (self.handles[b], n_runs))
        got, want = self.fr.resident_extent(self.handles[b], n_runs), b.extent(n_runs)
        self.check(got == want, "extent %s, want %s" % (got, want))
        return got

    def narrow(self, b, T, n_runs):
        self.log.append("narrow b%d n %d S %d -> %d child %d -> %d fields %#x -> %#x" % (
            self.handles[b], n_runs, b.L.steps_max, T.steps_max, b.L.child_nibbles, T.child_nibbles, b.L.fields, T.fields))
        try:
            want, refused = b.narrow(T, n_runs), None
        except RM.Refused as e:
            want, refused = getattr(e, "extent", None), e
        try:
            got, status = self.fr.resident_narrow(self.handles[b], T, n_runs), A.BF_OK
        except A.FrontierError as d:
            got, status = getattr(d, "extent", None), d.status
        self.check(status == (refused.status if refused else A.BF_OK),
                   "narrow status %d, the model says %s" % (status, refused or "accept"))
        if want is not None:
            self.check(got == want, "narrow extent %s, want %s" % (got, want))
        self.sync()
        return refused is None
