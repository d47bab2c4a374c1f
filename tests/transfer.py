"""The records a transfer must leave (bf_resident_transfer, bfh_batch_transfer), restated from the record format, and the host
model of tests/resident_model.py extended by the call: `transfer` over two model batches and TransferRig, for the tests of
test_gpu_transfer.py and the sequences of test_gpu_transfer_sequences.py.  The source side is the model's retire (tests/retire.py),
the re-layout that of tests/reshape.py and tests/narrowing.py in either direction, the fit test narrowing.numpy_extent over one run."""
import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import _pack_planes, pack_state
from tests import reshape as RS
from tests import resident_model as RM
from tests.narrowing import NarrowRig, baseline_runs, numpy_extent

COND, DEC, CHILD = A.F_COND, A.F_DECISION, A.F_CHILD


def relay_state(F, T, state):
    """state records at F -> the same codes packed at T, wider or narrower: header kept, each plane its low words (zero above
    them), planes F lacks zero, planes T lacks gone, the child area its low bytes"""
    n, w = state.shape[0], 32 * T.words
    out = np.zeros((n, T.state_stride), np.uint8)

    def code(name, nbits):
        fo, to = getattr(F, name), getattr(T, name)
        return RS._planes(state, fo, F.words, nbits)[:, :w] if fo != A.OFF_NONE and to != A.OFF_NONE else None
    slots = np.ascontiguousarray(state[:, 0:4]).view("<u4").reshape(n)
    pack_state(T, slots, state[:, 4], RS._planes(state, F.off_phase, F.words, 4)[:, :w], code("off_cond", 2),
               code("off_decision", 2), out=out)
    out[:, 0:16] = state[:, 0:16]
    if T.off_child != A.OFF_NONE:
        out[:, T.off_child:T.off_child + RS._area(T)] = 0
        if F.off_child != A.OFF_NONE:
            nb = min(RS._area(F), RS._area(T))
            out[:, T.off_child:T.off_child + nb] = state[:, F.off_child:F.off_child + nb]
    return out


def relay_result(F, T, result):
    """result records at F -> what a pass at T writes for an unchanged run: header kept, each mask its low words, masks T lacks
    gone, masks only T has zero"""
    out = np.zeros((result.shape[0], T.result_stride), np.uint8)
    out[:, 0:16] = result[:, 0:16]
    for name, nbits in RS.RESULT_FIELDS:
        fo, to = getattr(F, name), getattr(T, name)
        if fo != A.OFF_NONE and to != A.OFF_NONE:
            out[:, to:to + nbits * T.words * 4] = _pack_planes(RS._planes(result, fo, F.words, nbits)[:, :32 * T.words], T.words, nbits)
    return out


def map_slots(state, slot_map):
    """state records (in place) with the topology slot of each header, the first 4 bytes, replaced by slot_map[slot]"""
    w = np.ascontiguousarray(state[:, 0:4]).view("<u4").reshape(-1)
    state[:, 0:4] = np.asarray(slot_map, "<u4")[w.astype(np.int64)].reshape(-1, 1).view(np.uint8)
    return state


def placed(T):
    return (COND if T.off_cond != A.OFF_NONE else 0) | (DEC if T.off_decision != A.OFF_NONE else 0) | \
           (CHILD if T.off_child != A.OFF_NONE else 0)


def run_extent(b, r, n_runs, T):
    """the extent of run r of model batch b alone, as bf_resident_transfer's fit check takes it against layout T"""
    reg = b.reg
    S = {s: reg.stories[k].S for s, k in reg.live.items()}
    C = {s: reg.stories[k].child_nibbles() for s, k in reg.live.items()}
    names = [nm for nm, _ in RS.RESULT_FIELDS if getattr(T, nm) != A.OFF_NONE]
    counted = {0} if r in baseline_runs(b, n_runs) else set()
    e = numpy_extent(b.L, b.state[r:r + 1], b.cur[r:r + 1], 1, S, C, names, counted)
    if e["widest_run"] != A.EXTENT_NO_RUN:
        e["widest_run"] = r
    return e


def fits(e, T):
    return not (e["steps_max"] > T.steps_max or (T.off_child != A.OFF_NONE and e["child_nibbles"] > T.child_nibbles) or
                e["fields"] & ~placed(T))


def slot_reason(src, r, slot_map):
    """bf_resident_transfer_ctx's verdict on the slot of source run r: A.UNFIT_SLOT_PAST_MAP, _UNMAPPED, _DEAD (not live in the
    source's registry) or A.UNFIT_NONE"""
    s = int(np.ascontiguousarray(src.state[r, 0:4]).view("<u4")[0])
    if s >= len(slot_map):
        return A.UNFIT_SLOT_PAST_MAP
    if int(slot_map[s]) == A.SLOT_NONE:
        return A.UNFIT_SLOT_UNMAPPED
    return A.UNFIT_SLOT_DEAD if s not in src.reg.live else A.UNFIT_NONE


def bad_map_entry(src, dst, slot_map):
    """the first entry bf_resident_transfer_ctx refuses the whole call for: a source slot that is live, mapped to a slot that is
    not live in the destination's registry or holds another Story (another packed record) -> slot, or None"""
    for s, t in enumerate(int(x) for x in slot_map):
        if t != A.SLOT_NONE and s in src.reg.live and (t not in dst.reg.live or dst.reg.live[t] != src.reg.live[s]):
            return s
    return None


def transfer(src, dst, src_n, dst_n, runs, slot_map=None):
    """bf_resident_transfer over two model batches -> dict(src_n_runs, dst_n_runs, moves_from, moves_to).  A refusal raises
    RM.Refused with .unfit (and .why for a fit refusal).  slot_map: bf_resident_transfer_ctx, src and dst in two ctxs with their
    own registries: the map's entries are checked once the runs are, a run's slot verdict (.reason, A.UNFIT_*) counts with its
    fit in the order of runs, and each arrival's header slot is slot_map[its source slot]; the rest is the rule of one ctx"""
    runs = [int(r) for r in runs]

    def refuse(why, unfit=A.EXTENT_NO_RUN, e=None, reason=A.UNFIT_NONE):
        err = RM.Refused(A.BF_EINVAL, why)
        err.unfit, err.why, err.reason = unfit, e, reason
        return err
    if src is dst:
        raise refuse("a transfer from a batch to itself")
    if src_n > src.cap:
        raise refuse("src_n_runs exceeds the source batch")
    if dst_n + len(runs) > dst.cap:
        raise refuse("dst_n_runs + n exceeds the destination batch")
    if any(r >= src_n for r in runs) or len(set(runs)) != len(runs):
        raise refuse("runs")
    if runs and slot_map is not None and bad_map_entry(src, dst, slot_map) is not None:
        raise refuse("slot_map[%d]" % bad_map_entry(src, dst, slot_map))
    F, T = src.L, dst.L
    for i, r in enumerate(runs):
        why = A.UNFIT_NONE if slot_map is None else slot_reason(src, r, slot_map)
        if why != A.UNFIT_NONE:
            raise refuse("run %d: its slot" % r, i, None, why)
        e = run_extent(src, r, src_n, T)
        if not fits(e, T):
            raise refuse("run %d does not fit" % r, i, e, A.UNFIT_LAYOUT)
    if not runs:
        return {"src_n_runs": src_n, "dst_n_runs": dst_n, "moves_from": np.zeros(0, np.uint32), "moves_to": np.zeros(0, np.uint32)}
    ix, n = np.asarray(runs, np.int64), len(runs)
    st, cur = relay_state(F, T, src.state[ix]), relay_result(F, T, src.cur[ix])
    if slot_map is not None:
        map_slots(st, slot_map)
    src_baseline = src.prev_valid and all(r < src.prev_runs for r in runs)
    m, mf, mt = src.retire(src_n, runs, 0)
    dst._end_snapshot()
    dst.state[dst_n:dst_n + n], dst.cur[dst_n:dst_n + n] = st, cur
    new = set(range(dst_n, dst_n + n))
    dst.touched |= new
    dst.must |= new
    dst.uploaded |= {i for i in new if i >= dst.full_runs}
    if dst.prev_valid and dst.prev_runs == dst_n and src_baseline:
        dst.prev_runs = dst_n + n
    else:
        dst.prev_valid = False
    return {"src_n_runs": m, "dst_n_runs": dst_n + n, "moves_from": mf, "moves_to": mt}


class TransferRig(NarrowRig):
    """NarrowRig whose batches also take transfers between them, each checked against the model"""

    def transfer(self, src, dst, src_n, dst_n, runs):
        self.log.append("transfer b%d -> b%d n %d / %d runs %d" % (self.handles[src], self.handles[dst], src_n, dst_n, len(runs)))
        try:
            want, refused = transfer(src, dst, src_n, dst_n, runs), None
        except RM.Refused as e:
            want, refused = None, e
        try:
            got, status = self.fr.resident_transfer(self.handles[src], self.handles[dst], src_n, dst_n, np.asarray(runs, np.uint32)), A.BF_OK
        except A.FrontierError as d:
            got, status = d, d.status
        self.check(status == (refused.status if refused else A.BF_OK),
                   "transfer status %d, the model says %s" % (status, refused or "accept"))
        if refused is not None:
            self.check(got.unfit == refused.unfit, "unfit %d, want %d" % (got.unfit, refused.unfit))
            if refused.why is not None:
                self.check(got.why == refused.why, "why %s, want %s" % (got.why, refused.why))
        else:
            for k in ("src_n_runs", "dst_n_runs"):
                self.check(got[k] == want[k], "%s %d, want %d" % (k, got[k], want[k]))
            for k in ("moves_from", "moves_to"):
                self.check(np.array_equal(got[k], want[k]), "%s differ" % k)
        self.sync()
        return want

    def transfer_ctx(self, dst_rig, src, dst, src_n, dst_n, runs, slot_map):
        """bf_resident_transfer_ctx from batch src of this rig's ctx to batch dst of dst_rig's, against the model: status,
        unfit, unfit_reason, the extent of a fit refusal, counts and moves; then both ctxs' batches against their models"""
        self.log.append("transfer_ctx b%d -> ctx b%d n %d / %d runs %d map %d" % (self.handles[src], dst_rig.handles[dst], src_n,
                                                                                 dst_n, len(runs), len(slot_map)))
        try:
            want, refused = transfer(src, dst, src_n, dst_n, runs, slot_map), None
        except RM.Refused as e:
            want, refused = None, e
        try:
            got, status = self.fr.resident_transfer_ctx(dst_rig.fr, self.handles[src], dst_rig.handles[dst], src_n, dst_n,
                                                        np.asarray(runs, np.uint32), slot_map), A.BF_OK
        except A.FrontierError as d:
            got, status = d, d.status
        self.check(status == (refused.status if refused else A.BF_OK),
                   "transfer_ctx status %d, the model says %s (%s)" % (status, refused or "accept", got if status else ""))
        if refused is not None:
            self.check(got.unfit == refused.unfit, "unfit %d, want %d (%s)" % (got.unfit, refused.unfit, got))
            self.check(got.unfit_reason == refused.reason, "unfit_reason %d, want %d" % (got.unfit_reason, refused.reason))
            if refused.why is not None:
                self.check(got.why == refused.why, "why %s, want %s" % (got.why, refused.why))
        else:
            for k in ("src_n_runs", "dst_n_runs"):
                self.check(got[k] == want[k], "%s %d, want %d" % (k, got[k], want[k]))
            for k in ("moves_from", "moves_to"):
                self.check(np.array_equal(got[k], want[k]), "%s differ" % k)
        self.sync()
        dst_rig.sync()
        return want
