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


def transfer(src, dst, src_n, dst_n, runs):
    """bf_resident_transfer over two model batches -> dict(src_n_runs, dst_n_runs, moves_from, moves_to).  A refusal raises
    RM.Refused with .unfit (and .why for a fit refusal)"""
    runs = [int(r) for r in runs]

    def refuse(why, unfit=A.EXTENT_NO_RUN, e=None):
        err = RM.Refused(A.BF_EINVAL, why)
        err.unfit, err.why = unfit, e
        return err
    if src is dst:
        raise refuse("a transfer from a batch to itself")
    if src_n > src.cap:
        raise refuse("src_n_runs exceeds the source batch")
    if dst_n + len(runs) > dst.cap:
        raise refuse("dst_n_runs + n exceeds the destination batch")
    if any(r >= src_n for r in runs) or len(set(runs)) != len(runs):
        raise refuse("runs")
    F, T = src.L, dst.L
    for i, r in enumerate(runs):
        e = run_extent(src, r, src_n, T)
        if not fits(e, T):
            raise refuse("run %d does not fit" % r, i, e)
    if not runs:
        return {"src_n_runs": src_n, "dst_n_runs": dst_n, "moves_from": np.zeros(0, np.uint32), "moves_to": np.zeros(0, np.uint32)}
    ix, n = np.asarray(runs, np.int64), len(runs)
    st, cur = relay_state(F, T, src.state[ix]), relay_result(F, T, src.cur[ix])
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
