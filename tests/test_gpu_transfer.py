"""bf_resident_transfer: live runs move from one resident batch to another of the same ctx, re-laid to the destination's layout.
Every call goes to the device and to the host model of tests/transfer.py side by side (TransferRig): both batches' state records
and the moves after each transfer, every refusal's status, unfit position and extent, and the ticks that follow on both batches
(touched: listed runs, heads, events and `full`; changed-only; dense ticks single pass and fixpoint, which the model computes
with the packed oracle)."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200 import host as H
from bobrapet_b200.records import make_layout
from tests import migration as M
from tests.seqrig import NONE, random_records, story_pool
from tests.test_gpu_resident_sequences import _deltas
from tests.test_host_reshape import _fill, _host_story
from tests.transfer import TransferRig, relay_state, run_extent

pytestmark = pytest.mark.gpu

COND, DEC, CHILD, OUT = A.F_COND, A.F_DECISION, A.F_CHILD, A.F_ALL_OUT
INPUTS = COND | DEC | CHILD

# (source steps_max, source fields, destination steps_max, destination fields, Story steps lo, hi)
PAIRS = {"64-to-256": (64, 0, 256, COND | DEC | CHILD | OUT, 20, 60),
         "256-to-1024": (256, COND | CHILD | A.F_OUT_FAIL, 1024, COND | DEC | CHILD | OUT, 100, 250),
         "1024-to-64": (1024, COND | DEC | CHILD | OUT, 64, CHILD | A.F_OUT_SKIP_DEP, 20, 60),
         "equal": (256, COND | DEC | CHILD | OUT, 256, COND | DEC | CHILD | OUT, 100, 250)}
SIZES = [(1, 0), (512, 1), (2048, 512), (512, 2048)]   # runs of the source, runs of the destination


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _layouts(pool, pair):
    s_src, f_src, s_dst, f_dst, _, _ = PAIRS[pair]
    child = max(p.child_nibbles() for p in pool)
    Ls = make_layout(s_src, child + 8 if f_src & CHILD else 0, f_src)
    Ld = make_layout(s_dst, child if f_dst & CHILD else 0, f_dst)
    # the codes the runs hold: only in the input fields both layouts have, so that every run fits the destination
    Lg = make_layout(s_src, Ls.child_nibbles, f_src & f_dst & INPUTS)
    return Ls, Ld, Lg


def _records(rng, rig, Lg, L, slots, n):
    story = rng.integers(0, len(slots), n)
    recs = random_records(rng, Lg, [rig.reg.story(slots[k]) for k in story], [slots[k] for k in story])
    return relay_state(Lg, L, recs)


@pytest.mark.parametrize("dead", [False, True])
@pytest.mark.parametrize("sizes", SIZES, ids=["%d-%d" % s for s in SIZES])
@pytest.mark.parametrize("pair", list(PAIRS))
def test_transfer_records_ticks_and_parity(fr, pair, sizes, dead):
    n_src, n_dst = sizes
    seed = 100 * list(PAIRS).index(pair) + 10 * SIZES.index(sizes) + dead
    rng = np.random.default_rng(7000 + seed)
    lo, hi = PAIRS[pair][4:]
    pool = story_pool(rng, lo, hi, 2, 3)
    rig = TransferRig(fr, pool, "transfer %s %s dead %d" % (pair, sizes, dead))
    slots = [rig.put(k) for k in range(3)] + [rig.put(len(pool) - 1)]   # the last one is dropped for `dead`
    Ls, Ld, Lg = _layouts(pool, pair)
    k = max(1, n_src // 3) if n_src > 1 else 1
    runs = rng.choice(n_src, size=k, replace=False).astype(np.uint32)
    try:
        # A1 / B1 take touched ticks after the transfer, A2 / B2 (the same calls before it) changed-only ticks
        A1, A2 = rig.create(Ls, n_src + 8), rig.create(Ls, n_src + 8)
        B1, B2 = rig.create(Ld, n_dst + k + 8), rig.create(Ld, n_dst + k + 8)
        src_recs = _records(rng, rig, Lg, Ls, slots, n_src)
        dst_recs = _records(rng, rig, Lg, Ld, slots, n_dst)
        for a in (A1, A2):
            rig.upload(a, 0, src_recs)
        for b in (B1, B2):
            if n_dst:
                rig.upload(b, 0, dst_recs)
        d_src = _phase_only(_deltas(rng, rig, A1, n_src, 60), min(lo, Ld.steps_max))
        for a in (A1, A2):
            rig.tick(a, "touched", n_src)
            rig.apply(a, d_src)
        for b in (B1, B2):
            rig.tick(b, "changed", n_dst)
        if dead:
            rig.drop(slots[3])
        for a, b in ((A1, B1), (A2, B2)):
            out = rig.transfer(a, b, n_src, n_dst, runs)
            assert out is not None and out["dst_n_runs"] == n_dst + k
        m = n_src - k
        o = rig.tick(A1, "touched", m)
        p = rig.tick(B1, "touched", n_dst + k)
        if not dead:   # the transfer forces no full tick on either side
            assert o["full"] == 0 and p["full"] == 0
            assert set(range(n_dst, n_dst + k)) <= set(p["runs"].tolist())
        rig.tick(B2, "changed", n_dst + k)
        rig.tick(A2, "changed", m)
        for b in (B1, B2):   # parity: the arrivals evaluate as the packed oracle says on their re-laid records
            rig.tick(b, "dense", n_dst + k)
            rig.tick(b, "dense", n_dst + k, flags=A.EVAL_FIXPOINT)
        # the other way back, into the source's layout
        back = rng.choice(n_dst + k, size=min(3, n_dst + k), replace=False).astype(np.uint32)
        rig.transfer(B1, A1, n_dst + k, m, back)
        rig.tick(A1, "touched", m + len(back))
        rig.tick(B1, "touched", n_dst + k - len(back))
    finally:
        rig.destroy()


def _phase_only(d, steps):
    """phase deltas inside the Stories' common width, run flags and registered bits: the codes every destination holds"""
    keep = np.isin(d["field"], [A.DELTA_RUN_FLAGS, A.DELTA_REGISTERED]) | ((d["field"] == A.DELTA_PHASE) & (d["index"] < steps))
    return d[keep]


def test_transfer_refusals_change_nothing(fr):
    rng = np.random.default_rng(7901)
    pool = story_pool(rng, 20, 60, 2, 2) + story_pool(rng, 90, 120, 1, 1)[:1]   # the last Story is wider than 64 steps
    rig = TransferRig(fr, pool, "transfer refusals")
    slots = [rig.put(k) for k in range(2)]
    wide = rig.put(len(pool) - 1)
    Ls, Ld, Lg = _layouts(pool, "1024-to-64")
    n = 40
    try:
        a, b = rig.create(Ls, n), rig.create(Ld, 12)
        recs = _records(rng, rig, Lg, Ls, slots, n)
        recs[5] = relay_state(Lg, Ls, random_records(rng, Lg, [rig.reg.story(wide)], [wide]))[0]   # a wide Story
        rig.upload(a, 0, recs)
        rig.upload(b, 0, _records(rng, rig, Lg, Ld, slots, 4))
        for x, nx in ((a, n), (b, 4)):
            rig.tick(x, "touched", nx)
        # run 7: a non-PASS cond code; run 9 was on the wide Story: re-pointed at a narrow one and its codes above 64 steps
        # cleared by deltas, so only its result record (a baseline of later ticks) is still too wide
        d = [(7, 3, A.DELTA_COND, A.COND_SKIP), (9, wide & 0xFFFF, A.DELTA_TOPO_SLOT, wide >> 16)]
        rig.apply(a, np.array(d, dtype=Frontier.DELTA_DTYPE))
        rig.tick(a, "touched", n)
        ph = rig.reg.story(wide).S
        d = [(9, slots[0] & 0xFFFF, A.DELTA_TOPO_SLOT, slots[0] >> 16)] + [(9, i, A.DELTA_PHASE, 0) for i in range(60, ph)]
        rig.apply(a, np.array(d, dtype=Frontier.DELTA_DTYPE))
        cases = [(a, b, n, 4, [5]),           # the wide Story's slot
                 (a, b, n, 4, [1, 7]),        # a cond code the destination has no plane for
                 (a, a, n, n, [1]),           # a batch to itself
                 (a, b, n + 1, 4, [1]),       # src_n_runs above the capacity
                 (a, b, n, 4, list(range(9))),  # more runs than the destination holds
                 (a, b, n, 4, [n]),           # not a run
                 (a, b, n, 4, [2, 2])]        # twice
        for src, dst, sn, dn, runs in cases:
            assert rig.transfer(src, dst, sn, dn, np.array(runs, np.uint32)) is None, runs
        for x, nx in ((a, n), (b, 4)):   # nothing changed: the ticks and records are the model's, which did not change
            rig.tick(x, "changed", nx)
        with pytest.raises(A.FrontierError) as e:
            fr.resident_transfer(rig.handles[a], 99, n, 4, np.array([1], np.uint32))
        assert e.value.unfit == A.EXTENT_NO_RUN
        assert rig.transfer(a, b, n, 4, np.zeros(0, np.uint32))["src_n_runs"] == n   # a no-op
        # run 9's result record: refused exactly when the model's extent of it is wider than the destination (the rig compares)
        wide_result = run_extent(a, 9, n, Ld)["steps_max"] > Ld.steps_max
        assert (rig.transfer(a, b, n, 4, np.array([9], np.uint32)) is None) == wide_result
        if not wide_result:
            return
        rig.transfer(a, b, n, 4, np.array([0, 1, 2], np.uint32))
        rig.tick(b, "touched", 7)
    finally:
        rig.destroy()


def test_host_mirror_moves_pending_deltas(fr):
    """bfh_batch_transfer in resident mode: pending deltas of moved runs go to the destination under their new index (the device
    and the mirror stay identical: a resident pair evaluates as a non-resident twin pair), and a pending delta outside the
    destination layout blocks the call with both mirrors unchanged"""
    rng = np.random.default_rng(7950)
    steps = [M.random_story(rng, "h%d-" % j, 30, 2) for j in range(2)]
    ps, hs = [M.story_from_steps(s) for s in steps], [_host_story(s) for s in steps]
    c = max(p.child_nibbles() for p in ps)
    slots = [hs[j].upload(fr) for j in range(2)]
    both = make_layout(32, c, COND | CHILD)
    pairs = []
    for resident in (True, False):
        src = H.HostBatch(fr, 128, c, COND | DEC | CHILD | OUT, 48)
        dst = H.HostBatch(fr, 64, c, COND | CHILD | A.F_OUT_FAIL, 48)
        pairs.append((src, dst))
        for x, n in ((src, 30), (dst, 6)):
            for r in range(n):
                x.add_run(hs[r % 2], slots[r % 2])
                _fill(x, r, ps[r % 2], M.random_state(np.random.default_rng(r + 100 * n), ps[r % 2]), both)
            if resident:
                x.set_resident(True)
            x.eval()
    try:
        runs = np.array([3, 17, 28, 0], np.uint32)
        for src, dst in pairs:   # pending deltas (logged in resident mode) on moved and on staying runs
            for r in (3, 17, 5, 29):
                src.set_phase_code(r, 2, A.PHASE_RUNNING)
                src.set_cond(r, 1, A.COND_HOLD)
            dst.set_phase_code(2, 1, A.PHASE_SUCCEEDED)
        rs, rd = pairs[0]
        assert rs.traffic()[2] == 8 and rd.traffic()[2] == 1
        rs.set_decision(28, 1, A.DEC_PENDING)   # the destination has no decision planes: the call is refused
        before = [(x.size(), x.state().copy(), x.result().copy()) for x in (rs, rd)]
        with pytest.raises(A.FrontierError) as e:
            rs.transfer(rd, runs)
        assert e.value.status == A.BF_EINVAL
        for x, (n, st, res) in zip((rs, rd), before):
            assert x.size() == n and np.array_equal(x.state(), st) and np.array_equal(x.result(), res)
        rs.eval()   # sends the deltas
        pairs[1][0].set_decision(28, 1, A.DEC_PENDING)
        pairs[1][0].eval()
        for src, dst in pairs:
            for r in (3, 17, 5, 29):
                src.set_phase_code(r, 3, A.PHASE_SUCCEEDED)
        assert rs.traffic()[2] == 4
        moves = [src.transfer(dst, runs) for src, dst in pairs]
        assert all(np.array_equal(moves[0][i], moves[1][i]) for i in range(2))
        assert rs.traffic()[2] == 2 and rd.traffic()[2] == 1 + 2   # those of runs 3 and 17 moved, re-keyed to 6 and 7
        for src, dst in pairs:
            src.eval()
            dst.eval(A.EVAL_FIXPOINT)
        for i in range(2):
            assert np.array_equal(pairs[0][i].state(), pairs[1][i].state())
            assert np.array_equal(pairs[0][i].result(), pairs[1][i].result())
    finally:
        for p in pairs:
            for x in p:
                x.close()
