"""The device lists of bf_resident_status, bf_resident_resync, bf_resident_commit_journal and bf_resident_schedule at every launch
shape their offsets are built from, against the host models tests/runstatus.py, tests/resync.py, tests/commit_journal.py and
tests/sched_resident.py.

Each call counts per run, scans the per-CTA totals (cta_scan, in 1024-CTA chunks with a carry) and lists each run's entries from
the CTAs before it, the warps before it in its CTA and the lanes before it in its warp.  The cases here put 8 down to 1 warps in a
CTA (a dense topology record sizes each warp's shared stage), grids of 1 to 2049 CTAs with an uneven, non-zero count in every CTA,
output caps cut at every boundary those offsets have (with pinned outputs larger than the cap, whose bytes past it must stay as
they were), and topologies of every width edge, dropped slots and topologies past the layout's steps_max but within its words.
Beside the models, the offsets are checked directly: first_event is the exclusive prefix sum of n_events, items come in ascending
run order, and the drifted / written runs are the distinct runs of the full item list."""
import ctypes

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.frontier import TopologySet
from bobrapet_b200.records import PAR_DTYPE, make_layout, pack_state
from oracle.packed import child_first_of
from tests import commit_journal as J
from tests import resync as RS
from tests import runstatus as ST
from tests import schedref as SR
from tests.test_gpu_commit_timers import put_all, random_timings
from tests.test_gpu_resync import _subset
from tests.test_gpu_sched_resident import Resident, _inputs, _schedule

pytestmark = pytest.mark.gpu

NONE_D = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
STAGE_SMEM = 227 * 1024 - 32   # a status / resync CTA's dynamic shared memory: the opt-in maximum beside its 32 static bytes
CANARY = 0xA5
# step types without stops (a stop step hands the run to the host, and a commit then needs entries) and without parallel steps,
# which are placed apart
TYPES_P = np.array([0.45, 0.1, 0.0, 0.1, 0.0, 0.1, 0.05, 0.2])


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


# ---- topologies, records and launch shapes ----------------------------------------------------------------------------------------

def topologies(rng, specs):
    """one topology per (S, E, parallel steps, allowFailure share) spec: exactly E needs, each on an earlier step (the needs of a
    step spread as evenly as its index allows), random types, flags and groups, parallel descs of random branch counts"""
    S_l, E_l, P_l, rp_l, ci_l, fl_l, par_l, allow = [], [], [], [], [], [], [], []
    for S, E, n_par, af in specs:
        room = np.arange(S)   # step i may need any of steps [0, i)
        assert E <= room.sum()
        q = 0
        while np.minimum(room, q).sum() < E:
            q += 1
        deg = np.minimum(room, q)
        over = int(deg.sum()) - E
        if over:
            deg[rng.choice(np.flatnonzero(deg == q), size=over, replace=False)] -= 1
        rows = [np.sort(rng.choice(i, size=int(deg[i]), replace=False)) if deg[i] else np.zeros(0, np.int64) for i in range(S)]
        rp = np.zeros(S + 1, np.uint32)
        rp[1:] = np.cumsum(deg)
        types = rng.choice(8, size=S, p=TYPES_P).astype(np.uint8)
        par = np.sort(rng.choice(S, size=min(n_par, S), replace=False))
        types[par] = A.STEP_PARALLEL
        fl = types | (rng.random(S) < af).astype(np.uint8) * A.SF_ALLOW_FAILURE
        if af:   # at least one allowFailure step, not a parallel one when there is another
            plain = np.setdiff1d(np.arange(S), par)
            fl[rng.choice(plain if plain.size else np.arange(S))] |= A.SF_ALLOW_FAILURE
        fl |= (rng.random(S) < 0.4).astype(np.uint8) * A.SF_ON_TIMEOUT_SKIP
        fl |= (rng.random(S) < 0.3).astype(np.uint8) * A.SF_HAS_IF
        if rng.random() < 0.6:   # main ++ compensations ++ finally, contiguous
            cuts = np.sort(rng.integers(0, S + 1, size=2))
            g = np.zeros(S, np.uint8)
            g[cuts[0]:cuts[1]], g[cuts[1]:] = 1, 2
            fl |= g << A.SF_GROUP_SHIFT
        pd = np.zeros(par.size, PAR_DTYPE)
        for k, stp in enumerate(par):
            B = int(rng.choice([0, 1, 2, 3, 7, 8, 9, 31, 32, 33, 40]))
            pd[k] = (stp, B, len(allow))
            allow.extend((rng.random(B) < 0.3).tolist())
        S_l.append(S); E_l.append(E); P_l.append(par.size)
        rp_l.append(rp); ci_l.append(np.concatenate(rows).astype(np.uint16) if E else np.zeros(0, np.uint16))
        fl_l.append(fl); par_l.append(pd)
    bits = np.asarray(allow + [False] * ((-len(allow)) % 8), dtype=bool)
    return TopologySet(S_l, E_l, np.concatenate(rp_l), np.concatenate(ci_l), np.concatenate(fl_l), P_l,
                       np.concatenate(par_l) if sum(P_l) else None, np.packbits(bits, bitorder="little") if allow else None)


def _info(ts):
    """per topology: (S, step flags, parallel steps, child nibbles it needs)"""
    out, s0, p0 = [], 0, 0
    for i in range(ts.count):
        S, P = int(ts.S[i]), int(ts.P[i])
        par = ts.parallel[p0:p0 + P] if P else np.zeros(0, PAR_DTYPE)
        br = par["branches"].astype(np.int64)
        need = int(child_first_of(br)[-1] + br[-1]) if P else 0
        out.append((S, ts.step_flags[s0:s0 + S], par["step"].astype(np.int64), need))
        s0, p0 = s0 + S, p0 + P
    return out


def records(rng, L, ts, slots, topo, live_par=(), failed_af=0):
    """state records of runs on topologies ts[topo] (slot slots[topo]) in layout L: progress-shaped phases, random cond and
    decision codes, child nibbles (all of the layout's, the padding ones too), registered bits and run flags; the runs in live_par
    have a Running parallel step (stage H stages the topology record); with failed_af, each run has 1 to failed_af of its
    allowFailure steps Failed (an allowed-failure event each, whatever the run's outcome)"""
    n, width = topo.size, 32 * L.words
    info = _info(ts)
    S_run = ts.S[topo].astype(np.int64)
    idx = np.arange(width)[None, :]
    prog = rng.integers(0, S_run + 1)[:, None]
    done = rng.choice([3, 13, 4, 2, 8, 11, 6, 1], size=(n, width), p=[0.8, 0.04, 0.03, 0.05, 0.03, 0.01, 0.01, 0.03])
    todo = rng.choice([0, 14, 9, 10], size=(n, width), p=[0.93, 0.04, 0.02, 0.01])
    phase = np.where(idx < prog, done, todo).astype(np.uint8)
    cond = rng.choice(4, size=(n, width), p=[0.55, 0.2, 0.15, 0.1]).astype(np.uint8)
    dec = rng.integers(0, 4, size=(n, width)).astype(np.uint8)
    for r in range(n):
        S, fl, par, _ = info[topo[r]]
        if failed_af:   # never a parallel step, which may be the live one below
            af = np.setdiff1d(np.flatnonzero(fl & A.SF_ALLOW_FAILURE), par)
            assert af.size, "a run needs an allowFailure step"
            phase[r, rng.choice(af, size=min(af.size, 1 + r % failed_af), replace=False)] = A.PHASE_FAILED
    for r in live_par:
        par = info[topo[r]][2]
        phase[r, par[rng.integers(0, par.size)]] = A.PHASE_RUNNING
    pad = idx >= S_run[:, None]
    phase[pad] = cond[pad] = dec[pad] = 0
    child = None
    if L.off_child != A.OFF_NONE:
        nb = (L.child_nibbles + 1) // 2 * 2
        child = rng.choice([0, 2, 3, 3, 3, 3, 4, 13, 11, 1], size=(n, nb)).astype(np.uint8)
    reg = rng.integers(0, 2**63, size=n, dtype=np.uint64)
    rflags = ((rng.random(n) < 0.5) * A.RF_FAIL_FAST | (rng.random(n) < 0.25) * A.RF_REALTIME |
              (rng.random(n) < 0.3) * A.RF_TOPOLOGY_TERMINATED).astype(np.uint8)
    st = pack_state(L, np.asarray(slots, np.uint32)[topo], rflags, phase, cond, dec, None, reg)
    if child is not None:   # every nibble of the area, those past child_nibbles in its last byte as well
        st[:, L.off_child:L.off_child + nb // 2] = child[:, 0::2] | child[:, 1::2] << 4
    return st


def warps_per_cta(fr, L, ts, slots):
    """the launch rule of the status and resync calls, from the records the ctx holds: 8 warps per CTA, fewer when a warp's stage
    (the state record, the largest live record of at most L.words words, 256 bytes) times 8 passes the CTA's shared memory
    -> (warps per CTA, bytes per warp)"""
    if L.off_child == A.OFF_NONE:
        return 8, 0
    rec = max([fr.topology_record(int(s))[1] for s, S in zip(slots, ts.S) if (int(S) + 31) // 32 <= L.words] + [0])
    per_warp = L.state_stride + rec + 256
    return min(8, STAGE_SMEM // per_warp), per_warp


def cut_points(counts, wpb, inside=()):
    """the caps to cut a list at, from its entries per listed run: 0, 1, total - 1, total, total + 1, the first entry of CTA 1 and
    of CTA 1024, the middle of the longest run's list, and the points `inside` one run's list"""
    c = np.concatenate(([0], np.cumsum(counts, dtype=np.int64)))
    total = int(c[-1])
    pts = {0, 1, max(total - 1, 0), total, total + 1} | {int(x) for x in inside}
    for k in (1, 1024):
        if k * wpb < len(counts):
            pts.add(int(c[k * wpb]))
    i = int(np.argmax(counts))
    pts.add(int(c[i] + counts[i] // 2))
    return sorted(pts)


def pinned(fr, nbytes):
    """a pinned buffer of nbytes (at least 16) filled with the canary; it stays allocated until the ctx closes, so that nothing a
    failing assertion shows points at freed memory"""
    b = fr.alloc_pinned(max(nbytes, 16))
    b[:] = CANARY
    return b


def untouched(buf, used):
    assert (buf[used:] == CANARY).all(), ("written past the cap", used, np.flatnonzero(buf[used:] != CANARY)[:8] + used)


def same_bytes(got, want, what):
    assert got.tobytes() == want.tobytes(), (what, next((i, got[i], want[i]) for i in range(len(want))
                                                       if got[i].tobytes() != want[i].tobytes()))


# ---- bf_resident_status ---------------------------------------------------------------------------------------------------------

def check_status(fr, h, L, ts, slots, state, n_runs, wpb, runs=None, cuts=True):
    """the status of the listed runs against the model: every record, every event, first_event the exclusive prefix sum of
    n_events; with cuts, events_cap cut at every boundary, pageable and pinned (canary past the cap)"""
    k = n_runs if runs is None else runs.size
    want_recs, want_ev, total = ST.status(L, ts, slots, state, n_runs, runs)
    recs, ev, n_ev = fr.resident_status(h, n_runs, runs, events_cap=total)
    ne = recs["n_events"].astype(np.int64)
    assert np.array_equal(recs["first_event"], np.concatenate(([0], np.cumsum(ne)[:-1]))), "first_event is not the prefix sum"
    assert n_ev == total and ev.size == total
    same_bytes(recs, want_recs, "records")
    assert np.array_equal(ev, want_ev), np.flatnonzero(ev != want_ev)[:8]
    if not cuts:
        return want_recs, total
    p_runs = None
    if runs is not None:
        p_runs = pinned(fr, 4 * k).view(np.uint32)[:k]
        p_runs[:] = runs
    for cap in cut_points(want_recs["n_events"].astype(np.int64), wpb):
        used = min(cap, total)
        recs, ev, n_ev = fr.resident_status(h, n_runs, runs, events_cap=cap)
        assert n_ev == total and np.array_equal(ev, want_ev[:used]), cap
        same_bytes(recs, want_recs, ("records at cap", cap))
        p_recs, p_ev = pinned(fr, 32 * k + 64), pinned(fr, 2 * cap + 64)
        out = A.StatusOut(struct_size=ctypes.sizeof(A.StatusOut), records=p_recs.ctypes.data, events=p_ev.ctypes.data,
                          events_cap=cap)
        assert fr._lib.bf_resident_status(fr._ctx, h, n_runs, None if p_runs is None else p_runs.ctypes.data, k,
                                          ctypes.byref(out)) == A.BF_OK
        assert out.n_events == total, cap
        same_bytes(p_recs[:32 * k].view(Frontier.STATUS_DTYPE), want_recs, ("pinned records at cap", cap))
        untouched(p_recs, 32 * k)
        assert np.array_equal(p_ev[:2 * used].view(np.uint16), want_ev[:used]), cap
        untouched(p_ev, 2 * used)
    return want_recs, total


# ---- bf_resident_resync ---------------------------------------------------------------------------------------------------------

def drifted_records(rng, L, state, live_slots):
    """the device's records with every run drifted: a few, and those on a slot no put returned, on another live slot (one item),
    every other with a run flag flipped (one item) and 0 to 3 more random bits flipped in its phase, cond and decision planes,
    child area or registered bits"""
    out = state.copy()
    spans = [(L.off_phase, 16 * L.words), (8, 8)]
    for off, nb in ((L.off_cond, 8 * L.words), (L.off_decision, 8 * L.words)):
        if off != A.OFF_NONE:
            spans.append((off, nb))
    if L.off_child != A.OFF_NONE:
        spans.append((L.off_child, (L.child_nibbles + 1) // 2))
    for r in range(state.shape[0]):
        slot = int(out[r, :4].view("<u4")[0])
        if slot == 0xFFFF or rng.random() < 0.03:
            out[r, :4] = np.frombuffer(np.uint32(rng.choice([s for s in live_slots if s != slot])).tobytes(), np.uint8)
            continue
        out[r, 4] ^= 1 << (r % 3)
        for _ in range(r % 4):
            off, nb = spans[rng.integers(0, len(spans))]
            b = int(rng.integers(0, 8 * nb))
            out[r, off + b // 8] ^= 1 << (b % 8)
    return out


def _field_cuts(items, pos0):
    """the item positions between the fields of the run with the most kinds of field (its list starts at pos0 + its index)"""
    runs, first = np.unique(items["run"], return_index=True)
    kinds = [np.unique(items["field"][items["run"] == r]).size for r in runs]
    j = int(np.argmax(kinds))
    f = items["field"][first[j]:first[j] + int((items["run"] == runs[j]).sum())]
    return [pos0 + int(first[j]) + int(i) for i in np.flatnonzero(np.diff(f.astype(np.int64))) + 1], kinds[j]


def check_resync(fr, h, L, topos, state, recs, n_runs, wpb, runs=None, cuts=True, repair=True, misaligned=False):
    """a check of the listed runs against the model (items, drifted runs, ascending run order, drifted = the distinct runs of the
    items); with cuts, items_cap and drifted_cap cut at every boundary, between a run's fields too, pageable and pinned; with
    misaligned, pinned items 8 bytes off 16-byte alignment; with repair, the repair: the same lists, the model's records, and the
    next touched tick evaluates exactly the drifted runs"""
    k = n_runs if runs is None else runs.size
    items, drifted, after, _ = RS.resync(L, topos, state, recs, n_runs, runs)
    total, n_dr = items.size, drifted.size
    got = fr.resident_resync(h, n_runs, recs, runs=runs, check=True, drifted_cap=k, items_cap=max(total, 1))
    assert np.all(np.diff(got["items"]["run"].astype(np.int64)) >= 0), "items out of run order"
    assert got["drifted"].tolist() == np.unique(got["items"]["run"]).tolist(), "drifted is not the items' distinct runs"
    assert got["n_items"] == total and got["n_drifted"] == n_dr and got["n_written"] == 0
    same_bytes(got["items"], items, "items")
    assert np.array_equal(got["drifted"], drifted)
    assert fr.resident_download(h, 0, n_runs, L.state_stride).tobytes() == state.tobytes()
    listed = np.arange(n_runs) if runs is None else runs
    pos_of = np.searchsorted(listed, items["run"])
    per_run = np.bincount(pos_of, minlength=k)
    q = A.Resync(struct_size=ctypes.sizeof(A.Resync), n_runs=n_runs, runs=None if runs is None else runs.ctypes.data, n=k,
                 fields=A.RESYNC_ALL_FIELDS, records=recs.ctypes.data, flags=A.RESYNC_CHECK)

    def pinned_call(items_cap, drifted_cap, shift=0):
        p_items, p_dr = pinned(fr, 16 * items_cap + 64 + shift), pinned(fr, 4 * drifted_cap + 64)
        q.items, q.items_cap = p_items.ctypes.data + shift, items_cap
        q.drifted, q.drifted_cap = p_dr.ctypes.data, drifted_cap
        assert fr._lib.bf_resident_resync(fr._ctx, h, ctypes.byref(q)) == A.BF_OK
        assert (q.n_items, q.n_drifted) == (total, n_dr), (items_cap, drifted_cap)
        used_i, used_d = min(items_cap, total), min(drifted_cap, n_dr)
        same_bytes(p_items[shift:shift + 16 * used_i].view(Frontier.DRIFT_DTYPE), items[:used_i], ("pinned items", items_cap))
        untouched(p_items[shift:], 16 * used_i)
        assert (p_items[:shift] == CANARY).all()
        assert np.array_equal(p_dr[:4 * used_d].view(np.uint32), drifted[:used_d]), drifted_cap
        untouched(p_dr, 4 * used_d)

    if cuts:
        inside, n_kinds = _field_cuts(items, 0)
        assert n_kinds >= 3 or k < 64, n_kinds
        for cap in cut_points(per_run, wpb, inside):
            g = fr.resident_resync(h, n_runs, recs, runs=runs, check=True, drifted_cap=k, items_cap=cap)
            assert (g["n_items"], g["n_drifted"]) == (total, n_dr), cap
            same_bytes(g["items"], items[:min(cap, total)], ("items", cap))
            pinned_call(cap, k)
        for cap in cut_points((per_run > 0).astype(np.int64), wpb):
            g = fr.resident_resync(h, n_runs, recs, runs=runs, check=True, drifted_cap=cap, items_cap=max(total, 1))
            assert (g["n_items"], g["n_drifted"]) == (total, n_dr), cap
            assert np.array_equal(g["drifted"], drifted[:min(cap, n_dr)]), cap
            pinned_call(max(total, 1), cap)
    if misaligned:   # the staged path: the items go through the ctx's scratch and are copied after the call
        pinned_call(max(total, 1), k, shift=8)
        pinned_call(max(total // 2, 1), k, shift=8)
    if not repair:
        return items
    got = fr.resident_resync(h, n_runs, recs, runs=runs, drifted_cap=k, items_cap=max(total, 1))
    same_bytes(got["items"], items, "repair items")
    assert np.array_equal(got["drifted"], drifted) and got["n_written"] == n_dr
    same_bytes(fr.resident_download(h, 0, n_runs, L.state_stride), after, "records after the repair")
    return items


def touched_after_repair(fr, h, L, n_runs, items, dense0):
    """the touched tick after a repair evaluates exactly the drifted runs and lists those whose result changed and every one
    whose slot drifted: the touch marks were written at the right runs"""
    drifted = np.unique(items["run"])
    t = fr.resident_tick_touched(h, n_runs, NONE_D, n_runs, 64 * n_runs)
    assert t["full"] == 0 and t["n_evaluated"] == drifted.size, (t["full"], t["n_evaluated"], drifted.size)
    dense1, _ = fr.resident_tick(h, L, n_runs, NONE_D)
    changed = {int(r) for r in drifted if dense0[r].tobytes() != dense1[r].tobytes()}
    assert set(t["runs"].tolist()) == changed | set(RS.slot_drifted(items).tolist())


# ---- bf_resident_commit_journal -----------------------------------------------------------------------------------------------

def journal_commit(fr, L, st, n, K, items_cap, runs_cap, pin, shift=0):
    """a fresh batch of the records st (K timer slots per run) takes a tick and a journaled commit with no entries (its topologies
    have no stop steps), arming at now = 100 with K -> (n_items, n_runs_listed, items, runs, before, after, timers before / after)"""
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    if K:
        fr.resident_timers(h, K)
    fr.resident_tick(h, L, n, NONE_D)
    before = fr.resident_download(h, 0, n, L.state_stride)
    t0 = fr.resident_timers_download(h, 0, n, K).view("<u8").copy() if K else None
    if pin:
        ib, rb = pinned(fr, 16 * items_cap + 64 + shift), pinned(fr, 4 * runs_cap + 64)
    else:
        ib, rb = np.full(16 * items_cap + 64 + shift, CANARY, np.uint8), np.full(4 * runs_cap + 64, CANARY, np.uint8)
    out = A.CommitOut(struct_size=ctypes.sizeof(A.CommitOut))
    arm = A.CommitArm(struct_size=ctypes.sizeof(A.CommitArm), now=100) if K else None
    j = A.CommitJournal(struct_size=ctypes.sizeof(A.CommitJournal), items=ib.ctypes.data + shift, items_cap=items_cap,
                        runs=rb.ctypes.data, runs_cap=runs_cap)
    rc = fr._lib.bf_resident_commit_journal(fr._ctx, h, n, None, 0, ctypes.byref(out), None if arm is None else ctypes.byref(arm),
                                            ctypes.byref(j))
    assert rc == A.BF_OK, fr._lib.bf_last_error(fr._ctx).decode()
    after = fr.resident_download(h, 0, n, L.state_stride)
    t1 = fr.resident_timers_download(h, 0, n, K).view("<u8").copy() if K else None
    fr.resident_destroy(h)
    assert (ib[:shift] == CANARY).all()
    return int(j.n_items), int(j.n_runs_listed), ib[shift:], rb, before, after, t0, t1


def check_journal(fr, L, st, n, K=0, cuts=True, misaligned=False):
    """the journal against the byte difference of the records and timer slots, items in ascending run order and the runs listed
    the distinct runs of the items; with cuts, items_cap and runs_cap cut at every boundary, between a run's PHASE, REGISTERED
    and TIMER items too, pageable and pinned (canary past the cap); with misaligned, pinned items 8 bytes off alignment"""
    bound = n * (3 * 32 * L.words + 64)
    ni, nr, ib, rb, before, after, t0, t1 = journal_commit(fr, L, st, n, K, bound, n, True)
    want_items, want_runs = J.journal(L, before, after, n, t0, t1)
    total, n_w = len(want_items), len(want_runs)
    assert (ni, nr) == (total, n_w)
    got = J.as_tuples(ib[:16 * total].view(Frontier.COMMIT_WRITE_DTYPE))
    assert got == want_items
    runs = rb[:4 * n_w].view(np.uint32)
    assert runs.tolist() == want_runs
    assert want_runs == sorted({x[0] for x in got if x[2] != J.TIMER}), "runs are not the distinct runs of the record items"
    assert np.all(np.diff([x[0] for x in got]) >= 0), "items out of run order"
    per_run = np.bincount([x[0] for x in want_items], minlength=n)
    written = np.zeros(n, np.int64)
    written[want_runs] = 1
    ctas = np.add.reduceat(per_run, np.arange(0, n, 8))
    full = ctas[:-1] if ctas.size > 1 else ctas   # the last CTA may hold a single run, which may write nothing
    assert (full > 0).all() and (full.size < 2 or np.unique(full).size > 1), "every CTA needs items, in uneven counts"

    def one(items_cap, runs_cap, pin, shift=0):
        ni, nr, ib, rb, b0, a0, _, _ = journal_commit(fr, L, st, n, K, items_cap, runs_cap, pin, shift)
        assert (ni, nr) == (total, n_w), (items_cap, runs_cap)
        assert np.array_equal(b0, before) and np.array_equal(a0, after)
        ui, ur = min(items_cap, total), min(runs_cap, n_w)
        assert J.as_tuples(ib[:16 * ui].view(Frontier.COMMIT_WRITE_DTYPE)) == want_items[:ui], items_cap
        untouched(ib, 16 * ui)
        assert rb[:4 * ur].view(np.uint32).tolist() == want_runs[:ur], runs_cap
        untouched(rb, 4 * ur)

    if cuts:
        kinds = {}
        for x in want_items:
            kinds.setdefault(x[0], set()).add(x[2])
        r = max(kinds, key=lambda r: len(kinds[r]))
        assert n < 64 or kinds[r] == ({J.PHASE, J.REGISTERED, J.TIMER} if K else {J.PHASE, J.REGISTERED}), kinds[r]
        pos = [i for i, x in enumerate(want_items) if x[0] == r]
        inside = [pos[0] + i for i in range(1, len(pos)) if want_items[pos[i]][2] != want_items[pos[i - 1]][2]]
        for cap in cut_points(per_run, 8, inside):
            for pin in (False, True):
                one(cap, n, pin)
        for cap in cut_points(written, 8):
            for pin in (False, True):
                one(max(total, 1), min(cap, n), pin)
    if misaligned:
        one(max(total, 1), n, True, shift=8)
        one(max(total // 2, 1), n, True, shift=8)


# ---- the cases ------------------------------------------------------------------------------------------------------------------

def small_specs(rng, k, s_lo, s_hi, par=True):
    """k small topologies of S in [s_lo, s_hi], about S needs, a few parallel steps each (some none)"""
    out = []
    for _ in range(k):
        S = int(rng.integers(s_lo, s_hi + 1))
        out.append((S, min(S, S * (S - 1) // 2), int(rng.integers(0, 4)) if par else 0, 0.3))
    return out


def child_need(ts):
    return max(x[3] for x in _info(ts))


def spread(rng, n, k, wpb):
    """k distinct runs of [0, n), the first and last run of CTA 0, 1 and 1024 among them when there are such runs"""
    edge = [r for r in (0, wpb - 1, wpb, 2 * wpb - 1, 1024 * wpb, 1024 * wpb + 1) if r < n]
    rest = rng.choice(np.setdiff1d(np.arange(n), edge), size=max(0, min(k, n) - len(edge)), replace=False)
    return np.sort(np.concatenate([edge, rest]).astype(np.int64))


# (warps per CTA, needs of the 1024-step topology, layout child nibbles): the dense topology's record sizes each warp's shared
# stage (state record + largest record + 256 bytes); the child area of 65 535 nibbles (not a multiple of 8) is the largest a
# layout can have
WARPS = [(8, 4000, 2603), (7, 12000, 2603), (4, 8000, 65535), (2, 45000, 2603), (1, 65535, 2603)]


@pytest.mark.parametrize("wpb,E,child", WARPS, ids=["wpb%d" % w[0] for w in WARPS])
def test_warps_per_cta(fr, wpb, E, child):
    """status and resync at 8 down to 1 warps per CTA over 1026 CTAs: a few tens of runs on the dense topology with a live
    parallel step (stage H copies its record into the warp's stage), the others on small topologies in the 32-word layout"""
    rng = np.random.default_rng(wpb * 7919 + E)
    ts = topologies(rng, [(1024, E, 64, 0.2)] + small_specs(rng, 12, 8, 80))
    slots = fr.put_topologies(ts)
    L = make_layout(1024, child, ALL | A.F_CHILD)
    assert L.child_nibbles == child and child_need(ts) <= child
    got, per_warp = warps_per_cta(fr, L, ts, slots)
    assert got == wpb and wpb * per_warp > 48 << 10, (got, per_warp)
    n = 1025 * wpb + 3
    topo = rng.integers(1, ts.count, size=n)
    dense = spread(rng, n, 24, wpb)
    topo[dense] = 0
    st = records(rng, L, ts, slots, topo, live_par=dense, failed_af=4)
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    dense0, _ = fr.resident_tick(h, L, n, NONE_D)
    check_status(fr, h, L, ts, slots, st, n, wpb)
    runs = np.sort(rng.choice(n, size=n // 3, replace=False)).astype(np.uint32)
    check_status(fr, h, L, ts, slots, st, n, wpb, runs=runs, cuts=False)
    recs = drifted_records(rng, L, st, [int(s) for s in slots])
    items = check_resync(fr, h, L, RS.Topos(ts, slots), st, recs, n, wpb, misaligned=wpb in (1, 8))
    touched_after_repair(fr, h, L, n, items, dense0)


# (warps per CTA, CTAs): at 8 warps small one-word topologies; at 1 warp the 65 535-need topology in the ctx and a few runs on it
GRIDS = [(8, 1), (8, 1023), (8, 1024), (8, 1025), (8, 2048), (8, 2049), (1, 1025), (1, 2049)]


@pytest.mark.parametrize("wpb,ctas", GRIDS, ids=["wpb%d-%d" % g for g in GRIDS])
def test_grids_across_scan_chunks(fr, wpb, ctas):
    """status, resync (check and repair) and, at 8 runs per CTA, the journal over grids of 1 to 2049 CTAs, every CTA with a
    non-zero, uneven count; caps cut at every boundary; a sparse runs list spanning 1025 CTAs"""
    rng = np.random.default_rng(ctas * 31 + wpb)
    if wpb == 8:
        ts = topologies(rng, small_specs(rng, 12, 6, 32))
        L = make_layout(32, child_need(ts) | 1, ALL | A.F_CHILD)
        n = 8 * (ctas - 1) + 1 + ctas % 8   # the last CTA holds 1 to 8 runs
    else:
        ts = topologies(rng, [(1024, 65535, 64, 0.2)] + small_specs(rng, 12, 8, 80))
        L = make_layout(1024, 2603, ALL | A.F_CHILD)
        n = ctas
    assert L.child_nibbles >= child_need(ts)
    slots = fr.put_topologies(ts)
    got, per_warp = warps_per_cta(fr, L, ts, slots)
    assert got == wpb and (wpb * per_warp <= 48 << 10) == (wpb == 8), (got, per_warp)
    assert (n - 1) // wpb + 1 == ctas
    topo = rng.integers(1 if wpb == 1 else 0, ts.count, size=n)
    par = np.flatnonzero(ts.P[topo] > 0)
    live = rng.choice(par, size=min(par.size, 40), replace=False)
    if wpb == 1:
        live = spread(rng, n, 20, wpb)
        topo[live] = 0
    st = records(rng, L, ts, slots, topo, live_par=live, failed_af=5)
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    dense0, _ = fr.resident_tick(h, L, n, NONE_D)
    recs, _ = check_status(fr, h, L, ts, slots, st, n, wpb)
    per_cta = np.add.reduceat(recs["n_events"].astype(np.int64), np.arange(0, n, wpb))
    assert (per_cta > 0).all() and np.unique(per_cta).size > min(ctas - 1, 1), "every CTA needs events, in uneven counts"
    if ctas == 2049:   # a sparse list: every other run, 1025 CTAs at 8 warps
        runs = np.arange(0, n, 2, dtype=np.uint32)
        check_status(fr, h, L, ts, slots, st, n, wpb, runs=runs)
        check_resync(fr, h, L, RS.Topos(ts, slots), st, drifted_records(rng, L, st, [int(s) for s in slots])[runs], n, wpb,
                     runs=runs, repair=False)
    drift = drifted_records(rng, L, st, [int(s) for s in slots])
    items = check_resync(fr, h, L, RS.Topos(ts, slots), st, drift, n, wpb, cuts=ctas in (1, 1025, 2049))
    touched_after_repair(fr, h, L, n, items, dense0)
    if wpb == 8:
        timings = {}
        for slot, t in random_timings(rng, ts, slots).items():   # at most 8 per slot, as a run has 4 timer slots here
            timings[slot] = dict(sorted(t.items())[:4])
        put_all(fr, timings)
        check_journal(fr, L, st, n, K=4, cuts=ctas in (1, 1024, 1025, 2049), misaligned=ctas == 1025)


@pytest.mark.parametrize("steps_max", [1024, 100])
def test_width_edges(fr, steps_max):
    """topologies of 1 to 1024 steps in a layout of 32 words or of 4 (steps_max 100: those of 101 to 128 steps are live past
    steps_max, the wider ones dead), runs on a dropped slot and on a slot no put returned"""
    rng = np.random.default_rng(steps_max)
    widths = [1, 31, 32, 33, 63, 64, 65, 101, 128, 993, 1023, 1024]
    ts = topologies(rng, [(S, min(2 * S, S * (S - 1) // 2), 1 if S >= 8 else 0, 0.3) for S in widths])
    slots = fr.put_topologies(ts)
    L = make_layout(steps_max, child_need(ts) | 1, ALL | A.F_CHILD)
    n = 3000
    topo = rng.integers(0, ts.count, size=n)
    par = np.flatnonzero(ts.P[topo] > 0)
    wide = ts.S[topo] > 32 * L.words
    par = par[~wide[par]]
    st = records(rng, L, ts, slots, np.where(wide, 0, topo), live_par=rng.choice(par, size=40, replace=False), failed_af=3)
    st[:, :4] = np.asarray(slots, np.uint32)[topo].view(np.uint8).reshape(n, 4)   # the wide runs' codes are those of a 1-step run
    st[rng.choice(n, size=30, replace=False), :4] = np.frombuffer(np.uint32(0xFFFF).tobytes(), np.uint8)
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    gone = widths.index(33)
    fr.drop_topology(int(slots[gone]))
    keep = np.arange(ts.count) != gone
    live_ts, live_slots = _subset(ts, keep), slots[keep]
    wpb, _ = warps_per_cta(fr, L, live_ts, live_slots)
    dense0, _ = fr.resident_tick(h, L, n, NONE_D)
    recs, _ = check_status(fr, h, L, live_ts, live_slots, st, n, wpb)
    dead = recs["outcome"] == A.OUTCOME_DEAD
    assert np.array_equal(dead, ~np.isin(st[:, :4].copy().view("<u4")[:, 0], live_slots) | wide)
    drift = drifted_records(rng, L, st, [int(s) for s in live_slots])
    items = check_resync(fr, h, L, RS.Topos(live_ts, live_slots), st, drift, n, wpb)
    touched_after_repair(fr, h, L, n, items, dense0)


def test_status_lists_every_event_past_steps_max(fr):
    """a layout of steps_max 33 (two words) holds runs of a 64-step topology whose steps all allow failure and all failed: each
    has 64 allowed-failure events, and events_cap set to the true total gets every one of them, through the C ABI with pinned
    buffers and through the wrapper's default cap"""
    rng = np.random.default_rng(64)
    ts = topologies(rng, [(64, 64, 0, 1.0), (33, 33, 0, 0.5), (20, 20, 0, 0.5)])
    slots = fr.put_topologies(ts)
    L = make_layout(33, 0, A.F_COND | A.F_DECISION | A.F_ALL_OUT)
    assert L.words == 2 and (ts.step_flags[:64] & A.SF_ALLOW_FAILURE).all()
    n = 300
    topo = np.where(rng.random(n) < 0.8, 0, rng.integers(1, 3, size=n))
    st = records(rng, L, ts, slots, topo, failed_af=2)
    wide = np.flatnonzero(topo == 0)
    codes = np.full((wide.size, 64), A.PHASE_FAILED, np.uint8)
    st[wide, L.off_phase:L.off_phase + 16 * L.words] = pack_state(L, np.zeros(wide.size, np.uint32), np.zeros(wide.size, np.uint8),
                                                                   codes)[:, L.off_phase:L.off_phase + 16 * L.words]
    h = fr.resident_create(L, n)
    fr.resident_upload(h, 0, st)
    want_recs, want_ev, total = ST.status(L, ts, slots, st, n)
    assert (want_recs["n_events"][wide] == 64).all() and total > n * L.steps_max
    p_recs, p_ev = pinned(fr, 32 * n + 64), pinned(fr, 2 * total + 64)
    out = A.StatusOut(struct_size=ctypes.sizeof(A.StatusOut), records=p_recs.ctypes.data, events=p_ev.ctypes.data, events_cap=total)
    assert fr._lib.bf_resident_status(fr._ctx, h, n, None, n, ctypes.byref(out)) == A.BF_OK
    assert out.n_events == total
    same_bytes(p_recs[:32 * n].view(Frontier.STATUS_DTYPE), want_recs, "records")
    assert np.array_equal(p_ev[:2 * total].view(np.uint16), want_ev), "events past n * steps_max were not written"
    untouched(p_ev, 2 * total)
    recs, ev, n_ev = fr.resident_status(h, n)
    assert n_ev == total and ev.size == total and np.array_equal(ev, want_ev)
    check_status(fr, h, L, ts, slots, st, n, 8)
    items = check_resync(fr, h, L, RS.Topos(ts, slots), st, drifted_records(rng, L, st, [int(s) for s in slots]), n, 8)
    assert items.size


# (CTAs of 256 runs): bf_resident_schedule's listed runs and events are scanned across 1024-CTA chunks
SCHED_GRIDS = [1023, 1024, 1025, 2049]


@pytest.mark.parametrize("ctas", SCHED_GRIDS)
def test_schedule_grids_across_scan_chunks(fr, ctas):
    """bf_resident_schedule over grids of 1023 to 2049 CTAs: a first schedule lists every run; then, before each further
    schedule, the first 1 to 13 runs of every CTA (uneven counts) lose their baseline by an upload of their own record, and only
    they are listed: runs, heads, events and totals against the host model, with the caps at the totals and cut at the first
    listed run of CTA 1024 (of the last CTA on a grid of one chunk)"""
    rng = np.random.default_rng(ctas * 17)
    n = 256 * (ctas - 1) + 1 + ctas % 255
    ts = topologies(rng, small_specs(rng, 12, 6, 32))
    slots = fr.put_topologies(ts)
    L = make_layout(32, 0, A.F_COND | A.F_DECISION | A.F_ALL_OUT)
    st = records(rng, L, ts, slots, rng.integers(0, ts.count, size=n))
    now = 20_000
    tables = SR.random_tables(rng, 40, 5, n, maxprio_base=True)
    b = Resident(fr, L, st, n, SR.from_topology_set(ts, slots))
    try:
        b.put(_inputs(rng, n, 40, 5, now))
        fr.resident_tick(b.h, L, n, NONE_D)
        cur = [b.current()]
        got, _, _ = _schedule(fr, [b], tables, now, caps=[dict(runs_cap=n, events_cap=32 * n)], cur=cur)
        assert got["parts"][0]["full"] == 1
        first = np.arange(ctas) * 256
        lose = np.minimum(1 + np.arange(ctas) * 7 % 13, n - first)
        cut_cta = min(1024, ctas - 1)
        for cut in (False, True):
            for r0, k in zip(first, lose):
                fr.resident_upload(b.h, int(r0), st[r0:r0 + k])
                b.model.upload(int(r0), int(k))
            fr.resident_tick(b.h, L, n, NONE_D)
            caps = dict(runs_cap=n, events_cap=32 * n)
            if cut:   # the same runs as the schedule before are listed, so its list gives the offsets of CTA cut_cta
                j = int(lose[:cut_cta].sum())
                caps = dict(runs_cap=j, events_cap=int(want["heads"][:j, :3].sum()))
            got, w, _ = _schedule(fr, [b], tables, now, caps=[caps], cur=cur)
            want = w["parts"][0]
            assert np.array_equal(np.bincount(want["listed"] // 256, minlength=ctas), lose), "the listed runs per CTA"
            assert got["parts"][0]["runs"].size == min(caps["runs_cap"], want["listed"].size)
            assert got["parts"][0]["events"].size == min(caps["events_cap"], want["n_events"])
    finally:
        b.close()
