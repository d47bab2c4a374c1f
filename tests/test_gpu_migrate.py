"""bf_resident_migrate: the live runs of an edited Story move to its new generation on the device, each step keeping its state by
name.  Every case runs a resident batch whose runs of several Stories are interleaved, migrates the runs of some of them (one of
them twice), and checks the records byte for byte against records packed from scratch with the new topologies and the by-name
state, then the ticks that follow: touched, changed-only, compact, and bf_schedule."""
import ctypes as C

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200 import host as H
from bobrapet_b200.records import make_layout
from oracle import packed as PK
from tests import migration as M
from tests import packing as P

pytestmark = pytest.mark.gpu

NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT
# shape: (steps lo, hi, parallel steps per story, runs, layout fields)
SHAPES = {"cfg3": (200, 257, 0, 3000, 0),                       # phase only
          "cfg4": (200, 257, 6, 3000, ALL),                     # cond + decision, registered bits without a child area
          "cfg5": (513, 700, 20, 1200, ALL | A.F_CHILD)}        # S > 512, child nibbles and registered bits


@pytest.fixture
def fr():
    f = Frontier(0)
    yield f
    f.close()


def _ranges(runs):
    """sorted run indices -> contiguous [lo, hi) ranges"""
    out = []
    for r in runs:
        if out and out[-1][1] == r:
            out[-1][1] = r + 1
        else:
            out.append([r, r + 1])
    return out


def _sched(n):
    from oracle import limiters as LM
    sched = np.zeros(n, dtype=LM.SCHED_RUN_DTYPE)
    sched["story_key"], sched["queue_key"] = np.arange(n) % 7, np.arange(n) % 3
    sched["priority"], sched["queued_elapsed_s"], sched["run_phase"] = np.arange(n) % 5, LM.NONE_U32, 2
    return (sched, np.array([0, 1, 50, 400, 0, 3, 2000], np.int32), np.array([0, 300, 5000], np.int32), np.array([60, 0, 30], np.int32))


def _generations(rng, shape):
    """six Stories, edits of three of them, and an edit of an edit -> (step lists, migrations as (old, new) story indices)"""
    lo, hi, n_par, _, fields = SHAPES[shape]
    par = n_par > 0
    gens = [M.random_story(rng, "t%d-" % k, int(rng.integers(lo, hi)), n_par) for k in range(6)]
    edited = [0, 2, 3]
    gens += [M.edit_story(rng, gens[k], "t%d-e" % k, parallel=par) for k in edited]
    gens.append(M.edit_story(rng, gens[6], "t0-f", parallel=par))
    return gens, [(0, 6), (2, 7), (3, 8), (6, 9)]


def _layout(packed, fields):
    child = max(p.child_nibbles() for p in packed) if fields & A.F_CHILD else 0
    return make_layout(max(p.S for p in packed), child, fields)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_migrate_edits(fr, shape):
    rng = np.random.default_rng({"cfg3": 11, "cfg4": 12, "cfg5": 13}[shape])
    gens, migrations = _generations(rng, shape)
    packed = [M.story_from_steps(s) for s in gens]
    ts = P.topology_set(packed)
    slots = fr.put_topologies(ts)
    pt = PK.PackedTopologies(ts, slots)
    L = _layout(packed, SHAPES[shape][4])
    n = SHAPES[shape][3]
    cap = n + 64                                      # runs at or above n_runs are never migrated
    story = rng.integers(0, 6, cap)
    states = [M.random_state(rng, packed[story[r]]) for r in range(cap)]
    rflags = rng.choice([0, A.RF_FAIL_FAST, A.RF_FAIL_FAST | A.RF_REALTIME], size=cap).astype(np.uint8)
    rec0 = M.pack_by_name(L, packed, story, slots, states, rflags)
    hT, hC = fr.resident_create(L, cap), fr.resident_create(L, cap)
    try:
        fr.resident_upload(hT, 0, rec0)
        fr.resident_upload(hC, 0, rec0)
        assert fr.resident_tick_touched(hT, n, NONE, n, BIG)["full"] == 1
        fr.resident_tick_compact(hC, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        moved = set()
        for old, new in migrations:
            smap, added = M.migration_map(packed[old], packed[new])
            assert added == [x for x in packed[new].names if x not in packed[old].index]
            before = fr.resident_download(hT, 0, cap, L.state_stride)
            got = fr.resident_migrate(hT, slots[old], slots[new], smap, n)
            on = np.nonzero(story[:n] == old)[0]
            assert got == len(on) > 0
            story[on] = new
            for r in on:
                states[r] = M.forget(states[r], packed[new])
            want = M.pack_by_name(L, packed, story, slots, states, rflags)
            after = fr.resident_download(hT, 0, cap, L.state_stride)
            other = np.ones(cap, bool)
            other[on] = False
            assert np.array_equal(after[other], before[other]), "a run of another slot changed"
            bad = np.nonzero((after != want).any(axis=1))[0]
            assert bad.size == 0, (old, new, bad[:10])
            for lo, hi in _ranges(on.tolist()):
                fr.resident_upload(hC, int(lo), np.ascontiguousarray(want[lo:hi]))
            moved |= set(on.tolist())
        # the next touched tick is not a full one and lists every migrated run, exactly as the changed-only tick of the twin that
        # received the re-packed records by upload lists them (the uploads make it list every run: compare the migrated ones)
        out = fr.resident_tick_touched(hT, n, NONE, n, BIG)
        sched, story_limit, queue_limit, queue_aging = _sched(n)
        got_sched = fr.schedule(L, n, sched, story_limit, queue_limit, queue_aging, global_limit=20000)
        mig = sorted(moved)
        assert out["full"] == 0 and out["runs"].tolist() == mig and out["n_evaluated"] == len(mig)
        chead, cev, _, _, _ = fr.resident_tick_compact(hC, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        cst = np.concatenate(([0], np.cumsum(chead >> A.HEAD_COUNT_SHIFT))).astype(np.int64)
        assert np.array_equal(out["head"], chead[mig])
        assert np.array_equal(out["events"], np.concatenate([cev[cst[r]:cst[r + 1]] for r in mig]))
        state = fr.resident_download(hT, 0, n, L.state_stride)
        assert np.array_equal(state, fr.resident_download(hC, 0, n, L.state_stride))
        res, _ = PK.evaluate(pt, L, state, threads=8)
        whead, wev, _ = PK.compact_events(L, res)
        assert np.array_equal(out["head"], whead[mig])
        # bf_schedule after the touched tick saw the complete records: the same as after a full pass of the twin
        fr.resident_eval(hC, L, n)
        want_sched = fr.schedule(L, n, sched, story_limit, queue_limit, queue_aging, global_limit=20000)
        for k in got_sched:
            assert np.array_equal(np.asarray(got_sched[k]), np.asarray(want_sched[k])), k
        # a compact tick of the migrated batch equals the packed oracle
        head, ev, n_ev, _, _ = fr.resident_tick_compact(hT, n, NONE, BIG)
        assert np.array_equal(head, whead) and n_ev == len(wev) and np.array_equal(ev, wev)
        # nothing touched since: an empty touched tick; then dropping an old slot makes the next one full, as any drop does
        out = fr.resident_tick_touched(hT, n, NONE, n, BIG)
        assert out["full"] == 0 and out["n_evaluated"] == 0
        fr.drop_topology(int(slots[2]))
        assert fr.resident_tick_touched(hT, n, NONE, n, BIG)["full"] == 1
    finally:
        fr.resident_destroy(hT)
        fr.resident_destroy(hC)


def test_changed_only_tick_after_migration(fr):
    """a changed-only compact tick lists a migrated run only when its result record changed"""
    rng = np.random.default_rng(21)
    gens, migrations = _generations(rng, "cfg4")
    packed = [M.story_from_steps(s) for s in gens]
    ts = P.topology_set(packed)
    slots = fr.put_topologies(ts)
    pt = PK.PackedTopologies(ts, slots)
    L = _layout(packed, ALL)
    n = 2000
    story = rng.integers(0, 6, n)
    states = [M.random_state(rng, packed[story[r]]) for r in range(n)]
    rec0 = M.pack_by_name(L, packed, story, slots, states, np.ones(n, np.uint8))
    h = fr.resident_create(L, n)
    try:
        fr.resident_upload(h, 0, rec0)
        fr.resident_tick_compact(h, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        prev, _ = PK.evaluate(pt, L, rec0, threads=8)
        old, new = migrations[0]
        smap, _ = M.migration_map(packed[old], packed[new])
        assert fr.resident_migrate(h, slots[old], slots[new], smap, n) == int((story == old).sum())
        head, ev, n_ev, _, n_listed = fr.resident_tick_compact(h, n, NONE, BIG, flags=A.EVAL_CHANGED_ONLY)
        res, _ = PK.evaluate(pt, L, fr.resident_download(h, 0, n, L.state_stride), threads=8)
        whead, wev, wl = PK.compact_events(L, res, prev)
        assert n_listed == wl and np.array_equal(head, whead) and np.array_equal(ev, wev)
        assert 0 < wl <= int((story == old).sum())
    finally:
        fr.resident_destroy(h)


def _steps(spec):
    """[(name, group, type, branches)] -> step dicts without needs"""
    return [dict(name=nm, group=g, type=t, needs=[], branches=b) for nm, g, t, b in spec]


def test_migrate_rejects_bad_arguments(fr):
    E, PA = A.STEP_ENGRAM, A.STEP_PARALLEL
    old = M.story_from_steps(_steps([("a", 0, E, 0), ("p", 0, PA, 3), ("b", 0, E, 0), ("c", 1, E, 0)]))
    new = M.story_from_steps(_steps([("c", 0, E, 0), ("b", 0, E, 0), ("p", 0, PA, 3), ("x", 2, E, 0)]))
    wider = M.story_from_steps(_steps([("a", 0, E, 0), ("p", 0, PA, 5)]))                        # p changes its branch count
    big = M.story_from_steps(_steps([("s%d" % k, 0, E, 0) for k in range(70)]))                   # more steps than the layout
    kids = M.story_from_steps(_steps([("a", 0, E, 0), ("p", 0, PA, 3), ("q", 0, PA, 9)]))         # more child nibbles
    spare = M.story_from_steps(_steps([("a", 0, E, 0)]))
    packed = [old, new, wider, big, kids, spare]
    slots = fr.put_topologies(P.topology_set(packed))
    fr.drop_topology(int(slots[5]))
    L = make_layout(64, old.child_nibbles(), ALL | A.F_CHILD)
    n = 200
    rng = np.random.default_rng(3)
    story = np.where(np.arange(n) % 3 == 0, 1, 0)
    states = [M.random_state(rng, packed[s]) for s in story]
    rec = M.pack_by_name(L, packed, story, slots, states, np.ones(n, np.uint8))
    h = fr.resident_create(L, n)
    try:
        fr.resident_upload(h, 0, rec)
        smap, _ = M.migration_map(old, new)
        cases = [
            (A.BF_EINVAL, slots[0], slots[0], smap, n),                                  # a slot to itself
            (A.BF_ETOPO, slots[0], slots[5], smap, n),                                   # a dropped slot
            (A.BF_ETOPO, 9999, slots[1], smap, n),                                       # an unknown slot
            (A.BF_EINVAL, slots[0], slots[1], smap[:3], n),                              # not one entry per old step
            (A.BF_EINVAL, slots[0], slots[1], np.array([0, 0, 1, 2], np.uint16), n),     # not injective
            (A.BF_EINVAL, slots[0], slots[1], np.array([0, 1, 2, 4], np.uint16), n),     # a target past the new S
            (A.BF_EINVAL, slots[0], slots[2], M.migration_map(old, wider)[0], n),        # a kept parallel step changes its branches
            (A.BF_ETOPO, slots[0], slots[3], M.migration_map(old, big)[0], n),           # S beyond steps_max
            (A.BF_ETOPO, slots[0], slots[4], M.migration_map(old, kids)[0], n),          # child nibbles beyond the layout
            (A.BF_EINVAL, slots[0], slots[1], smap, n + 1),                              # n_runs beyond the batch
        ]
        for status, o, nw, m, nr in cases:
            with pytest.raises(A.FrontierError) as e:
                fr.resident_migrate(h, o, nw, m, nr)
            assert e.value.status == status, (e.value, o, nw, m)
            assert np.array_equal(fr.resident_download(h, 0, n, L.state_stride), rec)
        lib = A.load()
        m = A.Migration(struct_size=C.sizeof(A.Migration) - 4, old_slot=int(slots[0]), new_slot=int(slots[1]), n_runs=n,
                        step_map=smap.ctypes.data, n_old_steps=smap.shape[0])
        assert lib.bf_resident_migrate(fr._ctx, h, C.byref(m)) == A.BF_EINVAL
        assert lib.bf_resident_migrate(fr._ctx, h, None) == A.BF_EINVAL
        assert np.array_equal(fr.resident_download(h, 0, n, L.state_stride), rec)
        # the valid call after all of them
        assert fr.resident_migrate(h, slots[0], slots[1], smap, n) == int((story == 0).sum())
        story[story == 0] = 1
        want = M.pack_by_name(L, packed, story, slots, [M.forget(s, new) for s in states], np.ones(n, np.uint8))
        assert np.array_equal(fr.resident_download(h, 0, n, L.state_stride), want)
    finally:
        fr.resident_destroy(h)


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


def test_host_mirror_migrates_with_the_device():
    """bfh_batch_migrate in resident mode: the device and the mirror stay identical, pending deltas follow their steps (or are
    dropped with a removed step), and the records equal a packing by name"""
    fr = Frontier(0)   # a fresh ctx: the batch's resident handle is its first, 0
    try:
        rng = np.random.default_rng(5)
        gens = [M.random_story(rng, "a-", 180, 8), M.random_story(rng, "b-", 120, 4)]
        gens.append(M.edit_story(rng, gens[0], "a-e"))
        packed = [M.story_from_steps(s) for s in gens]
        hs = [_host_story(s) for s in gens]
        slots = [hs[k].upload(fr) for k in range(3)]
        n = 600
        fields = ALL | A.F_CHILD
        b = H.HostBatch(fr, max(p.S for p in packed), max(p.child_nibbles() for p in packed), fields, n)
        b.set_resident(True)
        story = rng.integers(0, 2, n)
        states = [M.random_state(rng, packed[s]) for s in story]

        def put(r, st, names=None):
            ps = packed[story[r]]
            for i, nm in enumerate(ps.names):
                if names is None or nm in names:
                    ph, cd, dc = st["codes"][nm]
                    b.set_phase_code(r, i, ph)
                    b.set_cond(r, i, cd)
                    b.set_decision(r, i, dc)
            for q, stp in enumerate(ps.par_steps):
                nm = ps.names[stp]
                if names is None or nm in names:
                    on, kids = st["par"][nm]
                    b.register_children(r, q, on)
                    for br, code in enumerate(kids):
                        b.set_child_phase(r, q, br, A.PHASE_NAMES[code] if code < 14 else "Pending")

        for r in range(n):
            assert b.add_run(hs[story[r]], slots[story[r]]) == r
            states[r]["codes"] = {k: (v[0] if v[0] < 14 else 1, v[1], v[2]) for k, v in states[r]["codes"].items()}
            states[r]["par"] = {k: (on, [c if c < 14 else 1 for c in kids]) for k, (on, kids) in states[r]["par"].items()}
            put(r, states[r])
        b.eval()
        # pending deltas: new codes for a third of each run's steps, some of which the edit removes
        for r in range(n):
            ps = packed[story[r]]
            pick = set(rng.choice(ps.names, size=ps.S // 3, replace=False).tolist())
            fresh = M.random_state(rng, ps)
            for nm in pick:
                c = fresh["codes"][nm]
                states[r]["codes"][nm] = (c[0] if c[0] < 14 else 1, c[1], c[2])
                if nm in states[r]["par"]:
                    on, kids = fresh["par"][nm]
                    states[r]["par"][nm] = (on, [c if c < 14 else 1 for c in kids])
            put(r, states[r], pick)
        assert b.traffic()[2] > 0
        on = np.nonzero(story == 0)[0]
        assert b.migrate(hs[0], hs[2], slots[0], slots[2]) == len(on)
        story[on] = 2
        for r in on:
            states[r] = M.forget(states[r], packed[2])
        want = M.pack_by_name(b.L, packed, story, slots, states, np.full(n, A.RF_FAIL_FAST, np.uint8))
        assert np.array_equal(b.state(), want)
        b.eval()   # the remapped deltas go up
        assert np.array_equal(fr.resident_download(0, 0, n, b.L.state_stride), b.state())
        b.close()
    finally:
        fr.close()


def _warps_per_block(L):
    """the launch rule of migrate_runs (resident.cu): 8 warps per CTA, fewer when the 16-byte count header and the warps' stages
    (the layout's code planes and child words) pass 48 KiB"""
    planes = 4 + (2 if L.off_cond != A.OFF_NONE else 0) + (2 if L.off_decision != A.OFF_NONE else 0)
    child_words = (L.child_nibbles + 7) // 8 if L.off_child != A.OFF_NONE else 0
    warp_bytes = 4 * (planes * L.words + child_words)
    w = 8
    while w > 1 and 16 + w * warp_bytes > 48 << 10:
        w -= 1
    return w


# layouts whose child area is far larger than the topologies need: at the 48 KiB boundary of eight warps (seven fit), a
# phase-only one there too, and the largest child area a layout can have (one warp per CTA); child_nibbles is not a multiple
# of 8, so the last child word has padding nibbles, which the uploaded records fill and the migration must keep
BIG_CHILD = [(1024, 10237, ALL | A.F_CHILD, 7), (256, 12029, A.F_CHILD, 7), (1024, 65535, ALL | A.F_CHILD, 1), (300, 597, ALL | A.F_CHILD, 8)]


@pytest.mark.parametrize("steps_max,child_nibbles,fields,wpb", BIG_CHILD, ids=[str(c[1]) for c in BIG_CHILD])
def test_migrate_large_and_padded_child_areas(fr, steps_max, child_nibbles, fields, wpb):
    rng = np.random.default_rng(child_nibbles)
    gens = [M.random_story(rng, "t%d-" % k, int(rng.integers(80, 200)), 10) for k in range(3)]
    gens.append(M.edit_story(rng, gens[0], "t0-e"))
    packed = [M.story_from_steps(s) for s in gens]
    assert max(p.child_nibbles() for p in packed) <= child_nibbles
    slots = fr.put_topologies(P.topology_set(packed))
    L = make_layout(steps_max, child_nibbles, fields)
    assert L.child_nibbles == child_nibbles and child_nibbles % 8 and _warps_per_block(L) == wpb
    n = 240
    story = rng.integers(0, 3, n)
    states = [M.random_state(rng, packed[s]) for s in story]
    rflags = np.ones(n, np.uint8)
    pad = rng.integers(1, 16, size=(n, 8 - child_nibbles % 8))
    rec0 = M.pack_by_name(L, packed, story, slots, states, rflags)
    M.set_child_padding(L, rec0, pad)
    h = fr.resident_create(L, n)
    try:
        fr.resident_upload(h, 0, rec0)
        smap, _ = M.migration_map(packed[0], packed[3])
        on = np.nonzero(story == 0)[0]
        assert fr.resident_migrate(h, slots[0], slots[3], smap, n) == len(on)
        story[on] = 3
        for r in on:
            states[r] = M.forget(states[r], packed[3])
        want = M.pack_by_name(L, packed, story, slots, states, rflags)
        M.set_child_padding(L, want, pad)
        got = fr.resident_download(h, 0, n, L.state_stride)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert bad.size == 0, bad[:10]
    finally:
        fr.resident_destroy(h)


def test_host_mirror_resyncs_a_diverged_device():
    """when the device copy was changed behind the mirror (here: one more run moved onto the old slot), bfh_batch_migrate
    reports it, leaves the mirror as it was, and the next bfh_batch_eval brings the device back to the mirror's records"""
    fr = Frontier(0)   # a fresh ctx: the batch's resident handle is its first, 0
    try:
        rng = np.random.default_rng(8)
        gens = [M.random_story(rng, "a-", 60, 3), M.random_story(rng, "b-", 40, 2)]
        gens.append(M.edit_story(rng, gens[0], "a-e"))
        hs = [_host_story(s) for s in gens]
        slots = [hs[k].upload(fr) for k in range(3)]
        n = 20
        b = H.HostBatch(fr, 80, 256, ALL | A.F_CHILD, n)
        b.set_resident(True)
        for r in range(n):
            b.add_run(hs[r % 2], slots[r % 2])
            b.set_phase_code(r, 1, 2)
        b.eval()
        b.set_phase_code(0, 2, 3)   # a pending delta
        d = np.zeros(1, dtype=Frontier.DELTA_DTYPE)
        d["run"], d["index"], d["field"], d["code"] = 1, slots[0] & 0xFFFF, A.DELTA_TOPO_SLOT, slots[0] >> 16
        fr.resident_apply(0, d)     # run 1 (Story b) now holds Story a's slot on the device only
        before = b.state().copy()
        with pytest.raises(A.FrontierError) as e:
            b.migrate(hs[0], hs[2], slots[0], slots[2])
        assert e.value.status == A.BF_EINVAL
        assert np.array_equal(b.state(), before)
        b.eval()
        assert np.array_equal(fr.resident_download(0, 0, n, b.L.state_stride), b.state())
        b.close()
    finally:
        fr.close()
