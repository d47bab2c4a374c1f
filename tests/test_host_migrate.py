"""Story edits in the C++ host mirror without a device: bfh_story_migration_map against the Python helper, and bfh_batch_migrate
re-packing the mirror's records exactly as a packing of the runs' by-name state against the new generation does."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import host as H
from tests import migration as M


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


def _codes(st):
    """child phases through bfh_run_set_child_phase take a phase name: code 14 (queued Pending) is not one"""
    return {"codes": st["codes"], "par": {k: (on, [c if c < 14 else 1 for c in kids]) for k, (on, kids) in st["par"].items()}}


def _fill(b, r, ps, st):
    for i, nm in enumerate(ps.names):
        ph, cd, dc = st["codes"][nm]
        b.set_phase_code(r, i, ph)
        b.set_cond(r, i, cd)
        b.set_decision(r, i, dc)
    for q, stp in enumerate(ps.par_steps):
        on, kids = st["par"][ps.names[stp]]
        b.register_children(r, q, on)
        for br, code in enumerate(kids):
            b.set_child_phase(r, q, br, A.PHASE_NAMES[code])


@pytest.mark.parametrize("seed", range(6))
def test_migration_map_matches_python_helper(seed):
    rng = np.random.default_rng(seed)
    old = M.random_story(rng, "s-", int(rng.integers(5, 300)), int(rng.integers(0, 10)))
    new = M.edit_story(rng, old, "s-e")
    ps_old, ps_new = M.story_from_steps(old), M.story_from_steps(new)
    hs_old, hs_new = _host_story(old), _host_story(new)
    assert [hs_new.name(i) for i in range(ps_new.S)] == ps_new.names
    want, added = M.migration_map(ps_old, ps_new)
    assert np.array_equal(hs_old.migration_map(hs_new), want)
    assert set(added) == set(ps_new.names) - set(ps_old.names) and added
    assert (want == A.MIGRATE_GONE).any()


@pytest.mark.parametrize("seed", range(4))
def test_batch_migrate_repacks_like_fresh_packing(seed):
    rng = np.random.default_rng(100 + seed)
    gens = [M.random_story(rng, "a-", int(rng.integers(40, 200)), 6), M.random_story(rng, "b-", 60, 3)]
    gens.append(M.edit_story(rng, gens[0], "a-e"))
    packed = [M.story_from_steps(s) for s in gens]
    hs = [_host_story(s) for s in gens]
    slots = [7, 9, 12]
    n = 80
    b = H.HostBatch(None, max(p.S for p in packed), max(p.child_nibbles() for p in packed),
                    A.F_COND | A.F_DECISION | A.F_CHILD | A.F_ALL_OUT, n)
    try:
        story = rng.integers(0, 2, n)
        states = [_codes(M.random_state(rng, packed[s])) for s in story]
        for r in range(n):
            b.add_run(hs[story[r]], slots[story[r]])
            _fill(b, r, packed[story[r]], states[r])
        rflags = np.full(n, A.RF_FAIL_FAST, np.uint8)
        assert np.array_equal(b.state(), M.pack_by_name(b.L, packed, story, slots, states, rflags))
        on = np.nonzero(story == 0)[0]
        assert b.migrate(hs[0], hs[2], slots[0], slots[2]) == len(on)
        story[on] = 2
        for r in on:
            states[r] = M.forget(states[r], packed[2])
        assert np.array_equal(b.state(), M.pack_by_name(b.L, packed, story, slots, states, rflags))
        # the migrated runs are runs of the new generation: its step indices address them
        r = int(on[0])
        nm = packed[2].names[0]
        b.set_phase_code(r, 0, 3)
        states[r]["codes"][nm] = (3,) + tuple(states[r]["codes"].get(nm, (0, 0, 0))[1:])
        assert np.array_equal(b.state(), M.pack_by_name(b.L, packed, story, slots, states, rflags))
    finally:
        b.close()


def test_batch_migrate_rejections_leave_the_mirror_unchanged():
    E, PA = A.STEP_ENGRAM, A.STEP_PARALLEL
    mk = lambda spec: [dict(name=nm, group=0, type=t, needs=[], branches=br) for nm, t, br in spec]
    old, wider, other = mk([("a", E, 0), ("p", PA, 3)]), mk([("p", PA, 4), ("a", E, 0)]), mk([("z", E, 0)])
    hs = [_host_story(s) for s in (old, wider, other)]
    b = H.HostBatch(None, 8, 16, A.F_CHILD, 4)
    try:
        b.add_run(hs[0], 1)
        b.add_run(hs[2], 2)
        b.set_phase_code(0, 0, 2)
        before = b.state().copy()
        with pytest.raises(A.FrontierError) as e:   # a kept parallel step changes its branch count
            b.migrate(hs[0], hs[1], 1, 3)
        assert e.value.status == A.BF_EINVAL
        with pytest.raises(A.FrontierError) as e:   # a run holds old_slot but belongs to another story
            b.migrate(hs[2], hs[0], 1, 3)
        assert e.value.status == A.BF_EINVAL
        with pytest.raises(A.FrontierError):        # a slot to itself
            b.migrate(hs[0], hs[0], 1, 1)
        assert np.array_equal(b.state(), before)
    finally:
        b.close()


def test_batch_migrate_keeps_child_padding():
    """with a child area of a nibble count that is not a multiple of 8, the nibbles past it up to the end of the last u32 word are
    kept, as the device migration keeps them"""
    rng = np.random.default_rng(77)
    gens = [M.random_story(rng, "a-", 90, 8)]
    gens.append(M.edit_story(rng, gens[0], "a-e"))
    packed = [M.story_from_steps(s) for s in gens]
    hs = [_host_story(s) for s in gens]
    child = max(p.child_nibbles() for p in packed) + 5
    b = H.HostBatch(None, max(p.S for p in packed), child, A.F_COND | A.F_DECISION | A.F_CHILD, 30)
    try:
        assert b.L.child_nibbles == child and child % 8
        states = [_codes(M.random_state(rng, packed[0])) for _ in range(30)]
        for r in range(30):
            b.add_run(hs[0], 4)
            _fill(b, r, packed[0], states[r])
        pad = rng.integers(1, 16, size=(30, 8 - child % 8))
        M.set_child_padding(b.L, b.state(), pad)
        assert b.migrate(hs[0], hs[1], 4, 6) == 30
        want = M.pack_by_name(b.L, packed, np.ones(30, int), [4, 6], [M.forget(s, packed[1]) for s in states],
                              np.full(30, A.RF_FAIL_FAST, np.uint8))
        M.set_child_padding(b.L, want, pad)
        assert np.array_equal(b.state(), want)
    finally:
        b.close()
