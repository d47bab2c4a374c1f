"""Redrive without a device: the object-level resets of the reference on hand cases shaped after its envtest specs, the packed
statement of bf_resident_redrive against them on random stories, the C++ host mirror's bfh_batch_redrive against both, and the
constants and struct size every binding shares."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import host as H
from bobrapet_b200.frontier import Frontier
from bobrapet_b200.records import make_layout
from oracle import pyoracle as O
from tests import migration as M
from tests import redrive as RD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = A.F_COND | A.F_DECISION | A.F_CHILD | A.F_ALL_OUT


def test_full_reset_clears_the_status():
    """storyrun_controller_test.go:185-271: a redrive token clears StepStates, Gates, PrimitiveChildren, AllowedFailures,
    Conditions and Phase"""
    srun = O.StoryRun(step_states={"step1": O.StepState("Running")}, gates={"gate1": O.GateStatus("Approved")},
                      primitive_children={"parallel": ["child-1"]}, topology_terminated=True, allowed_failures=["step0"],
                      phase="Running")
    RD.reset_for_redrive(srun)
    assert (srun.step_states, srun.gates, srun.primitive_children, srun.allowed_failures) == ({}, {}, {}, [])
    assert not srun.topology_terminated and srun.phase == ""


def test_step_redrive_drops_the_primitive_children_of_the_step():
    """storyrun_controller_test.go:573-637: after `step1:token` the PrimitiveChildren of step1 are gone; step1's downstream
    steps lose their state, an upstream step and a step of another group keep theirs"""
    story = O.Story([O.Step("step0", ref=True), O.Step("step1", ["step0"], type="parallel"), O.Step("step2", ["step1"], ref=True),
                     O.Step("side", ref=True)], [], [O.Step("fin", ["step1"], ref=True)])
    srun = O.StoryRun(step_states={n: O.StepState("Succeeded") for n in ("step0", "step1", "step2", "side", "fin")},
                      gates={"step2": O.GateStatus("Approved")}, primitive_children={"step1": ["primitive-branch-steprun"]},
                      topology_terminated=True, allowed_failures=["step0", "step2"], phase="Failed")
    got = RD.reset_for_step_redrive(srun, story, "step1")
    assert set(got) == {"step1", "step2"}
    assert "step1" not in srun.primitive_children and srun.primitive_children == {}
    assert set(srun.step_states) == {"step0", "side", "fin"} and srun.gates == {}
    assert srun.allowed_failures == ["step0"] and not srun.topology_terminated and srun.phase == ""
    with pytest.raises(KeyError):
        RD.reset_for_step_redrive(srun, story, "nope")          # "step %q not found", :541


def test_packed_hand_case():
    """the packed statement on the hand case of the step redrive: step1 (parallel, 3 branches) and step2 reset, step2's `if`
    held, the child nibbles of step1 zeroed, the padding after them kept"""
    steps = [dict(name="step0", group=0, type=A.STEP_ENGRAM, needs=[], branches=0),
             dict(name="step1", group=0, type=A.STEP_PARALLEL, needs=["step0"], branches=3),
             dict(name="step2", group=0, type=A.STEP_GATE, needs=["step1"], branches=0, **{"if": "{{ inputs.go }}"}),
             dict(name="p2", group=0, type=A.STEP_PARALLEL, needs=[], branches=2)]
    ps = RD.packed_story(steps)
    L = make_layout(4, ps.child_nibbles(), ALL)
    st = {"codes": {n: (3, 1, 1) for n in ps.names}, "par": {"step1": (True, [3, 4, 5]), "p2": (True, [6, 7])}}
    rec = M.pack_by_name(L, [ps], [0], [5], [st], np.array([A.RF_TOPOLOGY_TERMINATED | A.RF_FAIL_FAST], np.uint8))
    rec[0, L.off_child + 1] |= 0x90                      # padding nibble 3 of step1's word
    RD.reset_packed(L, rec[0], ps, ps.index["step1"])
    want_st = {"codes": {"step0": (3, 1, 1), "step1": (0, A.COND_PASS, 0), "step2": (0, A.COND_HOLD, 0), "p2": (3, 1, 1)},
               "par": {"p2": (True, [6, 7])}}
    want = M.pack_by_name(L, [ps], [0], [5], [want_st], np.array([A.RF_FAIL_FAST], np.uint8))
    want[0, L.off_child + 1] |= 0x90
    assert np.array_equal(rec, want)


def _cases(rng, n_stories=4, n_runs=60, lo=20, hi=90, n_par=5):
    gens = [RD.random_story(rng, "t%d-" % k, int(rng.integers(lo, hi)), n_par) for k in range(n_stories)]
    packed = [RD.packed_story(s) for s in gens]
    stories = [RD.oracle_story(s) for s in gens]
    story = rng.integers(0, n_stories, n_runs)
    states = [M.random_state(rng, packed[s]) for s in story]
    tt = rng.random(n_runs) < 0.5
    reqs = []   # (run, step name or None)
    for r in range(n_runs):
        ps = packed[story[r]]
        for _ in range(int(rng.integers(0, 4))):
            reqs.append((r, None if rng.random() < 0.15 else ps.names[int(rng.integers(0, ps.S))]))
        if reqs and reqs[-1][0] == r and rng.random() < 0.3:
            reqs.append(reqs[-1])                           # a duplicate
    return gens, packed, stories, story, states, tt, reqs


def _expected(L, packed, stories, story, states, tt, reqs, slots):
    out_states, out_tt = [], []
    for r in range(len(states)):
        mine = [s for rr, s in reqs if rr == r]
        st, t = RD.by_name_reset(states[r], bool(tt[r]), stories[story[r]], packed[story[r]], mine) if mine else (states[r], bool(tt[r]))
        out_states.append(st)
        out_tt.append(t)
    flags = np.array([A.RF_FAIL_FAST | (A.RF_TOPOLOGY_TERMINATED if t else 0) for t in out_tt], np.uint8)
    return M.pack_by_name(L, packed, story, slots, out_states, flags)


@pytest.mark.parametrize("seed", range(6))
def test_packed_reset_equals_object_level_reset(seed):
    rng = np.random.default_rng(500 + seed)
    gens, packed, stories, story, states, tt, reqs = _cases(rng)
    slots = list(range(3, 3 + len(packed)))
    L = make_layout(max(p.S for p in packed), max(p.child_nibbles() for p in packed), ALL)
    flags = np.array([A.RF_FAIL_FAST | (A.RF_TOPOLOGY_TERMINATED if t else 0) for t in tt], np.uint8)
    rec = M.pack_by_name(L, packed, story, slots, states, flags)
    for r, name in reqs:
        ps = packed[story[r]]
        RD.reset_packed(L, rec[r], ps, None if name is None else ps.index[name])
    want = _expected(L, packed, stories, story, states, tt, reqs, slots)
    bad = np.nonzero((rec != want).any(axis=1))[0]
    assert bad.size == 0, bad[:10]
    assert any(n is None for _, n in reqs) and tt.any()


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], if_expr=s.get("if"), needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


def fill_mirror(b, r, ps, st, tt):
    """the run's by-name state through the mirror's setters (child phases take a phase name: code 14 is not one)"""
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
    b.set_run_flags(r, topology_terminated=bool(tt))


def child_codes(st):
    return {"codes": st["codes"], "par": {k: (on, [c if c < 14 else 1 for c in kids]) for k, (on, kids) in st["par"].items()}}


@pytest.mark.parametrize("seed", range(4))
def test_host_mirror_redrive_matches_both(seed):
    rng = np.random.default_rng(900 + seed)
    gens, packed, stories, story, states, tt, reqs = _cases(rng)
    states = [child_codes(s) for s in states]
    hs = [_host_story(s) for s in gens]
    assert all(hs[k].name(i) == packed[k].names[i] for k in range(len(hs)) for i in range(packed[k].S))
    slots = list(range(3, 3 + len(packed)))
    n = len(states)
    b = H.HostBatch(None, max(p.S for p in packed), max(p.child_nibbles() for p in packed), ALL, n)
    try:
        for r in range(n):
            assert b.add_run(hs[story[r]], slots[story[r]]) == r
            fill_mirror(b, r, packed[story[r]], states[r], tt[r])
        packed_rec = b.state().copy()
        b.redrive([r for r, _ in reqs], [-1 if nm is None else packed[story[r]].index[nm] for r, nm in reqs])
        want = _expected(b.L, packed, stories, story, states, tt, reqs, slots)
        assert np.array_equal(b.state(), want)
        for r, nm in reqs:
            ps = packed[story[r]]
            RD.reset_packed(b.L, packed_rec[r], ps, None if nm is None else ps.index[nm])
        assert np.array_equal(b.state(), packed_rec)
        before = b.state().copy()
        with pytest.raises(A.FrontierError):
            b.redrive([0, n], [-1, -1])                     # a run out of range
        with pytest.raises(A.FrontierError):
            b.redrive([0], [packed[story[0]].S])            # a step past the story
        with pytest.raises(A.FrontierError):
            b.redrive([0], [-2])
        assert np.array_equal(b.state(), before)
    finally:
        b.close()


def test_redrive_constants_and_struct_size_agree():
    hdr = open(os.path.join(ROOT, "include", "bobrafrontier.h")).read()
    m = re.search(r"#define BF_REDRIVE_ALL (0x[0-9a-fA-F]+)u", hdr)
    go = open(os.path.join(ROOT, "go", "frontier", "frontier.go")).read()
    g = re.search(r"\bRedriveAll\s*=\s*(0x[0-9a-fA-F]+)", go)
    assert m and g and int(m.group(1), 16) == A.REDRIVE_ALL == int(g.group(1), 16) == 0xFFFFFFFF
    assert C.sizeof(A.Redrive) == Frontier.REDRIVE_DTYPE.itemsize == 16
    assert [f for f, _ in A.Redrive._fields_] == list(Frontier.REDRIVE_DTYPE.names) == ["run", "slot", "step", "reserved"]


def test_bf_redrive_is_16_bytes_in_c(tmp_path):
    src = tmp_path / "size.c"
    src.write_text('#include "bobrafrontier.h"\n#include <stddef.h>\n'
                   '_Static_assert(sizeof(bf_redrive) == 16, "bf_redrive");\n'
                   '_Static_assert(offsetof(bf_redrive, step) == 8, "bf_redrive.step");\n')
    out = subprocess.run(["gcc", "-std=c11", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
