"""Redrive on the test side: the reference's two status resets restated over the oracle's StoryRun, and the packed statement of
bf_resident_redrive on state records.

Object level (oracle/pyoracle.py's StoryRun: step_states, gates, primitive_children, topology_terminated):
  reset_for_redrive        resetStoryRunForRedrive, internal/controller/runs/storyrun_controller.go:415-439
  reset_for_step_redrive   resetStoryRunForStepRedrive :740-789 over resolveRedriveFromStepSet :535-558
Packed level: `reset_packed` clears the reset set R in one record by the rules of include/bobrafrontier.h (phase 0, decision
PENDING, cond HOLD for `if` steps and PASS for the others, R's parallel descs unregistered with zero child nibbles,
BF_RF_TOPOLOGY_TERMINATED cleared).  `by_name_reset` carries a run's by-name state (tests/migration.py's form) through the
object-level reset, so that pack_by_name of its result is the record a redrive must leave.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from bobrapet_b200 import _abi as A
from oracle import pyoracle as O
from tests import migration as M
from tests.packing import PackedStory


# ------------------------------------------------------------------------------------------------ object level
def reset_for_redrive(srun: O.StoryRun) -> None:
    """resetStoryRunForRedrive (storyrun_controller.go:415-439): the status is cleared as a whole; of what the oracle models,
    StepStates, Gates, PrimitiveChildren, AllowedFailures, Conditions (the Degraded/TopologyTerminated condition) and Phase."""
    srun.phase = ""
    srun.primitive_children = {}
    srun.step_states = {}
    srun.gates = {}
    srun.allowed_failures = []
    srun.topology_terminated = False


def reset_for_step_redrive(srun: O.StoryRun, story: O.Story, step_name: str) -> Dict[str, bool]:
    """resetStoryRunForStepRedrive (storyrun_controller.go:740-789) for the set resolveRedriveFromStepSet (:535-558) gives:
    StepStates, Gates and PrimitiveChildren of those steps deleted, AllowedFailures filtered, Conditions cleared, a terminal
    Phase emptied.  -> the reset set"""
    steps = O.resolve_redrive_from_step_set(story, step_name)
    if not steps:
        return steps
    for name in steps:
        srun.step_states.pop(name, None)
        srun.gates.pop(name, None)
        srun.primitive_children.pop(name, None)
    srun.allowed_failures = [s for s in srun.allowed_failures if s not in steps]
    srun.topology_terminated = False          # Conditions = nil
    if O.is_terminal(srun.phase):
        srun.phase = ""
    return steps


# ------------------------------------------------------------------------------------------------ stories with `if` steps
def random_story(rng, prefix: str, S: int, n_par: int) -> List[dict]:
    """tests/migration.py's random story (three groups, parallel steps) with an `if` on about a fifth of the steps; the
    expressions name no step, so they add no dependency"""
    steps = M.random_story(rng, prefix, S, n_par)
    for s in steps:
        if rng.random() < 0.2:
            s["if"] = "{{ inputs.go }}"
    return steps


def packed_story(steps: Sequence[dict]) -> PackedStory:
    ps = M.story_from_steps(steps)
    has_if = {s["name"] for s in steps if s.get("if")}
    ps.flags = np.array([f | (A.SF_HAS_IF if n in has_if else 0) for n, f in zip(ps.names, ps.flags)], np.uint8)
    return ps


def oracle_story(steps: Sequence[dict]) -> O.Story:
    """the oracle's Story of the same steps: groups, needs and `if` (the type does not enter the reset set)"""
    grp = {g: [O.Step(s["name"], list(s["needs"]), ref=True, if_=s.get("if")) for s in steps if s["group"] == g] for g in range(3)}
    return O.Story(grp[A.GROUP_MAIN], grp[A.GROUP_COMPENSATION], grp[A.GROUP_FINALLY])


# ------------------------------------------------------------------------------------------------ by-name state <-> StoryRun
def by_name_reset(state: Dict, tt: bool, story: O.Story, ps: PackedStory, requests: Sequence[Optional[str]]):
    """A run's by-name state (tests/migration.py: codes {name: (phase, cond, decision)}, par {name: (registered, kids)}) and its
    TopologyTerminated flag, carried through the object-level resets of `requests` (a step name, or None for the whole run), one
    after the other as the reference applies annotations.  Phase and decision live in StepStates and Gates, a registered parallel
    step's children in PrimitiveChildren; the cond code is a host input, which the reset of its step sets to HOLD (`if` steps)
    or PASS.  -> (state, tt)"""
    srun = O.StoryRun(topology_terminated=tt)
    for name, (ph, _cd, dc) in state["codes"].items():
        if ph:
            srun.step_states[name] = O.StepState(str(ph))
        if dc:
            srun.gates[name] = O.GateStatus(str(dc))
    for name, (on, kids) in state["par"].items():
        srun.primitive_children[name] = [str(on)] + [str(k) for k in kids]
    reset = set()
    for step in requests:
        if step is None:
            reset_for_redrive(srun)
            reset |= set(ps.names)
        else:
            reset |= set(reset_for_step_redrive(srun, story, step))
    has_if = {ps.names[i] for i in range(ps.S) if ps.flags[i] & A.SF_HAS_IF}
    codes = {}
    for name, (_ph, cd, _dc) in state["codes"].items():
        ss, gs = srun.step_states.get(name), srun.gates.get(name)
        if name in reset:
            cd = A.COND_HOLD if name in has_if else A.COND_PASS
        codes[name] = (int(ss.phase) if ss else 0, cd, int(gs.state) if gs else 0)
    par = {}
    for name, pc in srun.primitive_children.items():
        par[name] = (pc[0] == "True", [int(k) for k in pc[1:]])
    return {"codes": codes, "par": par}, srun.topology_terminated


# ------------------------------------------------------------------------------------------------ packed statement
def closure_mask(ps: PackedStory, step: Optional[int], words: int) -> np.ndarray:
    """R as `words` u32 words: every step for None, else the redrive closure of `step` (the fixed point of
    tests/test_redrive_closure.py)"""
    from tests.test_redrive_closure import closure_packed
    m = np.zeros(words, np.uint32)
    if step is None:
        bits = np.zeros(words * 32, bool)
        bits[:ps.S] = True
        m[:] = np.packbits(bits, bitorder="little").view("<u4")
    else:
        c = closure_packed(ps, step)
        m[:c.shape[0]] = c
    return m


def reset_packed(L, rec: np.ndarray, ps: PackedStory, step: Optional[int]) -> None:
    """Clear R of a redrive from `step` (None: the whole run) in record `rec` ([state_stride] uint8), in place"""
    W = L.words
    m = closure_mask(ps, step, W)
    bits = np.unpackbits(m.view(np.uint8), bitorder="little").astype(bool)
    hold = np.zeros(W * 32, bool)
    hold[:ps.S] = (ps.flags & A.SF_HAS_IF) != 0
    hold = np.packbits(hold & bits, bitorder="little").view("<u4")

    def plane(off, k):
        return rec[off + k * W * 4:off + (k + 1) * W * 4].view("<u4")

    for k in range(4):
        plane(L.off_phase, k)[:] &= ~m
    if L.off_decision != A.OFF_NONE:
        for k in range(2):
            plane(L.off_decision, k)[:] &= ~m
    if L.off_cond != A.OFF_NONE:
        plane(L.off_cond, 0)[:] &= ~m
        plane(L.off_cond, 1)[:] = (plane(L.off_cond, 1) & ~m) | hold
    reg = int(rec[8:16].view("<u8")[0])
    cf = ps.child_first()
    for q, stp in enumerate(ps.par_steps):
        if not bits[stp]:
            continue
        reg &= ~(1 << q)
        if L.off_child != A.OFF_NONE:
            for c in range(int(cf[q]), int(cf[q]) + len(ps.par_branches[q])):
                rec[L.off_child + c // 2] &= np.uint8(~(0xF << (4 * (c & 1))) & 0xFF)
    rec[8:16] = np.array([reg], "<u8").view(np.uint8)
    rec[4] &= np.uint8(~A.RF_TOPOLOGY_TERMINATED & 0xFF)


# ------------------------------------------------------------------------------------------------ the delta path
def redrive_deltas(closure, L, story_of_slot: Dict[int, PackedStory], requests: np.ndarray, run_flags: np.ndarray) -> np.ndarray:
    """What a batcher without bf_resident_redrive sends for the same requests: the closures (closure(slots, steps, words) ->
    masks, Frontier.closure = bf_topology_closure, one query per distinct (slot, step)), then one delta per reset step and code field, per child nibble and registered bit of every reset
    parallel desc, and per run-flags byte, coalesced per (run, field, index) as bf_resident_apply requires.  `requests` holds
    only requests whose run holds their slot (REDRIVE_DTYPE); run_flags[run] is the run's current flags byte."""
    from bobrapet_b200.frontier import Frontier
    W32 = L.words * 32
    steps = requests["step"].astype(np.int64)
    named = steps != A.REDRIVE_ALL
    keys = sorted({(int(s), int(t)) for s, t in zip(requests["slot"][named], steps[named])})
    kidx = {k: i for i, k in enumerate(keys)}
    masks = closure([k[0] for k in keys], [k[1] for k in keys], L.words) if keys else np.zeros((0, L.words), np.uint32)
    kbits = np.unpackbits(masks.view(np.uint8), axis=1, bitorder="little").astype(bool) if keys else np.zeros((0, W32), bool)
    runs, inv = np.unique(requests["run"], return_inverse=True)
    bits = np.zeros((runs.size, W32), bool)
    slot_of = np.zeros(runs.size, np.int64)
    slot_of[inv] = requests["slot"]
    for i in range(requests.shape[0]):
        if named[i]:
            bits[inv[i]] |= kbits[kidx[(int(requests["slot"][i]), int(steps[i]))]]
        else:
            bits[inv[i], :story_of_slot[int(requests["slot"][i])].S] = True
    out = []

    def add(run, index, field, code):
        d = np.zeros(run.shape[0], Frontier.DELTA_DTYPE)
        d["run"], d["index"], d["field"], d["code"] = run, index, field, code
        out.append(d)

    ri, st = np.nonzero(bits)
    add(runs[ri], st, A.DELTA_PHASE, 0)
    if L.off_decision != A.OFF_NONE:
        add(runs[ri], st, A.DELTA_DECISION, A.DEC_PENDING)
    if L.off_cond != A.OFF_NONE:
        has_if = np.zeros((runs.size, W32), bool)
        for slot, ps in story_of_slot.items():
            on = slot_of == slot
            has_if[np.ix_(on, np.arange(ps.S))] = (ps.flags & A.SF_HAS_IF) != 0
        add(runs[ri], st, A.DELTA_COND, np.where(has_if[ri, st], A.COND_HOLD, A.COND_PASS))
    for slot, ps in story_of_slot.items():
        cf = ps.child_first()
        for q, stp in enumerate(ps.par_steps):
            on = np.nonzero((slot_of == slot) & bits[:, stp])[0]
            if not on.size:
                continue
            add(runs[on], q, A.DELTA_REGISTERED, 0)
            if L.off_child != A.OFF_NONE:
                for br in range(len(ps.par_branches[q])):
                    add(runs[on], int(cf[q]) + br, A.DELTA_CHILD, 0)
    add(runs, 0, A.DELTA_RUN_FLAGS, run_flags[runs] & ~np.uint8(A.RF_TOPOLOGY_TERMINATED))
    return np.concatenate(out) if out else np.zeros(0, Frontier.DELTA_DTYPE)
