"""Story edits on the test side: the by-name step map of bf_resident_migrate and a by-name state packer.

The reference keys a StoryRun's step state by step name and walks the current Story's allStorySteps on every reconcile, so after
an edit a surviving step keeps its state, a new step has none and a removed one drops out.  A migrated record must equal what
packing that by-name state against the new generation gives; `pack_by_name` is that packing, over the PackedStory form of
tests/packing.py.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import pack_state
from tests.packing import PackedStory


def migration_map(old: PackedStory, new: PackedStory) -> Tuple[np.ndarray, List[str]]:
    """-> (step_map [old.S] uint16: index in `new` of each step of `old` by name, or A.MIGRATE_GONE;
    the names of `new` that `old` lacks, whose state a batcher re-sends when an earlier generation had them)"""
    m = np.array([new.index.get(n, A.MIGRATE_GONE) for n in old.names], dtype=np.uint16)
    return m, [n for n in new.names if n not in old.index]


def story_from_steps(steps: Sequence[dict]) -> PackedStory:
    """steps: dicts of name, group (A.GROUP_*), type (A.STEP_*), needs (names of the same group), branches (count, parallel
    steps) -> PackedStory in allStorySteps order (main ++ compensations ++ finally)"""
    order = [s for g in (A.GROUP_MAIN, A.GROUP_COMPENSATION, A.GROUP_FINALLY) for s in steps if s["group"] == g]
    names = [s["name"] for s in order]
    index = {n: i for i, n in enumerate(names)}
    assert len(index) == len(names), "duplicate step names"
    rows, flags = [], []
    ps = PackedStory(names, index, None, None, None)
    for i, s in enumerate(order):
        rows.append(sorted({index[d] for d in s["needs"] if d in index}))
        flags.append(s["type"] | (s["group"] << A.SF_GROUP_SHIFT))
        if s["type"] == A.STEP_PARALLEL:
            ps.par_steps.append(i)
            ps.par_branches.append(["%s-b%d" % (s["name"], b) for b in range(s["branches"])])
            ps.par_allow.append([False] * s["branches"])
    ps.row_ptr = np.asarray(np.cumsum([0] + [len(r) for r in rows]), dtype=np.uint32)
    ps.col_idx = np.asarray([c for r in rows for c in r], dtype=np.uint16)
    ps.flags = np.asarray(flags, dtype=np.uint8)
    return ps


TYPES = [A.STEP_ENGRAM] * 6 + [A.STEP_GATE, A.STEP_SLEEP, A.STEP_WAIT, A.STEP_CONDITION, A.STEP_STOP, A.STEP_EXECUTE_STORY]
PHASES = list(range(15))


def random_story(rng, prefix: str, S: int, n_par: int) -> List[dict]:
    """S steps over the three groups (mostly main), n_par of them parallel with 1-12 branches; needs name earlier steps of the
    same group, so the graph is acyclic"""
    groups = rng.choice([0] * 6 + [1, 2], size=S)
    par = set(rng.choice(S, size=n_par, replace=False).tolist()) if n_par else set()
    steps: List[dict] = []
    for k in range(S):
        g = int(groups[k])
        same = [s["name"] for s in steps if s["group"] == g]
        needs = [str(x) for x in rng.choice(same, size=min(len(same), int(rng.integers(0, 3))), replace=False)] if same else []
        t = A.STEP_PARALLEL if k in par else int(rng.choice(TYPES))
        steps.append(dict(name="%ss%d" % (prefix, k), group=g, type=t, needs=needs,
                          branches=int(rng.integers(1, 13)) if t == A.STEP_PARALLEL else 0))
    return steps


def edit_story(rng, steps: Sequence[dict], prefix: str, parallel: bool = True) -> List[dict]:
    """An edited generation: deletes, renames, type changes (parallel <-> other when `parallel`), moves between main /
    compensations / finally, a reordered window, and inserted steps (some parallel).  Needs that now cross groups or name a
    removed step are dropped, so the graph stays acyclic; a kept parallel step keeps its branch count."""
    steps = [dict(s, needs=list(s["needs"])) for s in steps]
    n = len(steps)
    kill = set(rng.choice(n, size=max(1, n // 12), replace=False).tolist())
    steps = [s for i, s in enumerate(steps) if i not in kill]
    for k, i in enumerate(rng.choice(len(steps), size=max(2, len(steps) // 40), replace=False)):
        steps[i]["name"] = "%sr%d" % (prefix, k)   # a rename: the old name's state drops out, the new name starts empty
    for i in rng.choice(len(steps), size=max(2, len(steps) // 25), replace=False):
        s = steps[i]
        if s["type"] == A.STEP_PARALLEL:
            s["type"], s["branches"] = int(rng.choice(TYPES)), 0
        elif parallel and rng.random() < 0.4:
            s["type"], s["branches"] = A.STEP_PARALLEL, int(rng.integers(1, 13))
        else:
            s["type"] = int(rng.choice(TYPES))
    for i in rng.choice(len(steps), size=max(2, len(steps) // 25), replace=False):
        steps[i]["group"] = int(rng.integers(0, 3))
    lo = int(rng.integers(0, max(1, len(steps) - 12)))
    window = steps[lo:lo + 12]
    rng.shuffle(window)
    steps[lo:lo + 12] = window
    for k in range(n // 12 + 1):
        g = int(rng.choice([0, 0, 0, 1, 2]))
        same = [s["name"] for s in steps if s["group"] == g]
        t = A.STEP_PARALLEL if parallel and rng.random() < 0.2 else int(rng.choice(TYPES))
        steps.insert(int(rng.integers(0, len(steps) + 1)), dict(
            name="%sn%d" % (prefix, k), group=g, type=t,
            needs=[str(x) for x in rng.choice(same, size=min(len(same), 2), replace=False)] if same else [],
            branches=int(rng.integers(1, 13)) if t == A.STEP_PARALLEL else 0))
    group_of = {s["name"]: s["group"] for s in steps}
    n_par = 0
    for s in steps:
        s["needs"] = [d for d in s["needs"] if group_of.get(d) == s["group"]]
        if s["type"] == A.STEP_PARALLEL:
            n_par += 1
            if n_par > A.MAX_PARALLEL:
                s["type"], s["branches"] = A.STEP_ENGRAM, 0
    return steps


def random_state(rng, ps: PackedStory) -> Dict:
    """a run's by-name state over story `ps` (the form pack_by_name takes)"""
    codes = {n: (int(rng.choice(PHASES)), int(rng.integers(0, 4)), int(rng.integers(0, 4))) for n in ps.names}
    par = {ps.names[stp]: (bool(rng.integers(0, 2)), [int(x) for x in rng.integers(0, 15, size=len(br))])
           for stp, br in zip(ps.par_steps, ps.par_branches)}
    return {"codes": codes, "par": par}


def forget(state: Dict, ps: PackedStory) -> Dict:
    """what a run keeps after moving to `ps`: the state of its steps, and of its parallel steps that are parallel there (an engine
    that stores state by index has no slot for the rest, which is why a re-added name starts empty)"""
    par_names = {ps.names[s] for s in ps.par_steps}
    return {"codes": {n: c for n, c in state["codes"].items() if n in ps.index},
            "par": {n: p for n, p in state["par"].items() if n in par_names}}


def set_child_padding(L, rec: np.ndarray, values: np.ndarray) -> None:
    """write values[r, k] into the k-th nibble past L.child_nibbles of record r, up to the end of the child area's last u32 word
    (padding no field reads; a migration keeps it)"""
    pad = range(L.child_nibbles, (L.child_nibbles + 7) // 8 * 8)
    for k, p in enumerate(pad):
        b = L.off_child + p // 2
        sh = 4 * (p & 1)
        rec[:, b] = (rec[:, b] & ~np.uint8(0xF << sh)) | ((values[:, k].astype(np.uint8) & 0xF) << sh)


def pack_by_name(L, stories: Sequence[PackedStory], story_of_run: Sequence[int], slots: Sequence[int],
                 states: Sequence[Dict], run_flags: np.ndarray) -> np.ndarray:
    """State records of runs whose state is held by name: states[r] = {"codes": {name: (phase, cond, decision)},
    "par": {parallel step name: (registered, [child phase per branch])}}.  A step without an entry packs as 0; a parallel
    desc takes the entry of its step's name, when there is one."""
    n = len(states)
    W32 = L.words * 32
    phase, cond, dec = (np.zeros((n, W32), np.uint8) for _ in range(3))
    child = np.zeros((n, max(L.child_nibbles, 1)), np.uint8)
    reg = np.zeros(n, np.uint64)
    sl = np.zeros(n, np.uint32)
    for r, st in enumerate(states):
        ps = stories[story_of_run[r]]
        sl[r] = slots[story_of_run[r]]
        for i, name in enumerate(ps.names):
            phase[r, i], cond[r, i], dec[r, i] = st["codes"].get(name, (0, 0, 0))
        cf = ps.child_first()
        for q, stp in enumerate(ps.par_steps):
            got = st["par"].get(ps.names[stp])
            if got is None:
                continue
            on, kids = got
            assert len(kids) == len(ps.par_branches[q])
            if on:
                reg[r] |= np.uint64(1) << np.uint64(q)
            if L.off_child != A.OFF_NONE:
                child[r, int(cf[q]):int(cf[q]) + len(kids)] = kids
    return pack_state(L, sl, run_flags, phase, cond, dec, child if L.off_child != A.OFF_NONE else None, reg)
