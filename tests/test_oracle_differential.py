"""Object-shaped oracle (pyoracle: the function-by-function restatement of dag.go) vs the packed C oracle
(packed_ref.c: what the kernel must equal) on random Stories — every step type, three step groups, template
references through sanitised aliases, gates/sleeps/waits with real timestamps, parallel joins, realtime,
fail-fast on/off, queued Pending, template-safety failures.  Both single-pass and fixpoint."""
import random

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import unpack_result
from oracle import packed as PK
from oracle import pyoracle as O
from tests import packing as P

PHASE_POOL = ["", "", "", "Pending", "Running", "Succeeded", "Succeeded", "Succeeded", "Failed", "Finished", "Canceled",
              "Compensated", "Paused", "Blocked", "Scheduling", "Timeout", "Aborted", "Skipped"]


def _rand_story(rng: random.Random):
    n_main, n_comp, n_fin = rng.randint(1, 14), rng.choice([0, 0, 1, 3]), rng.choice([0, 0, 1, 2])
    names = ["s-%d" % i if rng.random() < 0.5 else "s%d" % i for i in range(n_main + n_comp + n_fin)]
    codes = {}

    def mk(i, pool):
        name = names[i]
        t = rng.choice(["engram"] * 5 + ["condition", "parallel", "sleep", "stop", "wait", "executeStory", "gate", "gate"])
        st = O.Step(name=name, ref=(t == "engram"), type=("" if t == "engram" else t))
        earlier = [n for n in pool if n != name]
        if earlier:
            st.needs = rng.sample(earlier, k=min(len(earlier), rng.choice([0, 1, 1, 2, 3])))
        if rng.random() < 0.15:
            st.allow_failure = True
        r = rng.random()
        if r < 0.3:
            code = rng.choice([A.COND_PASS, A.COND_PASS, A.COND_SKIP, A.COND_HOLD, A.COND_FAIL])
            codes[name] = code
            ref = ""
            if earlier and rng.random() < 0.5:  # implicit dependency through a template reference (alias form)
                ref = " steps.%s.output.ok" % O.sanitize_step_identifier(rng.choice(earlier))
            st.if_ = ('{{ env "X" }}' if code == A.COND_FAIL else "{{ inputs.c_%s%s }}" % (O.sanitize_step_identifier(name), ref))
        if t == "gate":
            st.with_ = rng.choice([None, {"timeout": "10s"}, {"timeout": "10s", "onTimeout": "skip"}])
        elif t == "sleep":
            st.with_ = rng.choice([None, {"duration": "5s"}, {"duration": "50s"}, {"duration": "bogus"}])
        elif t == "wait":
            st.with_ = rng.choice([{"until": "{{ inputs.w_%s }}" % O.sanitize_step_identifier(name)},
                                   {"until": "{{ inputs.w_%s }}" % O.sanitize_step_identifier(name), "timeout": "10s", "onTimeout": rng.choice(["skip", "fail"])},
                                   None])
            codes["wait:" + name] = rng.random() < 0.4
        elif t == "parallel":
            st.with_ = {"steps": [{"name": "b%d" % k, **({"allowFailure": True} if rng.random() < 0.3 else {})}
                                  for k in range(rng.randint(1, 5))]}
        elif t == "engram" and earlier and rng.random() < 0.2:
            st.with_ = {"x": "{{ steps['%s'].output }}" % rng.choice(earlier)}
        return st

    main = [mk(i, names[:i]) for i in range(n_main)]
    comp = [mk(i, names[n_main:i]) for i in range(n_main, n_main + n_comp)]
    fin = [mk(i, names[n_main + n_comp:i]) for i in range(n_main + n_comp, len(names))]
    story = O.Story(main, comp, fin, realtime=rng.random() < 0.2,
                    continue_on_step_failure=rng.choice([None, None, True, False]))
    return story, codes


def _rand_run(rng: random.Random, story: O.Story):
    srun = O.StoryRun(topology_terminated=rng.random() < 0.3)
    step_runs = []
    progress = rng.random()
    for st in O.all_story_steps(story):
        ph = rng.choice(PHASE_POOL) if rng.random() < progress else rng.choice(["", "", "", "Pending"])
        if ph:
            msg = (O.QUEUED_PREFIXES[rng.randrange(4)] + " (2 running, limit 2)") if (ph == "Pending" and rng.random() < 0.5) else ""
            srun.step_states[st.name] = O.StepState(ph, msg, started_at=rng.choice([None, 90.0, 99.0]))
        if st.type == "gate" and not st.ref and rng.random() < 0.6:
            srun.gates[st.name] = O.GateStatus(rng.choice(["", "Pending", "Approved", "Rejected"]), "m")
        if st.type == "parallel" and not st.ref and rng.random() < 0.7:
            kids = []
            all_done = rng.random() < 0.5
            for b in O.parse_parallel_branches(st):
                nm = "%s-%s" % (st.name, b.name)
                kids.append(nm)
                if rng.random() < 0.9:
                    cp = rng.choice(["Succeeded", "Succeeded", "Skipped", "Failed"]) if all_done else \
                        rng.choice(["", "Running", "Succeeded", "Failed", "Pending"])
                    step_runs.append(O.StepRun(nm, b.name, cp))
            srun.primitive_children[st.name] = kids
    return srun, step_runs


def _evaluator(codes):
    def ev(step_name, expr, vars_):
        if expr.startswith("{{ inputs.w_"):
            return codes.get("wait:" + step_name, False)
        c = codes.get(step_name, A.COND_PASS)
        if c == A.COND_HOLD:
            raise O.EvaluationBlocked("blocked")
        return c == A.COND_PASS
    return ev


def _clone_run(srun):
    return O.StoryRun({k: v.copy() for k, v in srun.step_states.items()},
                      {k: O.GateStatus(v.state, v.message) for k, v in srun.gates.items()},
                      {k: list(v) for k, v in srun.primitive_children.items()}, srun.topology_terminated)


@pytest.mark.parametrize("seed", range(400))
def test_single_pass_object_vs_packed(seed):
    rng = random.Random(seed)
    story, codes = _rand_story(rng)
    if O.validate_runtime_dependency_graph(O.all_story_steps(story)) is not None:
        pytest.skip("generated an invalid graph")
    try:
        ps = P.pack_story(story)
    except ValueError:
        pytest.skip("dangling cross-group alias reference")
    srun, step_runs = _rand_run(rng, story)
    ev, now = _evaluator(codes), 100.0
    L, state = P.pack_runs([story], [ps], [_clone_run(srun)], [0], [0], [step_runs], ev, {"inputs": {}, "steps": {}}, now)
    res, counts = PK.evaluate(PK.PackedTopologies(P.topology_set([ps])), L, state)
    got = unpack_result(L, res, ps.S)
    names = ps.names
    pick = lambda key: [names[i] for i in np.nonzero(got[key][0])[0]]

    it = O.run_dag_iteration(srun, story, step_runs, ev, {"inputs": {}, "steps": {}}, now)
    order = {n: i for i, n in enumerate(names)}
    srt = lambda xs: sorted(xs, key=order.get)
    assert pick("ready") == srt(it.ready.ready)
    assert pick("skip") == srt(it.ready.skipped)                      # contract: skip_max
    assert set(it.ready_min.skipped) <= set(it.ready.skipped)        # and the other bound is a subset
    assert it.ready_min.ready == it.ready.ready
    assert pick("fail") == srt(it.ready.failed_now)
    assert pick("needs_cond") == srt(it.ready.evaluated_if)
    assert pick("skip_dep") == srt([n for n, r in it.ready.skip_reasons.items() if "failed dependency" in r])
    want_phase = [P.phase_code(srun.step_states.get(n)) for n in names]
    assert got["phase_out"][0].tolist() == want_phase
    summ = int(got["summary"][0])
    grp = {"main": 0, "compensation": 1, "finally": 2, "finalize": 3}[it.group]
    assert summ & A.SUM_GROUP_MASK == grp
    assert bool(summ & A.SUM_MAIN_DONE) == it.main_done and bool(summ & A.SUM_MAIN_FAILED) == it.main_failed
    assert bool(summ & A.SUM_COMP_DONE) == it.comp_done and bool(summ & A.SUM_FINAL_DONE) == it.final_done
    assert bool(summ & A.SUM_COMP_FAILED) == it.comp_failed and bool(summ & A.SUM_FINAL_FAILED) == it.final_failed


@pytest.mark.parametrize("seed", range(1000, 1250))
def test_fixpoint_object_vs_packed(seed):
    _fixpoint_object_vs_packed(seed, 0)


@pytest.mark.parametrize("cap", [1, 2, 3, "S+5"])
@pytest.mark.parametrize("seed", range(1000, 1250))
def test_fixpoint_iteration_cap_object_vs_packed(seed, cap):
    """max_iterations = cap: the object oracle's loop and the packed oracle's stop after the same iteration"""
    _fixpoint_object_vs_packed(seed, cap)


def _fixpoint_object_vs_packed(seed, cap):
    """cap: the iteration limit (max_iterations), 0 = the default S + 1"""
    rng = random.Random(seed)
    story, codes = _rand_story(rng)
    if O.validate_runtime_dependency_graph(O.all_story_steps(story)) is not None:
        pytest.skip("generated an invalid graph")
    try:
        ps = P.pack_story(story)
    except ValueError:
        pytest.skip("dangling cross-group alias reference")
    srun, step_runs = _rand_run(rng, story)
    ev, now = _evaluator(codes), 100.0
    L, state = P.pack_runs([story], [ps], [_clone_run(srun)], [0], [0], [step_runs], ev, {"inputs": {}, "steps": {}}, now)
    pt = PK.PackedTopologies(P.topology_set([ps]))
    max_iter = ps.S + 5 if cap == "S+5" else cap
    res, counts = PK.evaluate(pt, L, state, A.EVAL_FIXPOINT, max_iter)
    got = unpack_result(L, res, ps.S)
    names = ps.names
    pick = lambda key: [names[i] for i in np.nonzero(got[key][0])[0]]

    iters, launched, skipped, expansion, last = O.run_dag_iterations(srun, story, step_runs, ev, {"inputs": {}, "steps": {}},
                                                                     now, max_iterations=(max_iter or None), device_contract=True)
    if max_iter:
        assert iters <= max_iter
    order = {n: i for i, n in enumerate(names)}
    srt = lambda xs: sorted(set(xs), key=order.get)
    assert pick("ready") == srt(launched)
    assert pick("skip") == srt(skipped)
    assert (int(got["summary"][0]) >> A.SUM_ITER_SHIFT) == iters
    want_phase = [P.phase_code(srun.step_states.get(n)) for n in names]
    assert got["phase_out"][0].tolist() == want_phase
    exp, n = PK.expand(pt, L, state, res, 4096)
    assert n == len(set(expansion)) == int(got["n_expansion"][0])
    assert [(names[e["step"]], ps.par_branches[ps.par_steps.index(int(e["step"]))][int(e["branch"])]) for e in exp] == \
        sorted(set(expansion), key=lambda t: (order[t[0]], ps.par_branches[ps.par_steps.index(order[t[0]])].index(t[1])))


@pytest.mark.parametrize("mode", ["single", "fixpoint"])
@pytest.mark.parametrize("seed", range(4))
def test_packed_reads_reserved_and_padding_as_clean(seed, mode):
    """The reserved phase / child code 15 reads as 0, and codes at or past a run's own S are not read: the packed oracle
    gives a batch full of both the same bytes as its cleaned twin.  The GPU cases with `reserved=` / `padding=` rely on it."""
    from tests import randgen
    rng = np.random.default_rng(7000 + seed)
    smax = [40, 257, 96, 33][seed]
    ts = randgen.random_topologies(rng, 30, 1, smax, max_deg=4, fill=0.5, branch_choices=(0, 3, 8, 9, 33, 300))
    slots = np.arange(ts.count, dtype=np.uint32)
    fields = A.F_COND | A.F_DECISION | A.F_ALL_OUT
    L, dirty, topo = randgen.random_state(rng, ts, slots, 600, fields, phase_mix=("any" if seed % 2 else "progress"),
                                          reserved=0.1, padding=True)
    clean = randgen.cleaned(L, dirty, ts, topo)
    assert not np.array_equal(dirty, clean)
    flags = A.EVAL_FIXPOINT if mode == "fixpoint" else 0
    pt = PK.PackedTopologies(ts, slots)
    got, gc = PK.evaluate(pt, L, dirty, flags)
    want, wc = PK.evaluate(pt, L, clean, flags)
    assert np.array_equal(got, want) and gc == wc
    assert np.array_equal(randgen.cleaned(L, clean, ts, topo), clean)
    gexp, gn = PK.expand(pt, L, dirty, got, int(gc["expansion"]))
    wexp, wn = PK.expand(pt, L, clean, want, int(wc["expansion"]))
    assert gn == wn and np.array_equal(gexp, wexp)
