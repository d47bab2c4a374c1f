"""bf_resident_commit interleaved with every other resident call: after any call that changes the state records a commit is
refused (nothing changed) until a tick comes between, and the commit after that tick matches the host model over the records as
the device holds them."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import commit as M
from tests import runctl as R
from tests.test_gpu_commit import BIG, NONE_D, TABLES, _batch, entries_for

pytestmark = pytest.mark.gpu


def test_commit_after_every_resident_call():
    fr = Frontier(0)
    try:
        rng = np.random.default_rng(23)
        n, cap = 1200, 1400
        ts, slots, L, st = _batch(fr, rng, 128, A.F_COND | A.F_DECISION | A.F_ALL_OUT, True, n)
        topo = M.Topologies(ts, slots)
        h = fr.resident_create(L, cap)
        fr.resident_upload(h, 0, st)
        fr.resident_sched(h)
        fr.resident_timers(h, 2)
        fr.resident_runctl(h)
        other = fr.resident_create(L, cap)
        fr.resident_sched(other)
        fr.resident_timers(other, 2)
        fr.resident_runctl(other)
        state = {"n": n, "L": L, "rows": {}}

        def tick_and_commit():
            k = state["n"]
            res = fr.resident_tick(h, state["L"], k, NONE_D)[0]
            out = fr.resident_schedule([dict(handle=h, n_runs=k, runs_cap=k, events_cap=BIG)], TABLES, 50)
            rows = {r: v for r, v in state["rows"].items() if r < k}
            M.sched_rows(state["L"], out["parts"][0], rows)
            state["rows"] = rows
            before = fr.resident_download(h, 0, cap, state["L"].state_stride)
            ents = entries_for(rng, state["L"], topo, before, res, rows, k)
            want = M.commit(state["L"], topo, before, res, rows, k, ents)
            assert want[0] == 0
            assert fr.resident_commit(h, k, ents) == want[3]
            assert np.array_equal(fr.resident_download(h, 0, cap, state["L"].state_stride), before)
            return want[3]

        def refused():
            before = fr.resident_download(h, 0, cap, state["L"].state_stride)
            with pytest.raises(A.FrontierError):
                fr.resident_commit(h, state["n"])
            assert np.array_equal(fr.resident_download(h, 0, cap, state["L"].state_stride), before)

        def fresh_rows():   # moves and re-layouts give every run a new schedule row
            state["rows"] = {}

        tick_and_commit()
        d = np.zeros(2, dtype=Frontier.DELTA_DTYPE)
        d[0] = (3, 1, A.DELTA_PHASE, 0)
        d[1] = (4, 0, A.DELTA_RUN_FLAGS, 1)
        ops = [
            ("apply", lambda: fr.resident_apply(h, d)),
            ("upload", lambda: fr.resident_upload(h, 10, fr.resident_download(h, 10, 5, state["L"].state_stride))),
            ("fire", lambda: (fr.resident_apply(h, np.array([(7, 0, A.DELTA_DECISION, 0)], dtype=Frontier.DELTA_DTYPE)),
                              tick_and_commit(),
                              fr.resident_timers_arm(h, np.array([(7, 0, A.DEC_FAIL, 0, 5, 0)], dtype=Frontier.TIMER_DTYPE)),
                              fr.resident_fire(h, state["n"], 10))),
            ("runctl", lambda: fr.resident_runctl_put(h, np.array([(9, R.NONE, R.NONE, 2, (0, 0, 0))], dtype=R.PUT_DTYPE))),
            ("migrate", lambda: fr.resident_migrate(h, int(slots[1]), int(slots[2]), np.full(int(ts.S[1]), A.MIGRATE_GONE, np.uint16), state["n"])),
            ("redrive", lambda: fr.resident_redrive(h, np.array([(2, int(fr.resident_download(h, 2, 1, state["L"].state_stride)[0, :4].view("<u4")[0]),
                                                                   A.REDRIVE_ALL, 0)], dtype=Frontier.REDRIVE_DTYPE))),
            ("retire", lambda: (fr.resident_retire(h, state["n"], [0, 5]), state.update(n=state["n"] - 2), fresh_rows())),
            ("transfer", lambda: (fr.resident_transfer(h, other, state["n"], 0, [1, 2]), state.update(n=state["n"] - 2), fresh_rows())),
            ("reshape", lambda: (fr.resident_reshape(h, make_layout(160, L.child_nibbles, L.fields), cap),
                                 state.update(L=make_layout(160, L.child_nibbles, L.fields)), fresh_rows())),
            ("narrow", lambda: (fr.resident_narrow(h, L, state["n"]), state.update(L=L), fresh_rows())),
        ]
        for _name, op in ops:
            op()
            refused()
            tick_and_commit()
        # a schedule or a limiter put between a tick and its commit changes no state record: the commit goes on
        fr.resident_tick(h, state["L"], state["n"], NONE_D)
        fr.resident_schedule([dict(handle=h, n_runs=state["n"], runs_cap=state["n"], events_cap=BIG)], TABLES, 60)
        q = np.zeros(1, dtype=Frontier.SCHED_PUT_DTYPE)
        q[0] = (0, 1, 1, 3, A.SCHED_NONE, A.PHASE_RUNNING, (0, 0))
        fr.resident_sched_put(h, q)
        fr.resident_commit(h, state["n"])
    finally:
        fr.close()
