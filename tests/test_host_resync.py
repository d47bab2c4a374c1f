"""The host model of bf_resident_resync (tests/resync.py) on hand-built records: states that differ only by the rewrites a pass
never stores list nothing, one perturbed code of each field lists exactly that item, code 15 against 0 and codes past S list
nothing, a slot change lists one item, `fields` selects what is compared and written, and a repair leaves nothing to list."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import make_layout, pack_state
from tests import resync as M
from tests.test_host_commit import E, PAR, SLEEP, topo

F = A.resync_field
TYPES = [E, E, SLEEP, PAR, E]
S = len(TYPES)
FIELDS_IN = A.F_COND | A.F_DECISION | A.F_CHILD
R, P, SU, FA, SK = A.PHASE_RUNNING, A.PHASE_PAUSED, A.PHASE_SUCCEEDED, A.PHASE_FAILED, A.PHASE_SKIPPED


def _setup():
    ts = topo(TYPES, [2])
    ts2 = topo([E] * 3)
    from bobrapet_b200.frontier import TopologySet
    both = TopologySet([S, 3], [0, 0], np.concatenate([ts.row_ptr, ts2.row_ptr]), np.zeros(0, np.uint16),
                       np.concatenate([ts.step_flags, ts2.step_flags]), [1, 0], ts.parallel)
    L = make_layout(S, 8, FIELDS_IN)
    return M.Topos(both, [0, 1]), L


def _rec(L, phase, flags=0, cond=None, dec=None, child=(0, 0), reg=0, slot=0):
    ph = np.zeros((1, S), np.uint8)
    ph[0, :len(phase)] = phase
    c = np.zeros((1, S), np.uint8) if cond is None else np.asarray([cond], np.uint8)
    d = np.zeros((1, S), np.uint8) if dec is None else np.asarray([dec], np.uint8)
    ch = np.zeros((1, 8), np.uint8)
    ch[0, :len(child)] = child
    return pack_state(L, np.asarray([slot], np.uint32), np.asarray([flags], np.uint8), ph, c, d, ch, np.asarray([reg], np.uint64))[0]


BASE = dict(phase=[SU, R, P, R, 0], child=(R, 0), reg=1)


def _items(topos, L, dev, rec, fields=A.RESYNC_ALL_FIELDS):
    state = np.asarray([dev])
    return M.resync(L, topos, state, np.asarray([rec]), 1, fields=fields)


def test_identical_records_list_nothing():
    topos, L = _setup()
    d = _rec(L, **BASE)
    items, drifted, st, _ = _items(topos, L, d, d.copy())
    assert items.size == 0 and drifted.size == 0 and st.tobytes() == d.tobytes()


@pytest.mark.parametrize("case", ["fired_sleep", "joined_parallel", "fail_fast_skip"])
def test_unstored_rewrites_list_nothing(case):
    """the device's state before a pass's rewrites against the cluster's after them"""
    topos, L = _setup()
    if case == "fired_sleep":   # Paused with decision SUCCEED here, Succeeded without a decision there
        dev = _rec(L, [SU, R, P, 0, 0], dec=[0, 0, A.DEC_SUCCEED, 0, 0])
        rec = _rec(L, [SU, R, SU, 0, 0])
    elif case == "joined_parallel":   # Running with every child terminal here, Succeeded there
        dev = _rec(L, [SU, R, 0, R, 0], child=(SU, SU), reg=1)
        rec = _rec(L, [SU, R, 0, SU, 0], child=(SU, SU), reg=1)
    else:   # a fail-fast run's skips: 0 here, Skipped there
        dev = _rec(L, [FA, 0, 0, 0, 0], flags=A.RF_FAIL_FAST)
        rec = _rec(L, [FA, SK, SK, SK, SK], flags=A.RF_FAIL_FAST)
    assert _items(topos, L, dev, rec)[0].size == 0


PERTURB = [   # field, index, the caller's record's change, device value, record value
    (A.DELTA_PHASE, 1, dict(phase=[SU, FA, P, R, 0]), R, FA),
    (A.DELTA_COND, 1, dict(cond=[0, A.COND_HOLD, 0, 0, 0]), 0, A.COND_HOLD),
    (A.DELTA_DECISION, 4, dict(dec=[0, 0, 0, 0, A.DEC_FAIL]), 0, A.DEC_FAIL),
    (A.DELTA_CHILD, 1, dict(child=(R, R)), 0, R),
    (A.DELTA_RUN_FLAGS, 0, dict(flags=A.RF_REALTIME), 0, A.RF_REALTIME),
    (A.DELTA_REGISTERED, 0, dict(reg=0), 1, 0),
]


@pytest.mark.parametrize("field,index,change,dv,rv", PERTURB)
def test_one_perturbed_code_lists_that_item(field, index, change, dv, rv):
    topos, L = _setup()
    dev = _rec(L, **BASE)
    rec = _rec(L, **{**BASE, **change})
    items, drifted, st, _ = _items(topos, L, dev, rec)
    assert items.tolist() == [(0, index, field, 0, dv, rv)]
    assert drifted.tolist() == [0] and st[0].tobytes() == rec.tobytes()
    assert _items(topos, L, st[0], rec)[0].size == 0   # repaired: nothing left
    others = A.RESYNC_ALL_FIELDS & ~F(field)
    items, _, st, _ = _items(topos, L, dev, rec, fields=others)   # not selected: neither compared nor written
    assert items.size == 0 and st[0].tobytes() == dev.tobytes()


def test_code_15_padding_and_codes_past_S_list_nothing():
    topos, L = _setup()
    dev = _rec(L, [SU, R, P, R, 15], child=(R, 0), reg=1)
    rec = _rec(L, **BASE)
    rec[L.off_phase] |= 1 << 7           # step 7 >= S
    rec[L.off_cond] |= 1 << 6
    rec[L.off_child + 2] = 0x33          # nibbles past the desc's two branches
    rec[5:8] = 0xAA                      # reserved header bytes
    rec[9] |= 0x80                       # registered bit 15: no such desc
    assert _items(topos, L, dev, rec)[0].size == 0


def test_slot_change_lists_one_item_and_takes_the_whole_record():
    topos, L = _setup()
    dev = _rec(L, **BASE)
    rec = _rec(L, [SU, SU, SU], slot=1, dec=[1, 2, 3, 0, 0])
    items, drifted, st, _ = _items(topos, L, dev, rec)
    assert items.tolist() == [(0, 0, A.DELTA_TOPO_SLOT, 0, 0, 1)]
    assert st[0].tobytes() == rec.tobytes()


def test_terminal_steps_do_not_compare_their_inputs():
    topos, L = _setup()
    dev = _rec(L, [SU, SU, SU, SU, 0], child=(SU, SU), reg=1)
    rec = _rec(L, [SU, SU, SU, SU, 0], cond=[1, 2, 3, 1, 0], dec=[1, 2, 3, 1, 0], child=(FA, SK), reg=0)
    assert _items(topos, L, dev, rec)[0].size == 0


def test_dead_slot_compares_every_code_as_stored():
    topos, L = _setup()
    dev = _rec(L, [SU, R], slot=7)
    rec = _rec(L, [SU, R], slot=7)
    rec[L.off_phase] |= 1 << 7    # step 7: compared on a dead slot
    rec[L.off_child + 3] = 0x20   # nibble 7
    rec[15] |= 0x80               # registered bit 63
    items = _items(topos, L, dev, rec)[0]
    assert items[["field", "index"]].tolist() == [(A.DELTA_PHASE, 7), (A.DELTA_CHILD, 7), (A.DELTA_REGISTERED, 63)]


def test_stopped_run_keeps_its_stop():
    from tests import runctl as RC
    topos, L = _setup()
    dev = _rec(L, **BASE)
    area = RC.defaults(1)
    state = np.asarray([dev])
    RC.stop(area, state, 0, A.STOP_HOST)
    rec = _rec(L, **{**BASE, "flags": A.RF_FAIL_FAST})
    items, _, st, rc = M.resync(L, topos, state, np.asarray([rec]), 1, runctl=area)
    assert items.tolist() == [(0, 0, A.DELTA_RUN_FLAGS, 0, 0, A.RF_FAIL_FAST)]
    assert st[0].tobytes() == state[0].tobytes() and int(rc[0]["saved_flags"]) == A.RF_FAIL_FAST
