"""The host models of a transfer to a batch of another ctx (bf_resident_transfer_ctx), without a GPU: tests/lifecycle.py's
AreaBatch.transfer and tests/transfer.py's transfer with a slot map.  Through an identity map they leave exactly what the
transfer within one ctx leaves; through a permuted map they differ from it only in the arrivals' header slot word.  The slot
verdicts and the map-entry refusals follow the header's order."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import make_layout
from tests import resident_model as RM
from tests import transfer as TR
from tests.lifecycle import MOVED, RUNCTL, SCHED, TIMERS, records_of, seeded, template_records
from tests.seqrig import random_records, story_pool

FIELDS = A.F_COND | A.F_DECISION | A.F_OUT_FAIL | A.F_OUT_SKIP_DEP
L = make_layout(64, 0, FIELDS)
S = [22, 20]
NOW = 5000


def _area_pair(slots):
    a = seeded(L, 24, TIMERS | SCHED | RUNCTL, 5, records_of(template_records(L, slots, S), 16), S[0] - 1, NOW)[0]
    b = seeded(L, 24, TIMERS | SCHED | RUNCTL, 5, records_of(template_records(L, slots, S), 4), S[0] - 1, NOW)[0]
    return a, b


def _areas(b):
    return [b.state, b.timers, b.runctl, b.sched.download(0, b.cap)]


def test_area_batch_identity_map_is_the_in_ctx_transfer():
    a1, b1 = _area_pair([3, 7])
    a2, b2 = _area_pair([3, 7])
    assert a1.transfer(b1, b1.n, MOVED) == a2.transfer(b2, b2.n, MOVED, slot_map=np.arange(8, dtype=np.uint32))
    for x, y in zip(_areas(a1) + _areas(b1), _areas(a2) + _areas(b2)):
        assert np.array_equal(x, y)


def test_area_batch_permuted_map_changes_only_the_slot_words():
    a1, b1 = _area_pair([3, 7])
    a2, b2 = _area_pair([3, 7])
    m = np.full(8, A.SLOT_NONE, np.uint32)
    m[3], m[7] = 11, 2
    a1.transfer(b1, b1.n, MOVED)
    a2.transfer(b2, b2.n, MOVED, slot_map=m)
    for x, y in zip(_areas(a1) + _areas(b1)[1:], _areas(a2) + _areas(b2)[1:]):
        assert np.array_equal(x, y)
    arrivals = slice(4, 4 + len(MOVED))
    diff = np.nonzero((b1.state != b2.state).any(axis=0))[0]
    assert set(diff.tolist()) <= {0, 1, 2, 3} and diff.size
    assert np.array_equal(b1.state[:, 4:], b2.state[:, 4:])
    w1 = np.ascontiguousarray(b1.state[arrivals, 0:4]).view("<u4").ravel()
    w2 = np.ascontiguousarray(b2.state[arrivals, 0:4]).view("<u4").ravel()
    assert np.array_equal(w2, m[w1])


def _rm_pair(order1):
    """two registries over one pool (the second with the Stories in order1) and a source batch of 12 runs in the first"""
    rng = np.random.default_rng(5)
    pool = story_pool(rng, 10, 20, 1, 2)
    regs = [RM.Registry(pool), RM.Registry(pool)]
    for k in range(len(pool)):
        regs[0].put(k)
    for k in order1:
        regs[1].put(k)
    Ls = make_layout(32, max(p.child_nibbles() for p in pool), A.F_COND | A.F_CHILD | A.F_ALL_OUT)
    src = RM.Batch(regs[0], Ls, 16)
    story = rng.integers(0, 2, 12)
    src.upload(0, random_records(rng, Ls, [pool[k] for k in story], story))
    dst = RM.Batch(regs[1], Ls, 16)
    m = np.full(len(pool) + 2, A.SLOT_NONE, np.uint32)
    for s, k in regs[0].live.items():
        m[s] = next(t for t, j in regs[1].live.items() if j == k)
    return src, dst, m, len(pool)


@pytest.mark.parametrize("permuted", [False, True])
def test_transfer_model_with_a_slot_map(permuted):
    n_pool = len(story_pool(np.random.default_rng(5), 10, 20, 1, 2))
    order = list(range(n_pool))[::-1] if permuted else list(range(n_pool))
    s1, d1, _, _ = _rm_pair(list(range(n_pool)))
    s2, d2, m, _ = _rm_pair(order)
    runs = [7, 0, 11, 3]
    want = TR.transfer(s1, d1, 12, 0, runs)
    got = TR.transfer(s2, d2, 12, 0, runs, slot_map=m)
    for k in want:
        assert np.array_equal(np.asarray(want[k]), np.asarray(got[k])), k
    assert np.array_equal(s1.state, s2.state) and np.array_equal(s1.cur, s2.cur) and np.array_equal(d1.cur, d2.cur)
    assert np.array_equal(d1.state[:, 4:], d2.state[:, 4:])
    w1 = np.ascontiguousarray(d1.state[:4, 0:4]).view("<u4").ravel()
    w2 = np.ascontiguousarray(d2.state[:4, 0:4]).view("<u4").ravel()
    assert np.array_equal(w2, m[w1])
    assert (not np.array_equal(w1, w2)) == permuted
    for k in ("touched", "must", "uploaded", "prev_valid", "prev_runs"):
        assert getattr(d1, k) == getattr(d2, k), k


def test_transfer_model_slot_verdicts_and_map_entries():
    src, dst, m, n_pool = _rm_pair(list(range(6))[::-1])

    def slot(r):
        return int(np.ascontiguousarray(src.state[r, 0:4]).view("<u4")[0])
    r_other = next(r for r in range(12) if slot(r) != slot(0))
    um = m.copy()
    um[slot(r_other)] = A.SLOT_NONE
    with pytest.raises(RM.Refused) as e:
        TR.transfer(src, dst, 12, 0, [0, r_other], slot_map=um)
    assert (e.value.unfit, e.value.reason) == (1, A.UNFIT_SLOT_UNMAPPED)
    with pytest.raises(RM.Refused) as e:
        TR.transfer(src, dst, 12, 0, [r_other, 0], slot_map=m[:max(slot(0), slot(r_other))])
    assert e.value.reason == A.UNFIT_SLOT_PAST_MAP and e.value.unfit == (0 if slot(r_other) > slot(0) else 1)
    # an entry of a live source slot that no moved run uses, naming a dead destination slot: the whole call
    bad = m.copy()
    spare = next(s for s in src.reg.live if s not in (slot(0), slot(r_other)))
    bad[spare] = 40
    with pytest.raises(RM.Refused) as e:
        TR.transfer(src, dst, 12, 0, [0], slot_map=bad)
    assert e.value.unfit == A.EXTENT_NO_RUN and e.value.reason == A.UNFIT_NONE
    # the same entry once its source slot is dead is ignored; a moved run on a dead slot is unfit
    src.reg.drop(spare)
    assert TR.transfer(src, dst, 12, 0, [0], slot_map=bad)["dst_n_runs"] == 1
    src, dst, m, _ = _rm_pair(list(range(6))[::-1])
    src.reg.drop(slot(0))
    with pytest.raises(RM.Refused) as e:
        TR.transfer(src, dst, 12, 0, [r_other, 0], slot_map=m)
    assert (e.value.unfit, e.value.reason) == (1, A.UNFIT_SLOT_DEAD)
