"""Rejected deltas across every call that scatters them.  A call whose deltas include some outside the record (a run at or
past the capacity, an index past the layout width, a field the layout does not have, the reserved phase code 15) applies the
others, runs its pass, and fails with BF_EINVAL naming how many it rejected.  Each test runs one ordered pair of call kinds
(K1, K2) on a batch and on a twin batch in a ctx of its own that receives only the valid deltas: K1 must fail with the exact
count and leave the twin's records; K2, with valid deltas only, must succeed with the twin's outputs, so a rejected-delta
counter that K1 left behind shows up there."""
import re

import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from bobrapet_b200.records import make_layout
from tests import randgen

pytestmark = pytest.mark.gpu

ALL = A.F_COND | A.F_DECISION | A.F_ALL_OUT   # no child area: DELTA_CHILD is a field the layout does not have
NONE = np.zeros(0, dtype=Frontier.DELTA_DTYPE)
BIG = 4_000_000
# the touched kinds: incremental, full (a dropped slot forces it), and each at n_runs = 0 (incremental: no launch beyond the
# scatter; full: a compact tick without runs)
KINDS = ["apply", "tick", "tick_chunked", "compact", "compact_changed", "touched", "touched_full", "touched_empty",
         "touched_full_empty", "compact_empty"]
PINNED_KIND = "compact"   # K1's deltas also come from pinned memory (read by the scatter kernel over PCIe)


def _setup():
    """topologies, layout, records and capacity shared by every pair: the results of all runs take at least 2 MB, so the
    dense tick may be cut into chunks"""
    rng = np.random.default_rng(5150)
    ts = randgen.random_topologies(rng, 30, 30, 256, parallel=False)
    spare = randgen.random_topologies(rng, 1, 10, 20, parallel=False)
    slots = np.arange(ts.count, dtype=np.uint32)   # what a fresh ctx returns for the first put (checked below)
    n = (2 << 20) // make_layout(int(ts.S.max()), 0, ALL).result_stride + 100
    L, state, _ = randgen.random_state(rng, ts, slots, n, ALL, phase_mix="progress")
    assert L.off_child == A.OFF_NONE and n * L.result_stride >= (2 << 20)
    return ts, spare, slots, L, state, n + 16


SETUP = None


def _valid(rng, L, n):
    """valid deltas, at most one per (run, field, index), over the fields the layout has"""
    W32 = 32 * L.words
    recs = {}
    for r in rng.integers(0, n, size=300):
        f = int(rng.choice([A.DELTA_PHASE] * 4 + [A.DELTA_COND, A.DELTA_DECISION, A.DELTA_RUN_FLAGS, A.DELTA_REGISTERED]))
        if f == A.DELTA_PHASE:
            idx, code = int(rng.integers(0, W32)), int(rng.choice([0, 1, 2, 3, 4, 9, 13, 14]))
        elif f in (A.DELTA_COND, A.DELTA_DECISION):
            idx, code = int(rng.integers(0, W32)), int(rng.integers(0, 4))
        elif f == A.DELTA_RUN_FLAGS:
            idx, code = 0, int(rng.choice([0, A.RF_FAIL_FAST, A.RF_TOPOLOGY_TERMINATED]))
        else:
            idx, code = int(rng.integers(0, 64)), int(rng.integers(0, 2))
        recs[(int(r), f, idx)] = code
    d = np.zeros(len(recs), dtype=Frontier.DELTA_DTYPE)
    for i, ((r, f, idx), code) in enumerate(recs.items()):
        d[i] = (r, idx, f, code)
    return d


def _bad(rng, L, cap, valid):
    """1-3 deltas of distinct kinds outside the record.  Those on a live run go to runs the valid deltas touch, so both
    batches end with the same touch marks (the scatter raises a run's mark before it checks the delta)."""
    W32 = 32 * L.words
    runs = np.unique(valid["run"])
    taken = {(int(d["run"]), int(d["field"]), int(d["index"])) for d in valid}
    out = []
    for kind in rng.choice(4, size=int(rng.integers(1, 4)), replace=False):
        r = int(rng.choice(runs))
        if kind == 0:
            out.append((cap + int(rng.integers(0, 1000)), 0, A.DELTA_PHASE, 3))
        elif kind == 1:
            out.append((r, W32 + int(rng.integers(0, 64)), A.DELTA_PHASE, 3))
        elif kind == 2:
            out.append((r, int(rng.integers(0, W32)), A.DELTA_CHILD, 2))
        else:
            idx = next(i for i in range(W32) if (r, A.DELTA_PHASE, i) not in taken)
            out.append((r, idx, A.DELTA_PHASE, 15))
    return np.array(out, dtype=Frontier.DELTA_DTYPE)


class Side:
    """one ctx and one resident batch of the shared records"""

    def __init__(self):
        ts, self.spare, slots, self.L, state, self.cap = SETUP
        self.n = state.shape[0]
        self.fr = Frontier(0)
        assert np.array_equal(self.fr.put_topologies(ts), slots)
        self.h = self.fr.resident_create(self.L, self.cap)
        self.fr.resident_upload(self.h, 0, state)
        self.fr.resident_tick_compact(self.h, self.n, NONE, BIG)   # the last full tick covers every run

    def close(self):
        self.fr.close()

    def records(self):
        return self.fr.resident_download(self.h, 0, self.cap, self.L.state_stride)

    def prepare(self, kind):
        """what the kind needs before its call (the same on both sides, without deltas)"""
        if kind in ("touched", "touched_empty"):    # a full tick with the touched ticks' parameters: the next one is incremental
            self.fr.resident_tick_compact(self.h, self.n, NONE, BIG)
        elif kind in ("touched_full", "touched_full_empty"):   # a slot drop: the next touched tick evaluates every run
            self.fr.drop_topology(self.fr.put_topologies(self.spare)[0])

    def call(self, kind, d, monkeypatch):
        """K's call with deltas d -> its outputs"""
        fr, h, n = self.fr, self.h, self.n
        if kind == "apply":
            fr.resident_apply(h, d)
            return ()
        if kind in ("tick", "tick_chunked"):
            with monkeypatch.context() as m:
                m.setenv("BF_E2E_CHUNKS", "4" if kind == "tick_chunked" else "1")
                got, counts = fr.resident_tick(h, self.L, n, d)
            assert fr.stats()["last_eval_chunks"] == (4 if kind == "tick_chunked" else 1)
            return got, counts
        if kind in ("compact", "compact_changed", "compact_empty"):
            return fr.resident_tick_compact(h, 0 if kind == "compact_empty" else n, d, BIG,
                                            flags=A.EVAL_CHANGED_ONLY if kind == "compact_changed" else 0)
        out = fr.resident_tick_touched(h, 0 if kind.endswith("_empty") else n, d, n, BIG)
        assert out["full"] == (1 if kind.startswith("touched_full") else 0), (kind, out["full"])
        return out


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    return a == b


@pytest.mark.parametrize("k1,k2,pinned", [(a, b, False) for a in KINDS for b in KINDS] + [(PINNED_KIND, b, True) for b in KINDS])
def test_rejected_deltas_reported(k1, k2, pinned, monkeypatch):
    global SETUP
    if SETUP is None:
        SETUP = _setup()
    rng = np.random.default_rng([KINDS.index(k1), KINDS.index(k2), int(pinned)])
    T, W = Side(), Side()   # the batch under test, and its twin that receives only the valid deltas
    buf = None
    try:
        valid = _valid(rng, T.L, T.n)
        bad = _bad(rng, T.L, T.cap, valid)
        mixed = np.concatenate([valid, bad])[rng.permutation(len(valid) + len(bad))]
        if pinned:
            buf = T.fr.alloc_pinned(mixed.nbytes)
            buf[:] = mixed.view(np.uint8)
            mixed = buf.view(Frontier.DELTA_DTYPE)
        for side in (T, W):
            side.prepare(k1)
        with pytest.raises(A.FrontierError) as e:
            T.call(k1, mixed, monkeypatch)
        assert e.value.status == A.BF_EINVAL
        m = re.search(r"\(-?\d+\): bf_\w+: (\d+) delta\(s\) outside the record", str(e.value))
        assert m and int(m.group(1)) == len(bad), str(e.value)
        W.call(k1, valid, monkeypatch)
        assert np.array_equal(T.records(), W.records()), "K1 = %s: the records differ from the twin's" % k1

        valid2 = _valid(rng, T.L, T.n)
        for side in (T, W):
            side.prepare(k2)
        got, want = T.call(k2, valid2, monkeypatch), W.call(k2, valid2, monkeypatch)
        assert _same(got, want), "K2 = %s after K1 = %s: the outputs differ from the twin's" % (k2, k1)
        assert np.array_equal(T.records(), W.records()), "K2 = %s after K1 = %s: the records differ from the twin's" % (k2, k1)
    finally:
        if buf is not None:
            T.fr.free_pinned(buf)
        T.close()
        W.close()
