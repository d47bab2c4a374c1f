"""The one-dependency probe generator (tests/depprobe.py), checked without a GPU: each probe topology gets the row format it is
meant for in the device record, and flipping one probe target's status changes the verdicts of that target's readers, and
of nothing else, in most runs.  A probe batch that no misread could flip would pass its GPU comparisons quietly."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200.records import pack_state, unpack_result
from oracle import packed as PK
from tests import depprobe as DP
from tests.test_record_formats import HDR, _build

SETS = {   # name: (kinds, topology widths)
    "byte2": (["byte2"], [1, 2, 3, 4, 5, 6, 7, 8]),
    "byte4": (["byte4"], [1, 2, 3, 4, 5, 6, 7, 8]),
    "u16-2": (["u16-2"], [1, 2, 3, 4, 7, 9, 16]),
    "u16-4": (["u16-4"], [1, 2, 3, 4, 7, 9, 16]),
    "csr4": (["csr4"], [1, 2, 4, 8, 16]),
    "csrL": (["csrL"], [1, 2, 4, 8, 16]),
    "mixed": (["byte2", "byte4", "csrL"], [1, 2, 4, 8]),
    "mixed-u16": (["u16-2", "u16-4", "csrL"], [1, 2, 4, 7]),
}


def _record_kind(rec):
    S, W, max_deg, P, n_main, n_comp, n_final, child_nib, off_col, ell, off_planes, off_par, rec_bytes = \
        HDR.unpack_from(rec.tobytes(), 0)
    if ell == 0:
        return "csr4" if max_deg <= 4 else "csrL"
    if ell & 0x200:
        return "p10"
    return ("byte%d" if ell & 0x100 else "u16-%d") % (ell & 0xFF)


@pytest.mark.parametrize("name", list(SETS))
def test_probe_topologies_get_their_row_format(monkeypatch, name):
    kinds, ws = SETS[name]
    forced = DP.forced_format(kinds)
    if forced:
        monkeypatch.setenv("BF_TOPO_FORMAT", forced)
    else:
        monkeypatch.delenv("BF_TOPO_FORMAT", raising=False)
    rng = np.random.default_rng(7000 + list(SETS).index(name))
    pt = DP.probe_topologies(rng, kinds, ws, forced, count=3 * len(ws))
    got = [_record_kind(_build(pt.ts, t)) for t in range(pt.ts.count)]
    assert got == pt.kinds, list(zip(got, pt.kinds, pt.ts.S))
    assert set(int(w) for w in pt.W) >= set(ws) - ({8} if kinds[0].startswith("u16") else set())
    # the probe positions the walk's edge cases need, each read from below and from above
    d, i = [], []
    for t in range(pt.ts.count):
        rd = np.nonzero(pt.roles[t] == DP.READER)[0]
        d.append(pt.probes[t][rd])
        i.append(rd)
    d, i = np.concatenate(d), np.concatenate(i)
    for lo in (0, 15, 16, 31):
        at = (d & 31) == lo
        assert at.sum() >= 10 and (at & (d < i)).any() and (at & (d > i)).any(), lo
    for x in (127, 128, 255):
        if x < int(pt.ts.S.max()):
            assert ((d == x) & (d > i)).any() and (x == 255 or ((d == x) & (d < i)).any()), x   # 255: the last step


def _verdicts(L, res, S):
    u = unpack_result(L, res, S)
    return sum(u[k].astype(np.uint8) << b for b, k in enumerate(("ready", "skip", "fail", "needs_cond", "skip_dep")))


def _flip(pt, ps, slots, runs, t_of, a, b, cond_a=None, cond_b=None):
    """evaluate the batch twice with target t_of[r] of each run r in `runs` at phase a / b (cond cond_a / cond_b); -> the
    [n, width] mask of steps whose verdict changed"""
    L = ps.L
    width = 32 * L.words
    out = []
    for ph_v, c_v in ((a, cond_a), (b, cond_b)):
        phase, cond = ps.phase.copy(), ps.cond.copy()
        phase[runs, t_of[runs]] = ph_v[runs] if isinstance(ph_v, np.ndarray) else ph_v
        if c_v is not None:
            cond[runs, t_of[runs]] = c_v
        st = pack_state(L, np.asarray(slots)[ps.topo], ps.rflags, phase, cond if L.off_cond != A.OFF_NONE else None)
        res, _ = PK.evaluate(PK.PackedTopologies(pt.ts, slots), L, st, threads=8)
        out.append(_verdicts(L, res, width))
    return out[0] != out[1]


@pytest.mark.parametrize("fields", [A.F_ALL_OUT, A.F_COND | A.F_ALL_OUT])
@pytest.mark.parametrize("name", ["byte4", "u16-4", "csrL", "mixed"])
def test_one_status_read_decides_each_reader(monkeypatch, name, fields):
    kinds, ws = SETS[name]
    rng = np.random.default_rng(7100 + list(SETS).index(name) + fields)
    pt = DP.probe_topologies(rng, kinds, ws, DP.forced_format(kinds), count=12)
    slots = np.arange(pt.ts.count, dtype=np.uint32)
    words = max(ws)
    n = 3000
    ps = DP.probe_state(rng, pt, slots, n, words, fields, any_fd=True)
    width = 32 * words
    # one target per run, and the readers of that target (role planes padded to the layout width)
    t_of = np.zeros(n, np.int64)
    readers = np.zeros((n, width), bool)
    after = np.zeros((n, width), bool)
    nonaf = np.zeros(n, bool)
    for r in range(n):
        t = int(ps.topo[r])
        tg = np.nonzero(pt.roles[t] == DP.TARGET)[0]
        t_of[r] = int(rng.choice(tg))
        rd = pt.probes[t] == t_of[r]
        readers[r, :rd.size] = rd
        after[r, :rd.size] = rd & (np.arange(rd.size) > t_of[r])
        nonaf[r] = not pt.af[t][t_of[r]]
    own = np.zeros((n, width), bool)
    own[np.arange(n), t_of] = True
    allowed = readers | own
    rt = (ps.rflags & A.RF_REALTIME) != 0
    sof = (ps.rflags & A.RF_FAIL_FAST) == 0
    all_runs = np.arange(n)

    # satisfied vs not: Succeeded against Running (realtime runs: Blocked, Running is satisfied for them)
    changed = _flip(pt, ps, slots, all_runs, t_of, 3, np.where(rt, 9, 2).astype(np.uint8))
    assert not (changed & ~allowed).any(), np.argwhere(changed & ~allowed)[:5]
    frac = (changed & readers).sum() / readers.sum()
    assert frac >= 0.8, frac

    # failed vs not, in skip-on-failed runs on targets without allowFailure
    runs = np.nonzero(sof & nonaf)[0]
    changed = _flip(pt, ps, slots, runs, t_of, 4, 2)
    assert not (changed & ~allowed).any()
    assert not changed[~np.isin(all_runs, runs)].any()
    frac = (changed[runs] & readers[runs]).sum() / readers[runs].sum()
    assert frac >= 0.8, frac

    if fields & A.F_COND:
        # the fix-up probe: a pending target failed by its cond inside the pass is a failed dependency of the readers after
        # it only; readers before it still see it pending
        runs = np.nonzero(sof)[0]
        changed = _flip(pt, ps, slots, runs, t_of, 0, 0, A.COND_FAIL, A.COND_PASS)
        assert not (changed & ~(after | own)).any()
        frac = (changed[runs] & after[runs]).sum() / after[runs].sum()
        assert frac >= 0.8, frac
