"""The packed-lanes walk reads each dependency's status from per-run 32-bit status words (frontier_pack.cu, stage C): U and FD
interleaved by half word, pairs at st0 + g * 16 Wq + 8 w, PAD entries of u16 rows reading lane W of the run or the zero pair
behind it, and the in-place byte-entry path at Wq = 8.  These cases aim one-dependency probe batches (tests/depprobe.py) at
every row format, every Wq, runs narrower than Wq, the cond-FAIL fix-up and the other kernel and entry paths, so that a
misaddressed or mis-shifted status read flips about half the verdicts that rest on it.  Every case compares whole result
records and counts with the packed oracle and checks the kernel and runs per trip that really ran."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import Frontier
from oracle import packed as PK
from tests import depprobe as DP
from tests.test_gpu_shapes import KNOBS, _assert_pack, _pack_plan

pytestmark = pytest.mark.gpu

FORMATS = {   # name: the row formats of the batch's topologies (several: groups of mixed formats)
    "byte2": ["byte2"], "byte4": ["byte4"], "u16-2": ["u16-2"], "u16-4": ["u16-4"], "csr4": ["csr4"], "csrL": ["csrL"],
    "mixed": ["byte2", "byte4", "csrL"], "mixed-u16": ["u16-2", "u16-4", "csrL"],
}
# (any failed-dependency class, F_COND): the four builds <CD, XO> = 00, 01, 10, 11
MODES = [(False, False), (True, False), (False, True), (True, True)]


def _fields(any_fd, cond):
    return (A.F_ALL_OUT if any_fd else 0) | (A.F_COND if cond else 0)


@pytest.fixture(scope="module")
def sms():
    f = Frontier(0)
    try:
        return f.stats()["sm_count"]
    finally:
        f.close()


def _fresh(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("BF_E2E_CHUNKS", "1")
    for k, v in env.items():
        if v is not None:
            monkeypatch.setenv(k, str(v))
    return Frontier(0)


def _topologies(rng, f, kinds, wq, count=24, w_choices=None):
    forced = DP.forced_format(kinds)
    ws = w_choices or list(range(1, wq + 1))
    ws = [w for w in ws if any(w in DP.widths(k, wq, forced) for k in kinds)]
    pt = DP.probe_topologies(rng, kinds, ws, forced, count=count)
    slots = f.put_topologies(pt.ts)
    return pt, slots


def _want(pt, slots, ps):
    return PK.evaluate(PK.PackedTopologies(pt.ts, slots), ps.L, ps.state, threads=16)


def _check(f, pt, slots, ps, kernel=1, R=None):
    want, wc = _want(pt, slots, ps)
    got, gc = f.eval(ps.L, ps.state, flags=A.EVAL_VALIDATE)
    st = f.stats()
    assert st["last_kernel"] == kernel, st
    if R is not None:
        assert st["last_runs_per_trip"] == R, st
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, (bad.size, len(got), bad[:10], [pt.kinds[int(ps.topo[r])] for r in bad[:10]])
    assert gc == wc, (gc, wc)


def _matrix():
    out = []
    for name, kinds in FORMATS.items():
        for wq in (1, 2, 4, 8, 16):
            forced = DP.forced_format(kinds)
            if all(DP.widths(k, wq, forced) for k in kinds):
                out.append((name, wq))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# row format x Wq (layout width 32 Wq over topologies of 1 .. Wq words), any-FD and F_COND on / off
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,wq", _matrix())
def test_status_words_row_format_by_wq(monkeypatch, name, wq):
    kinds = FORMATS[name]
    f = _fresh(monkeypatch, {"BF_TOPO_FORMAT": DP.forced_format(kinds)})
    try:
        rng = np.random.default_rng(8000 + 16 * list(FORMATS).index(name) + wq)
        pt, slots = _topologies(rng, f, kinds, wq)
        for any_fd, cond in MODES:
            ps = DP.probe_state(rng, pt, slots, 6007, wq, _fields(any_fd, cond), any_fd=any_fd)
            _check(f, pt, slots, ps, R=32 // wq)
    finally:
        f.close()


@pytest.mark.parametrize("name,wq,force", [("byte4", 4, 16), ("u16-4", 4, 32), ("mixed", 8, 16), ("csrL", 2, 32),
                                           ("u16-2", 16, 32), ("mixed-u16", 2, 16)])
def test_status_words_forced_wq(monkeypatch, name, wq, force):
    """BF_WQ = 16 / 32 (R = 2 / 1) over layouts narrower than that: every run is narrower than Wq"""
    kinds = FORMATS[name]
    f = _fresh(monkeypatch, {"BF_TOPO_FORMAT": DP.forced_format(kinds), "BF_WQ": force})
    try:
        rng = np.random.default_rng(8200 + force + wq + list(FORMATS).index(name))
        pt, slots = _topologies(rng, f, kinds, wq)
        for any_fd, cond in MODES:
            ps = DP.probe_state(rng, pt, slots, 4001, wq, _fields(any_fd, cond), any_fd=any_fd)
            _check(f, pt, slots, ps, R=32 // force)
    finally:
        f.close()


# ---------------------------------------------------------------------------------------------------------------------
# the in-place byte-entry walk (uniform byte4 groups at Wq = 8, probes at d >= 128) and the generic one at Wq = 16
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("force", [None, 16])
def test_status_words_byte4_in_place_and_generic(monkeypatch, force):
    f = _fresh(monkeypatch, {"BF_WQ": force})
    try:
        rng = np.random.default_rng(8300)   # the same topologies and batches for both walks
        pt, slots = _topologies(rng, f, ["byte4"], 8, w_choices=[5, 6, 7, 8])
        assert all(k == "byte4" for k in pt.kinds) and int(pt.W.min()) >= 5
        for any_fd, cond in MODES:
            ps = DP.probe_state(rng, pt, slots, 8009, 8, _fields(any_fd, cond), any_fd=any_fd)
            _check(f, pt, slots, ps, R=4 if force is None else 2)
    finally:
        f.close()


# ---------------------------------------------------------------------------------------------------------------------
# narrow runs: u16 PAD entries reading lane W of the run (W < Wq) or the zero pair (W = Wq), in groups of mixed widths,
# over batches long enough that every slot group and every warp's status scratch is reused many times
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wq,fields", [(2, A.F_ALL_OUT), (4, A.F_COND | A.F_ALL_OUT), (16, A.F_COND)])
def test_status_words_narrow_u16_runs(monkeypatch, sms, wq, fields):
    f = _fresh(monkeypatch, {"BF_TOPO_FORMAT": "ell16"})
    try:
        rng = np.random.default_rng(8400 + wq)
        pt, slots = _topologies(rng, f, ["u16-2", "u16-4"], wq, count=32)
        assert (pt.W < wq).any() and (pt.W == wq).any()
        L = DP.probe_state(rng, pt, slots, 1, wq, fields).L
        R, nw, ng, smem = _pack_plan(f, L, slots)
        n = 4 * R * ng * sms + R - 1
        ps = DP.probe_state(rng, pt, slots, n, wq, fields, any_fd=True)
        _check(f, pt, slots, ps, R=R)
        _assert_pack(f.stats(), R, nw, ng, sms, smem)
    finally:
        f.close()


# ---------------------------------------------------------------------------------------------------------------------
# the other kernel and entry paths over probe batches
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,wq", [("mixed", 4), ("u16-4", 2), ("byte4", 8), ("csrL", 16)])
def test_status_words_general_kernel(monkeypatch, name, wq):
    """the one-run-per-warp kernel walks status bytes; its cond-FAIL fix-up reads them through its own status reader"""
    kinds = FORMATS[name]
    f = _fresh(monkeypatch, {"BF_TOPO_FORMAT": DP.forced_format(kinds), "BF_KERNEL": "general"})
    try:
        rng = np.random.default_rng(8500 + wq)
        pt, slots = _topologies(rng, f, kinds, wq)
        for any_fd, cond in MODES:
            ps = DP.probe_state(rng, pt, slots, 3001, wq, _fields(any_fd, cond), any_fd=any_fd)
            _check(f, pt, slots, ps, kernel=0)
    finally:
        f.close()


@pytest.mark.parametrize("chunks", [1, 5])
def test_status_words_chunked_eval(monkeypatch, chunks):
    f = _fresh(monkeypatch, {})
    monkeypatch.setenv("BF_E2E_CHUNKS", str(chunks))
    try:
        rng = np.random.default_rng(8600 + chunks)
        pt, slots = _topologies(rng, f, FORMATS["mixed"], 8)
        ps = DP.probe_state(rng, pt, slots, 20011, 8, A.F_COND | A.F_ALL_OUT)
        _check(f, pt, slots, ps, R=4)
        assert f.stats()["last_eval_chunks"] == chunks
    finally:
        f.close()


def test_status_words_pipelined_device_passes_and_resident_tick(monkeypatch):
    """two probe batches of other widths and formats back to back as pipelined device passes (EVAL_PIPELINED |
    EVAL_COUNTS_SET), then a resident tick over the first batch's records"""
    import torch
    f = _fresh(monkeypatch, {"BF_TOPO_FORMAT": "ell16"})
    try:
        rng = np.random.default_rng(8700)
        sets = []
        for kinds, wq, fields in ((["u16-2", "u16-4", "csrL"], 4, A.F_COND | A.F_ALL_OUT), (["u16-4", "csrL"], 16, A.F_ALL_OUT)):
            pt, slots = _topologies(rng, f, kinds, wq)
            ps = DP.probe_state(rng, pt, slots, 30011, wq, fields)
            want, wc = _want(pt, slots, ps)
            sets.append((ps, want, wc))
        dev = torch.device("cuda", 0)
        bufs = [(torch.from_numpy(ps.state).to(dev), torch.zeros((len(ps.state), ps.L.result_stride), dtype=torch.uint8, device=dev),
                 torch.zeros(4, dtype=torch.int64, device=dev)) for ps, _, _ in sets]
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for _ in range(2):
                for (ps, _, _), (d_state, d_result, d_counts) in zip(sets, bufs):
                    f.eval_device(ps.L, len(ps.state), d_state.data_ptr(), d_result.data_ptr(), d_counts.data_ptr(), s.cuda_stream,
                                  flags=A.EVAL_COUNTS_SET | A.EVAL_PIPELINED)
        torch.cuda.synchronize()
        assert f.stats()["last_kernel"] == 1, f.stats()
        for (ps, want, wc), (_, d_result, d_counts) in zip(sets, bufs):
            got = d_result.cpu().numpy()
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, (bad.size, bad[:10])
            assert d_counts.cpu().numpy().tolist() == [wc["ready"], wc["skip"], wc["expansion"], wc["evals"]]
        ps, want, wc = sets[0]
        n = len(ps.state)
        h = f.resident_create(ps.L, n)
        try:
            f.resident_upload(h, 0, ps.state)
            got, gc = f.resident_tick(h, ps.L, n, np.zeros(0, dtype=Frontier.DELTA_DTYPE))
            assert f.stats()["last_kernel"] == 1 and f.stats()["last_runs_per_trip"] == 8, f.stats()
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0 and gc == wc, (bad.size, bad[:10], gc, wc)
        finally:
            f.resident_destroy(h)
    finally:
        f.close()
