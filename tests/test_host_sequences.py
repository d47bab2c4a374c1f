"""The C++ host mirror (HostBatch without a device) driven through random sequences of add_run, the set_* calls, migrate, redrive,
reshape, retire, narrow and transfer; after every call its records equal those of the host model in tests/resident_model.py
(narrow: tests/narrowing.py, transfer: tests/transfer.py).  CPU only."""
import numpy as np
import pytest

from bobrapet_b200 import _abi as A
from bobrapet_b200 import host as H
from bobrapet_b200.records import make_layout
from tests import migration as M
from tests import redrive as RD
from tests import resident_model as RM
from tests import transfer as TR
from tests.narrowing import NarrowBatch

FIELDS = A.F_COND | A.F_DECISION | A.F_CHILD | A.F_ALL_OUT
BIG = 4096


def _host_story(steps):
    hs = H.HostStory()
    for s in steps:
        hs.add_step(s["name"], s["group"], s["type"], if_expr=s.get("if"), needs=s["needs"],
                    branches=[("%s-b%d" % (s["name"], b), False) for b in range(s["branches"])])
    assert hs.finalize() == 0, hs.error()
    return hs


@pytest.mark.parametrize("seed", range(8))
def test_host_mirror_follows_the_model(seed):
    rng = np.random.default_rng(300 + seed)
    base = [RD.random_story(rng, "h%d-" % k, int(rng.integers(20, 60)), 2) for k in range(3)]
    steps = base + [M.edit_story(rng, s, "h%d-e" % k) for k, s in enumerate(base)]
    pool = [RD.packed_story(s) for s in steps]
    hss = [_host_story(s) for s in steps]
    reg = RM.Registry(pool)
    slots = [reg.put(k) for k in range(len(pool))]
    child = max(p.child_nibbles() for p in pool)
    S = max(p.S for p in pool)
    cap = 64   # until the first reshape
    hb = H.HostBatch(None, S, child, FIELDS, cap)
    b = NarrowBatch(reg, A.Layout.from_buffer_copy(hb.L), BIG)   # (hb.L follows the mirror's reshapes)
    # the destination of transfers: the runs of the Stories up to the median width fit it, the others are refused
    S_fit = sorted(p.S for p in pool)[len(pool) // 2]
    hd = H.HostBatch(None, S_fit, child + 8, FIELDS, BIG)
    bd = RM.Batch(reg, A.Layout.from_buffer_copy(hd.L), BIG)
    story_of = []
    log = []

    def check():
        n = hb.size()
        assert np.array_equal(hb.state(), b.state[:n]), "seed %d op %d\n  %s" % (seed, len(log) - 1, "\n  ".join(log))

    try:
        for _ in range(int(rng.integers(60, 101))):
            n = hb.size()
            op = rng.choice(["add", "set", "set", "set", "migrate", "redrive", "reshape", "retire", "narrow", "transfer"])
            if op == "add" or n == 0:
                k = int(rng.integers(0, 3))
                for _ in range(min(int(rng.integers(1, 30)), cap - n)):
                    r = hb.add_run(hss[k], slots[k])
                    b.upload(r, hb.state()[r:r + 1].copy())   # the record add_run packs (the mirror's own packing is tested elsewhere)
                    story_of.append(k)
                log.append("add runs -> %d" % hb.size())
            elif op == "set":
                for _ in range(int(rng.integers(1, 40))):
                    r = int(rng.integers(0, n))
                    ps = pool[story_of[r]]
                    i = int(rng.integers(0, ps.S))
                    W = b.L.words
                    what = int(rng.integers(0, 5))
                    if {1: b.L.off_cond, 2: b.L.off_decision, 4: b.L.off_child}.get(what) == A.OFF_NONE:
                        continue   # a narrow dropped the field
                    if what == 0:
                        code = int(rng.integers(0, 15))
                        hb.set_phase_code(r, i, code)
                        RM._set_plane(b.state[r], b.L.off_phase, W, 4, i, code)
                    elif what == 1:
                        code = int(rng.integers(0, 4))
                        hb.set_cond(r, i, code)
                        RM._set_plane(b.state[r], b.L.off_cond, W, 2, i, code)
                    elif what == 2:
                        code = int(rng.integers(0, 4))
                        hb.set_decision(r, i, code)
                        RM._set_plane(b.state[r], b.L.off_decision, W, 2, i, code)
                    elif ps.par_steps:
                        q = int(rng.integers(0, len(ps.par_steps)))
                        if what == 3:
                            on = int(rng.integers(0, 2))
                            hb.register_children(r, q, bool(on))
                            v = b.state[r, 8:16].view("<u8")
                            v[0] = (int(v[0]) & ~(1 << q)) | (on << q)
                        else:
                            br = int(rng.integers(0, len(ps.par_branches[q])))
                            code = int(rng.choice([0, 2, 3, 4, 13]))
                            hb.set_child_phase(r, q, br, A.PHASE_NAMES[code])
                            RM._nibble(b.state[r], b.L.off_child, int(ps.child_first()[q]) + br, code)
                log.append("set codes")
            elif op == "migrate":
                k = int(rng.integers(0, 3))
                got = hb.migrate(hss[k], hss[k + 3], slots[k], slots[k + 3])
                want = b.migrate(slots[k], slots[k + 3], M.migration_map(pool[k], pool[k + 3])[0], n)
                story_of = [k + 3 if s == k else s for s in story_of]
                log.append("migrate %d -> %d: %d runs" % (k, k + 3, want))
                assert got == want, log
            elif op == "redrive":
                runs = rng.integers(0, n, size=int(rng.integers(1, 12)))
                st = np.array([-1 if rng.random() < 0.3 else int(rng.integers(0, pool[story_of[r]].S)) for r in runs], np.int32)
                hb.redrive(runs, st)
                req = np.zeros(len(runs), dtype=np.dtype([("run", "<u4"), ("slot", "<u4"), ("step", "<u4"), ("reserved", "<u4")]))
                req["run"], req["slot"] = runs, b.slots(BIG)[runs]
                req["step"] = np.where(st < 0, A.REDRIVE_ALL, st)
                b.redrive(req)
                log.append("redrive %d requests" % len(runs))
            elif op == "reshape":
                L = b.L
                T = make_layout(L.steps_max + int(rng.choice([0, 32])), L.child_nibbles + int(rng.choice([0, 8])), L.fields)
                hb.reshape(T.steps_max, T.child_nibbles, T.fields, BIG)
                b.reshape(T, BIG)
                cap = BIG
                log.append("reshape to S %d child %d" % (T.steps_max, T.child_nibbles))
            elif op == "narrow":
                # never below the widest Story of the pool, which a later migrate or redrive needs
                L = b.L
                T = make_layout(max(S, L.steps_max - int(rng.choice([0, 32, 64]))),
                                max(child, L.child_nibbles - int(rng.choice([0, 8]))),
                                L.fields & ~int(rng.choice([0, 0, A.F_DECISION, A.F_COND, A.F_CHILD, A.F_OUT_FAIL])))
                got = want = A.BF_OK
                try:
                    hb.narrow(T.steps_max, T.child_nibbles, T.fields)
                except A.FrontierError as e:
                    got = e.status
                try:
                    b.narrow(T, n)
                except RM.Refused as e:
                    want = e.status
                log.append("narrow to S %d child %d fields %#x: %d" % (T.steps_max, T.child_nibbles, T.fields, want))
                assert got == want, log
                assert bytes(hb.L) == bytes(b.L), log
            elif op == "transfer":
                fit = [r for r in range(n) if pool[story_of[r]].S <= S_fit]
                runs = rng.permutation(fit)[:int(rng.integers(0, min(len(fit), 20) + 1))].tolist()
                extra = int(rng.integers(0, n))   # half the time any run: refused unless its Story fits
                if rng.random() < 0.5 and extra not in runs:
                    runs.append(extra)
                D = hd.size()
                got = want = A.BF_OK
                try:
                    mf, mt = hb.transfer(hd, np.asarray(runs, np.uint32))
                except A.FrontierError as e:
                    got = e.status
                try:
                    w = TR.transfer(b, bd, n, D, runs)
                except RM.Refused as e:
                    want = e.status
                log.append("transfer %d of %d: %d" % (len(runs), n, want))
                assert got == want, log
                if want == A.BF_OK:
                    assert np.array_equal(mf, w["moves_from"]) and np.array_equal(mt, w["moves_to"]), log
                    assert (hb.size(), hd.size()) == (w["src_n_runs"], w["dst_n_runs"]), log
                    story_of = [story_of[i] for i in RM.RT.order(n, runs)]
                assert np.array_equal(hd.state(), bd.state[:hd.size()]), log
            else:
                runs = rng.choice(n, size=int(rng.integers(0, n // 2 + 1)), replace=False)
                mf, mt = hb.retire(runs)
                _, wf, wt = b.retire(n, runs)
                keep = RM.RT.order(n, runs)
                story_of = [story_of[i] for i in keep]
                log.append("retire %d of %d" % (len(runs), n))
                assert np.array_equal(mf, wf) and np.array_equal(mt, wt), log
            check()
    finally:
        hb.close()
        hd.close()
