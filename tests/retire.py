"""The move rule of a retirement (bf_resident_retire, bfh_batch_retire) and the records it leaves, restated in numpy."""
import numpy as np


def moves(n_runs, runs):
    """-> (m, moves_from, moves_to): with m = n_runs - len(runs), the retired indices below m (ascending) receive the live indices
    of [m, n_runs) (ascending), one each"""
    gone = np.zeros(n_runs, bool)
    gone[np.asarray(runs, np.int64)] = True
    m = n_runs - int(gone.sum())
    holes = np.flatnonzero(gone[:m])
    sources = m + np.flatnonzero(~gone[m:])
    assert holes.shape == sources.shape
    return m, sources.astype(np.uint32), holes.astype(np.uint32)


def order(n_runs, runs):
    """old index of the run at each new index of [0, m)"""
    m, src, dst = moves(n_runs, runs)
    out = np.arange(m, dtype=np.int64)
    out[dst] = src
    return out


def new_index(n_runs, runs):
    """new index of every old run of [0, n_runs), -1 for a retired one"""
    out = np.full(n_runs, -1, np.int64)
    out[order(n_runs, runs)] = np.arange(n_runs - len(runs))
    return out


def retire_records(records, n_runs, runs, capacity):
    """state records [cap, stride] -> what the batch holds afterwards over [0, capacity): each target the source's record, [m,
    n_runs) zero, every other record (those at or above n_runs included) as it was"""
    m, src, dst = moves(n_runs, runs)
    out = records.copy()
    out[dst] = records[src]
    out[m:n_runs] = 0
    return out[:capacity]
