"""Cases of the independent-rows tests (options={'independent_rows': True}), shared by
tests/test_independent_rows_cpu.py (premises, on the oracle) and tests/test_independent_rows_gpu.py (the kernel).

Every case runs under the exact schedule of tests/exact_schedule.py, so each row's solve is a chain of correctly rounded
operations and must equal the oracle's solve of that row alone bit for bit.  To make rows take different schedules, a case
draws its rows from a POOL: the problem's usual cluster of initial states and copies of it scaled by 3, 10, 30 and 100
(a larger state needs more halvings of the step), plus the cluster scaled by 0 -- the origin, a fixed point of both systems,
where the error estimate is zero and no attempt is rejected.  A scaled row whose solve fails in the oracle (the first
step overflows the state) is left out of the pool.  A seeded random map tiles the pool over the batch; the oracle solves
each pool row once as a (1, dim) state, and every batch row must equal its pool entry.

This module is a plain helper (no fixtures); both test files import it.
"""
import numpy as np

import exact_schedule as es

SCALES = (1.0, 3.0, 10.0, 30.0, 100.0, 0.0)
CLUSTER = 3                    # rows of the problem's usual cluster in the pool
BATCHES = (1, 31, 33, 4099)    # rows of the batch; 1 000 003 more for dopri5 (BIG)
BIG = 1000003

CASES = [es._case(pr, me, dt, rev, "rows") for pr in ("lorenz", "lv") for me in es.METHODS for dt in es.DTYPES
         for rev in (False, True)]
# first_step=None: the initial-step heuristic per row
INITIAL = [es._case("lorenz", me, dt, False, "rows", first_step=None) for me in ("dopri5", "dopri8") for dt in es.DTYPES]
ALL = {c.name: c for c in CASES + INITIAL}


def candidates(case):
    """The cluster scaled by each of SCALES in turn (in the state dtype).  Not the origin with first_step=None: there the
    initial-step heuristic picks 1e-6, a million steps over the horizon."""
    base = es.initial_state(case._replace(outlier=None), CLUSTER)
    scales = SCALES if case.first_step is not None else [s for s in SCALES if s]
    return np.concatenate([base * base.dtype.type(s) for s in scales]).astype(case.dtype)


def tile(n_pool, n, seed=3):
    """Pool index of every batch row: a seeded random map that uses every pool entry when n allows it."""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, n_pool, n)
    if n >= n_pool:
        idx[rng.permutation(n)[:n_pool]] = np.arange(n_pool)
    return idx


_POOLS = {}


def pool_solves(case):
    """(pool, solves): the candidate rows whose solve alone, as a (1, dim) state, completes in the oracle, and those
    exact_schedule.Solve records (cached per case: both the premises and the kernel tests use them)."""
    if case.name not in _POOLS:
        opts = dict(es.OPTIONS)
        if case.first_step is not None:
            opts["first_step"] = case.first_step
        f = es.numpy_rhs(case)
        rows, solves = [], []
        with np.errstate(all="ignore"):
            for y in candidates(case):
                try:
                    s = es.oracle_solve(f, y[None], case.t, case.method, case.rtol, case.atol, opts)
                except AssertionError:
                    continue
                rows.append(y)
                solves.append(s)
        _POOLS.clear()
        _POOLS[case.name] = (np.stack(rows), solves)
    return _POOLS[case.name]
