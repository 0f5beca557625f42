"""Cases of the independent-rows adjoint tests (odeint_adjoint with options={'independent_rows': True, 'fused_vjp': True}),
shared by tests/test_rows_adjoint_cpu.py (premises, on the oracle) and tests/test_rows_adjoint_gpu.py (the kernel).

Every case is a case of tests/rows_cases.py: the same pools of initial rows (the problem's cluster scaled by 1, 3, 10, 30,
100 and 0), tiled over the batch by the same seeded map.  Each pool row carries its own loss weights, +-2**k with about one
entry in eight zero and no weight at all on the second output time (as exact_adjoint.loss_weights), and they are tiled with
it.  The oracle of a pool row is exact_adjoint.adjoint_oracle on the torch-CPU built-in module with the row as a (1, dim)
state, under the exact schedule (es.OPTIONS, first_step given, max_num_steps = exact_adjoint.MAX_NUM_STEPS): every batch
row's gradient must equal its pool row's bit for bit.  A pool row whose oracle adjoint fails, or one whose forward solve or
backward intervals take a decision within the margin of es.premises, is left out.

This module is a plain helper (no fixtures); both test files import it.
"""
import numpy as np
import torch

import exact_adjoint as xa
import exact_schedule as es
import rows_cases as rc

CASES = rc.CASES
INITIAL = rc.INITIAL
ALL = rc.ALL
BATCHES = rc.BATCHES
BIG = rc.BIG


def module(case):
    """The torch-CPU built-in right-hand side of a case."""
    import tfdiffeq_b200
    return tfdiffeq_b200.rhs.Lorenz() if case.problem == "lorenz" else tfdiffeq_b200.rhs.LotkaVolterra()


def options(case, first_step=True):
    opts = dict(es.OPTIONS, max_num_steps=xa.MAX_NUM_STEPS)
    if first_step and case.first_step is not None:
        opts["first_step"] = case.first_step
    return opts


def weights(case, n_pool, dim, seed=0):
    """(n_pool, T, dim) loss weights, one set per pool row."""
    rng = np.random.default_rng(seed + 2000)
    T = len(case.t)
    w = xa._pow2(rng, (n_pool, T, dim), -3, 1) * (rng.random((n_pool, T, dim)) >= 0.125)
    w[:, 1] = 0.0
    return w.astype(case.dtype)


_POOLS = {}


def pool_adjoints(case):
    """(pool, w, adjoints): the candidate rows (rows_cases.candidates) whose oracle adjoint completes with the premises of
    an exact comparison, their loss weights and those exact_adjoint.Adjoint records (cached per case).  With first_step
    None (rows_cases.INITIAL) only completion is required: those cases are compared within a bound."""
    if case.name not in _POOLS:
        cand = rc.candidates(case)
        w_all = weights(case, len(cand), cand.shape[1])
        m = module(case)
        rows, ws, res = [], [], []
        with np.errstate(all="ignore"):
            for y, w in zip(cand, w_all):
                try:
                    a = xa.adjoint_oracle(m, (y[None],), case.t, (w[:, None, :],), case.method, case.rtol, case.atol,
                                          options(case))
                except AssertionError:
                    continue
                exact = all(q["dyadic"] and q["decisions_agree"] and q["margin"] > es.MARGIN[case.dtype]
                            for q in premises(a, case))
                if case.first_step is not None and not exact:
                    continue                   # a decision too close to the threshold: no exact comparison possible
                rows.append(y)
                ws.append(w)
                res.append(a)
        _POOLS.clear()
        _POOLS[case.name] = (np.stack(rows), np.stack(ws), res)
    return _POOLS[case.name]


def premises(a, case):
    """es.premises of the forward solve and of every backward interval of one oracle adjoint."""
    return [es.premises(a.forward, case.first_step)] + [es.premises(s, case.first_step) for s in a.backward]


def expected(res, idx):
    """Per batch row: y0.grad (n, dim), summed backward counts, the last interval's dt_next; and t.grad with its error
    scale, summed over the batch rows in float64."""
    g = np.stack([a.g_y0[0][0] for a in res])[idx]
    acc = np.array([sum(s.stats.n_acc for s in a.backward) for a in res])[idx]
    rej = np.array([sum(s.stats.n_rej for s in a.backward) for a in res])[idx]
    dt = np.array([a.backward[-1].dt_next for a in res])[idx]
    counts = np.bincount(idx, minlength=len(res)).astype(np.float64)
    g_t = np.stack([a.g_t for a in res])
    g_t_scale = np.stack([np.maximum(a.g_t_scale, np.abs(a.g_t)) for a in res])
    return g, acc, rej, dt, counts @ g_t, counts @ g_t_scale


def run(func, y0, w, case, dev, first_step=True, **extra):
    """The engine: odeint_adjoint on a (n, dim) batch with loss sum(w * sol); returns (y0.grad, t.grad, last_stats)."""
    import tfdiffeq_b200
    from tfdiffeq_b200 import adjoint as _adj
    y = torch.tensor(y0, device=dev, requires_grad=True)
    t = torch.tensor(case.t, dtype=torch.float64, device=dev, requires_grad=True)
    opts = dict(options(case, first_step), independent_rows=True, fused_vjp=True, **extra)
    sol = tfdiffeq_b200.odeint_adjoint(func, y, t, rtol=case.rtol, atol=case.atol, method=case.method, options=opts)
    (sol * torch.tensor(np.ascontiguousarray(w.transpose(1, 0, 2)), device=dev)).sum().backward()
    return y.grad, t.grad, dict(_adj.last_stats)
