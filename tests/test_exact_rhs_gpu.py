"""GPU: Kepler (pow) and CubicMLP (tanh) solves bit for bit against an oracle whose right-hand side is the device's own
evaluation, and Lorenz / Lotka-Volterra with non-default parameters against the numpy oracle, on every kernel family.

pow and tanh are not correctly rounded, so numpy cannot restate them.  ``b2ode_rhs_eval`` can stand in: it is elementwise
and deterministic, and a row's result depends on that row alone.  The oracle (oracle/np_ref.py under the exact step
schedule of tests/exact_schedule.py) keeps its own driver, stage combines, error norm, controller and dense output on the
CPU and fetches only f(t, y) from the device, always with time_sign = +1 (it applies the reverse-time wrapper itself).
tests/test_rhs_eval_gpu.py pins those values to the mathematics; this file pins every other instantiation of ``eval`` --
the stage kernels with stage terms, the persistent, per-row and fixed-grid kernels -- to them."""
import numpy as np
import pytest
import torch

import exact_schedule as es
import np_ref
import rhs_cases as rc
from test_exact_schedule_gpu import _assert_exact, _ratio_bar

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def dev_rhs(module):
    """f(t, y) for the numpy oracle, evaluated by ``b2ode_rhs_eval`` in y's dtype."""
    def f(t, y):
        return rc.device_eval(module, torch.from_numpy(np.ascontiguousarray(y)).to(DEV)).cpu().numpy()
    return f


def _oracle_func(case, module):
    return dev_rhs(module) if rc.solve_kind(case) in ("kepler", "mlp") else rc.numpy_rhs(case, module)


_SOLVES = {}


def _oracle(case, module, y0, t, rtol, atol, opts):
    """The oracle's solve of a case, shared by the paths that run the same system, method, dtype and direction."""
    key = (case.system, case.method, case.dtype, case.reverse)
    if key not in _SOLVES:
        _SOLVES.clear()
        _SOLVES[key] = es.oracle_solve(_oracle_func(case, module), y0, t, case.method, rtol, atol, opts)
    return _SOLVES[key]


def _engine(module, y0, t, case, rtol, atol, opts):
    kw = {} if rtol is None else dict(rtol=rtol, atol=atol)
    sol = tfd().odeint(module, torch.tensor(y0, device=DEV), torch.tensor(t), method=case.method, options=opts, **kw)
    return sol.cpu().numpy(), dict(tfd().last_stats)


_ORDER = sorted(rc.SOLVE_CASES, key=lambda c: (c.system, c.method, c.dtype, c.reverse, c.path))


@pytest.mark.parametrize("name", [c.name for c in _ORDER if c.path in ("persistent", "stages", "stages_graph")])
def test_shared_step_solves_equal_the_oracle(name):
    case = rc.SOLVE[name]
    module = rc.solve_module(case).to(DEV)
    y0, t, rtol, atol, opts = rc.solve_setup(case)
    s = _oracle(case, module, y0, t, rtol, atol, opts)
    p = es.premises(s, opts["first_step"])
    assert p["dyadic"] and p["decisions_agree"] and p["n_rej"] >= 1 and p["margin"] > es.MARGIN[case.dtype], p
    extra = {"persistent": {}, "stages": dict(fused_rhs="stages"),
             "stages_graph": dict(fused_rhs="stages", cuda_graph=True)}[case.path]
    got, st = _engine(module, y0, t, case, rtol, atol, dict(opts, **extra))
    assert st["fused_rhs"] == (case.path == "persistent") and st["stage_rhs"] == (case.path != "persistent"), st
    assert st["cuda_graph"] == (case.path == "stages_graph")
    _assert_exact(got, st, s, case.dtype)


@pytest.mark.parametrize("name", [c.name for c in _ORDER if c.path == "rows"])
def test_independent_rows_equal_the_oracle_row_by_row(name):
    """options={'independent_rows': True}: each of the first rows of the batch against the oracle's solve of that row
    alone, with its own counts and final step size."""
    case = rc.SOLVE[name]
    module = rc.solve_module(case).to(DEV)
    y0, t, rtol, atol, opts = rc.solve_setup(case)
    y0 = np.ascontiguousarray(y0.reshape(-1, rc.row_dim(case))[:24])
    got, st = _engine(module, y0, t, case, rtol, atol, dict(opts, independent_rows=True))
    assert st["independent_rows"] and st["fused_rhs"]
    f = _oracle_func(case, module)
    n_rej = 0
    for r in range(0, len(y0), 3):
        s = es.oracle_solve(f, y0[r:r + 1], t, case.method, rtol, atol, opts)
        p = es.premises(s, opts["first_step"])
        assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[case.dtype], p
        n_rej += p["n_rej"]
        assert np.array_equal(got[:, r], s.sol[:, 0]), r
        assert (int(st["row_accepted"][r]), int(st["row_rejected"][r])) == (s.stats.n_acc, s.stats.n_rej), r
        assert float(st["row_dt_next"][r]) == s.dt_next, r
        m = s.rec.m[-1]
        assert abs(float(st["row_error_ratio"][r]) - m) <= _ratio_bar(case.dtype) * m, r
    assert n_rej >= 1


@pytest.mark.parametrize("name", [c.name for c in _ORDER if c.path == "fixed"])
def test_fixed_grid_solves_equal_the_oracle(name):
    """k_fused_fixed on a step_size grid finer than the outputs: interpolated rows, both directions."""
    case = rc.SOLVE[name]
    module = rc.solve_module(case).to(DEV)
    y0, t, _, _, opts = rc.solve_setup(case)
    st_o = np_ref.Stats()
    want = np_ref.odeint(_oracle_func(case, module), y0, t, method=case.method, options=opts, stats=st_o)
    got, st = _engine(module, y0, t, case, None, None, opts)
    assert st["fused_rhs"] and st["nfe"] == st_o.nfe
    assert got.dtype == want.dtype and np.array_equal(got, want), "%d values differ" % int((got != want).sum())


# --------------------------------------------------------------------------------------------------
# a state whose last axis holds several rows
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lorenz", "lv", "mlp", "kepler"])
@pytest.mark.parametrize("method", ["dopri5", "rk4"])
def test_a_state_of_several_rows_per_batch_entry_is_solved_row_by_row(kind, method):
    """rhs.py: a ``(..., k * dim)`` state is k rows per entry.  The kernels solve it as rows, and ``forward`` accepts it
    for every built-in system, so the generic path does too: the wide state gives the bits of the reshaped one."""
    system = {"lorenz": "lorenz-a", "lv": "lv-a", "mlp": "mlp-h50-cube", "kepler": "kepler"}[kind]
    case = rc._sc(system, method, "float64", False, "fixed" if method == "rk4" else "persistent")
    module = rc.solve_module(case).to(DEV)
    y0, t, rtol, atol, opts = rc.solve_setup(case)
    dim = rc.row_dim(case)
    narrow = np.ascontiguousarray(y0.reshape(-1, dim)[:64])
    wide = narrow.reshape(2, 32 * dim)
    a, sa = _engine(module, narrow, t, case, rtol, atol, opts)
    b, sb = _engine(module, wide, t, case, rtol, atol, opts)
    assert sa["fused_rhs"] and sb["fused_rhs"]
    assert np.array_equal(a.reshape(b.shape), b)
    c, sc = _engine(module, wide, t, case, rtol, atol, dict(opts, fused_rhs=False))
    assert not sc["fused_rhs"] and c.shape == b.shape
    if kind == "mlp":
        # forward's products go through cuBLAS: to rounding, at the bar of test_cubic_mlp_builtin_fixed_and_adaptive_vs_generic
        assert method != "rk4" or np.abs(c - b).max() <= 1e-9 * max(1.0, np.abs(b).max())
    else:
        assert np.array_equal(c, b)
