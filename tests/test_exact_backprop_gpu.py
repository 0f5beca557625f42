"""odeint(..., options={'backprop': True}) bit for bit against tests/exact_backprop.py's restated reverse sweep: y0.grad
and every parameter gradient equal (torch.equal), and the accepted and rejected counts equal the oracle's, for the
generic path (adaptive and fixed grid, at sizes where k_bp_combine strides over its grid), tuple states, the linear
funcs, the built-in right-hand sides through k_bp_rhs, a record that grows while the solve runs and the independent-rows
kernel k_rows_bp.  A trainable CubicMLP, whose tanh rules out bit-exactness, is checked against fused_rhs=False and for
run-to-run equality."""
import copy

import numpy as np
import pytest
import torch

import exact_adjoint as ea
import exact_backprop as eb
import exact_schedule as es
import rows_cases as rc
from test_exact_backprop_cpu import check_premises, check_recompute

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _engine(case, module, y0, w, **extra):
    """(y0 grads, parameter grads, solver stats) of the engine's backprop for the loss sum <w, sol>."""
    mod = copy.deepcopy(module).to(DEV)
    ys = tuple(torch.tensor(v, device=DEV).requires_grad_(True) for v in y0)
    ti = eb.tensor_input(case)
    opts = dict(eb.options(case), backprop=True, **extra)
    sol = tfd().odeint(mod, ys[0] if ti else ys, torch.tensor(case.t), rtol=case.rtol or 1e-7, atol=case.atol or 1e-9,
                       method=case.method, options=opts)
    stats = dict(tfd().solvers.last_stats)
    sol = (sol,) if ti else sol
    live = [(s, torch.tensor(g, device=DEV)) for s, g in zip(sol, w) if g is not None]
    params = [p for p in mod.parameters() if p.requires_grad]
    gs = torch.autograd.grad([s for s, _ in live], list(ys) + params, [g for _, g in live])
    return [g.cpu() for g in gs[:len(ys)]], [g.cpu() for g in gs[len(ys):]], stats


def _check(name):
    case = eb.ALL[name]
    module, y0, w, fwd, want = eb.solve_case(case)
    check_premises(case, fwd)
    check_recompute(case, fwd)
    gy, gp, stats = _engine(case, module, y0, w)
    assert (stats["n_accepted"], stats["n_rejected"]) == (fwd.n_acc, fwd.n_rej)
    for i, (a, b) in enumerate(zip(gy, want.y0)):
        assert torch.equal(a, torch.from_numpy(np.ascontiguousarray(b))), (name, "y0", i, _where(a, b))
    assert len(gp) == len(want.params)
    for i, (a, b) in enumerate(zip(gp, want.params)):
        assert torch.equal(a, b), (name, "param", i, _where(a, b.numpy()))
    return case, fwd


def _where(a, b):
    b = torch.as_tensor(np.asarray(b))
    bad = (a != b).nonzero()
    return int(bad.shape[0]), float((a - b).abs().max())


@pytest.mark.parametrize("name", [c.name for c in eb.GENERIC])
def test_generic_adaptive(name):
    _check(name)


@pytest.mark.parametrize("name", [c.name for c in eb.LARGE])
def test_generic_at_striding_sizes(name):
    _check(name)


@pytest.mark.parametrize("name", [c.name for c in eb.FIXED_CASES])
def test_fixed_grid(name):
    _check(name)


@pytest.mark.parametrize("name", [c.name for c in eb.TUPLE])
def test_tuple5(name):
    _check(name)


@pytest.mark.parametrize("name", [c.name for c in eb.LINEAR])
def test_linear_funcs(name):
    _check(name)


@pytest.mark.parametrize("name", [c.name for c in eb.BUILTIN])
def test_builtin_through_k_bp_rhs(name):
    _check(name)


@pytest.mark.parametrize("name", [c.name for c in eb.GROWTH])
def test_record_grows_while_the_solve_runs(name):
    case, fwd = _check(name)
    assert fwd.n_acc > 2 * eb.RECORD_SLOTS and tfd().backprop.last_stats["steps"] == fwd.n_acc


# every case but Lotka-Volterra under bosh3 and fp64 dopri5, whose scaled pool rows take thousands of steps in the
# restatement; the rest still cover every tableau, dtype and direction
ROWS_CASES = [c.name for c in rc.CASES if not (c.problem == "lv" and (c.method == "bosh3" or
                                                                     (c.method, c.dtype) == ("dopri5", "float64")))]


@pytest.mark.parametrize("name", ROWS_CASES)
def test_independent_rows_against_the_restated_sweep(name):
    """Row r of a 4 099-row independent-rows solve gets the restated sweep of its pool row solved alone."""
    case = rc.ALL[name]
    pool, _ = rc.pool_solves(case)
    module = {"lorenz": tfd().rhs.Lorenz, "lv": tfd().rhs.LotkaVolterra}[case.problem]()
    idx = rc.tile(len(pool), rc.BATCHES[-1])
    rng = np.random.default_rng(9)
    w_pool = (np.where(rng.random((len(case.t),) + pool.shape) < 0.5, -1.0, 1.0)
              * 2.0 ** rng.integers(-3, 2, (len(case.t),) + pool.shape)).astype(case.dtype)
    opts = dict(es.OPTIONS, first_step=case.first_step)
    f = ea.numpy_func(module, case.dtype, True)
    want = []
    for p in range(len(pool)):
        fwd = eb.forward(f, (pool[p:p + 1],), case.t, case.method, case.rtol, case.atol, opts)
        g = eb.reverse_sweep(fwd, case.method, module, (pool[p:p + 1],), (w_pool[:, p:p + 1],), True, case.reverse)
        want.append(g.y0[0][0])
    y = torch.tensor(pool[idx], device=DEV).requires_grad_(True)
    sol = tfd().odeint(module.to(DEV), y, torch.tensor(case.t), rtol=case.rtol, atol=case.atol, method=case.method,
                       options=dict(opts, independent_rows=True, backprop=True))
    (gy,) = torch.autograd.grad(sol, y, torch.tensor(w_pool[:, idx], device=DEV))
    assert torch.equal(gy.cpu(), torch.from_numpy(np.stack([want[i] for i in idx])))


@pytest.mark.parametrize("hidden", [1, 50, 128])
def test_trainable_cubic_mlp_at_a_striding_size(hidden):
    """k_bp_rhs's CubicMLP weight sums over two row passes with a partial last tile: within 1e-10 of the unfused path
    (autograd of the module), and the same bits on a second run."""
    rows = 270336 + 1001
    g = torch.Generator().manual_seed(1)
    y0 = (torch.tensor([2.0, 0.0], dtype=torch.float64) + 0.1 * torch.randn(rows, 2, generator=g, dtype=torch.float64))
    w = torch.randn(3, rows, 2, generator=g, dtype=torch.float64).to(DEV)
    t = torch.tensor([0.0, 0.25, 0.5], dtype=torch.float64)
    base = tfd().rhs.CubicMLP(hidden, dtype=torch.float64, std=0.5, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        base.b1.normal_(0, 0.1, generator=g)
        base.b2.normal_(0, 0.1, generator=g)
    out = []
    for extra in ({}, {}, {"fused_rhs": False}):
        mod = copy.deepcopy(base).to(DEV)
        y = y0.to(DEV).requires_grad_(True)
        sol = tfd().odeint(mod, y, t, rtol=1e-6, atol=1e-8, method="dopri5",
                           options=dict(extra, backprop=True, first_step=0.125))
        out.append(torch.autograd.grad(sol, [y] + list(mod.parameters()), w))
    for a, b in zip(out[0], out[1]):
        assert torch.equal(a, b)
    for a, b in zip(out[0][1:], out[2][1:]):
        assert float((a - b).abs().max()) <= 1e-10 * max(1.0, float(b.abs().max())), (hidden, a.shape)
