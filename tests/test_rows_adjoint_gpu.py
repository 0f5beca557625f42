"""GPU: odeint_adjoint with options={'independent_rows': True, 'fused_vjp': True} (k_rows_adjoint) -- every row's
gradients are those of odeint_adjoint on that row alone.

Under the exact schedule every row's y0.grad, summed backward counts and last dt_next must equal the oracle adjoint of its
pool row (tests/rows_adjoint_cases.py; tests/test_rows_adjoint_cpu.py checks the premises); t.grad, a sum over rows of dot
products, is held to the bound of tests/test_exact_adjoint_gpu.py.  Right-hand sides that are not +, -, * only are compared
with the stage-kernel backward pass (fused_vjp) of each row alone."""
import numpy as np
import pytest
import torch

import exact_adjoint as xa
import exact_schedule as es
import rows_adjoint_cases as rac
from golden_util import max_rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
T_GRAD_BOUND = {"float64": 1e-11, "float32": 1e-4}


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _launches():
    from tfdiffeq_b200 import _lib
    return int(_lib.lib.b2ode_launch_count())


def _batches(case):
    return rac.BATCHES + ((rac.BIG,) if case.method == "dopri5" and not case.reverse else ())


def _check_stats(st, case, rows, first_step=True):
    b = st["backward"]
    assert isinstance(b, dict) and b["independent_rows"] and b["fused_vjp"] and b["rows"] == rows
    assert b["intervals"] == len(case.t) - 1
    assert b["n_accepted"] == int(b["row_accepted"].sum()) and b["n_rejected"] == int(b["row_rejected"].sum())
    per = 1 + (0 if first_step else 1)
    att = int((b["row_accepted"] + b["row_rejected"]).sum())
    assert b["nfe"] == (len(case.t) - 1) * rows * per + (es.N_K[case.method] - 1) * att
    assert b["status"] == 0 and int(b["row_status"].abs().sum()) == 0
    assert st["forward"]["independent_rows"]


@pytest.mark.parametrize("name", [c.name for c in rac.CASES])
def test_rows_equal_the_oracle_adjoint_row_by_row(name):
    case = rac.ALL[name]
    pool, w, res = rac.pool_adjoints(case)
    func = rac.module(case)
    for n in _batches(case):
        idx = rac.rc.tile(len(pool), n)
        g_want, acc, rej, dt, gt_want, gt_scale = rac.expected(res, idx)
        g, gt, st = rac.run(func, pool[idx], w[idx], case, DEV)
        g = g.cpu().numpy()
        assert g.dtype == g_want.dtype and g.shape == g_want.shape
        bad = g != g_want
        assert not bad.any(), "n=%d: %d of %d gradient values differ (first at %s)" % (
            n, int(bad.sum()), bad.size, np.argwhere(bad)[0])
        b = st["backward"]
        assert np.array_equal(b["row_accepted"].cpu().numpy(), acc), n
        assert np.array_equal(b["row_rejected"].cpu().numpy(), rej), n
        assert np.array_equal(b["row_dt_next"].cpu().numpy(), dt), n
        err = np.abs(gt.cpu().numpy() - gt_want)
        assert np.all(err <= T_GRAD_BOUND[case.dtype] * gt_scale), (n, float(np.max(err / np.maximum(gt_scale, 1e-300))))
        _check_stats(st, case, n)
        del g, bad, st


def _non_basic():
    kep = es._case("kepler", "dopri5", "float64", False, "r1")
    t = np.array([0.0, 0.0731, 0.1313, 0.1875, 0.25])
    out = [kep._replace(name="kepler-dopri5-f64", t=t), kep._replace(name="kepler-dopri8-f64", method="dopri8", t=t)]
    for dt in es.DTYPES:
        c = es._case("cubic", "dopri5", dt, False, "r1")
        out.append(c._replace(name="cubic-dopri5-" + dt, t=t * 4))
    return out


NON_BASIC = _non_basic()


@pytest.mark.parametrize("k", range(len(NON_BASIC)))
def test_pow_and_tanh_rows_equal_the_stage_kernels_alone(k):
    """Kepler (pow) and a frozen CubicMLP (tanh), 132 rows: each row's y0.grad and summed counts equal those of the
    stage-kernel backward pass (fused_vjp) of that row alone, bit for bit -- the same RHS::eval / vjp bits, and decisions
    that the exact schedule's margin fixes."""
    case = NON_BASIC[k]
    if case.problem == "kepler":
        func = tfd().rhs.Kepler()
        y0 = es.initial_state(case, 17)                     # (17, 32): 136 orbits of 4
        dim = 4
    else:
        g = torch.Generator().manual_seed(0)
        func = tfd().rhs.CubicMLP(hidden=50, dtype=torch.float64 if case.dtype == "float64" else torch.float32,
                                  generator=g).to(DEV)
        for p in func.parameters():
            p.requires_grad_(False)
        y0 = es.initial_state(case, 132)
        dim = 2
    rows = y0.reshape(-1, dim)
    rng = np.random.default_rng(5)
    w = (xa._pow2(rng, (len(rows), len(case.t), dim), -3, 1) * (rng.random((len(rows), len(case.t), dim)) >= 0.125))
    w[:, 1] = 0.0
    w = w.astype(case.dtype)
    gb, _, st = rac.run(func, rows, w, case, DEV)
    gb = gb.cpu().numpy()
    b = st["backward"]
    for r in range(len(rows)):
        y = torch.tensor(rows[r:r + 1], device=DEV, requires_grad=True)
        t = torch.tensor(case.t, dtype=torch.float64, device=DEV)
        sol = tfd().odeint_adjoint(func, y, t, rtol=case.rtol, atol=case.atol, method=case.method,
                                   options=rac.options(case), adjoint_options=dict(rac.options(case), fused_vjp=True))
        (sol * torch.tensor(w[r][:, None, :], device=DEV)).sum().backward()
        one = tfd().adjoint.last_stats["backward"]
        assert np.array_equal(gb[r:r + 1], y.grad.cpu().numpy()), r
        assert int(b["row_accepted"][r]) == sum(s["n_accepted"] for s in one), r
        assert int(b["row_rejected"][r]) == sum(s["n_rejected"] for s in one), r
        assert float(b["row_dt_next"][r]) == one[-1]["dt_next"], r


@pytest.mark.parametrize("name", [c.name for c in rac.INITIAL])
def test_initial_step_per_row_and_interval(name):
    """first_step=None: the heuristic per row and interval; fp64 gradients within 1e-12 of the oracle's and fp64 counts
    equal.  In fp32 pow and the sums' order differ from numpy in the last ulps, which can move a decision and so a whole
    interval's schedule: fp32 gradients are held to the parity bar of the forward solve (1e-3)."""
    case = rac.ALL[name]
    pool, w, _ = rac.pool_adjoints(case)
    m = rac.module(case)
    res = [xa.adjoint_oracle(m, (y[None],), case.t, (ww[:, None, :],), case.method, case.rtol, case.atol,
                             rac.options(case, first_step=False)) for y, ww in zip(pool, w)]
    idx = rac.rc.tile(len(pool), 4099)
    g_want, acc, rej, _, _, _ = rac.expected(res, idx)
    g, _, st = rac.run(m, pool[idx], w[idx], case, DEV, first_step=False)
    bar = 1e-12 if case.dtype == "float64" else 1e-3
    assert max_rel_err(g.cpu().numpy(), g_want) <= bar
    if case.dtype == "float64":
        assert np.array_equal(st["backward"]["row_accepted"].cpu().numpy(), acc)
        assert np.array_equal(st["backward"]["row_rejected"].cpu().numpy(), rej)
    _check_stats(st, case, 4099, first_step=False)


def test_ordinary_controller_at_benchmark_size():
    """65 536 Lorenz rows, fp64 dopri5, t = arange(11) * 0.01, default tolerances: 64 random rows against the oracle adjoint
    of each alone, within 1e-6 relative."""
    rng = np.random.default_rng(0)
    y0 = 1.0 + 0.1 * rng.standard_normal((65536, 3))
    t_np = np.arange(11) * 0.01
    w = rng.standard_normal((11, 65536, 3))
    y = torch.tensor(y0, device=DEV, requires_grad=True)
    t = torch.tensor(t_np, device=DEV, requires_grad=True)
    sol = tfd().odeint_adjoint(tfd().rhs.Lorenz(), y, t, method="dopri5",
                               options={"independent_rows": True, "fused_vjp": True})
    (sol * torch.tensor(w, device=DEV)).sum().backward()
    g = y.grad.cpu().numpy()
    b = tfd().adjoint.last_stats["backward"]
    att = (b["row_accepted"] + b["row_rejected"]).cpu().numpy()
    assert b["status"] == 0 and len(np.unique(att)) > 1
    m = tfd().rhs.Lorenz()
    for r in np.random.default_rng(1).choice(65536, 64, replace=False):
        a = xa.adjoint_oracle(m, (y0[r:r + 1],), t_np, (w[:, r:r + 1],), "dopri5", 1e-6, 1e-12, {})
        assert max_rel_err(g[r:r + 1], a.g_y0[0]) <= 1e-6, r


def test_nan_weight_fails_that_row_only():
    case = rac.ALL["lorenz-dopri5-f64-fwd-rows"]
    pool, w, _ = rac.pool_adjoints(case)
    idx = rac.rc.tile(len(pool), 10000)
    ww = w[idx].copy()
    ww[4321, -1, 1] = np.nan
    with pytest.raises(AssertionError, match=r"(?s)non-finite values in state .*\[row 4321; 1 of 10000 rows failed\]"):
        rac.run(rac.module(case), pool[idx], ww, case, DEV)
    st = tfd().adjoint.last_stats["backward"]
    bad = torch.nonzero(st["row_status"]).flatten().tolist()
    assert bad == [4321] and int(st["row_status"][4321]) & 2


def test_max_num_steps_marks_only_the_rows_that_exceed_it():
    """A max_num_steps for the backward solves alone.  An interval's solve has one output time, so under the exact schedule
    it fails exactly when the oracle's interval took more attempts than the limit (every attempt before the last one
    leaves the output cursor in place); exactly the batch rows tiled from such pool rows are marked."""
    case = rac.ALL["lorenz-dopri5-f64-fwd-rows"]
    pool, w, res = rac.pool_adjoints(case)
    most = np.array([max(s.stats.n_acc + s.stats.n_rej for s in a.backward) for a in res])
    limit = int(np.median(most))
    fails = most > limit
    assert fails.any() and not fails.all()
    idx = rac.rc.tile(len(pool), 4099)
    y = torch.tensor(pool[idx], device=DEV, requires_grad=True)
    t = torch.tensor(case.t, dtype=torch.float64, device=DEV)
    opts = dict(rac.options(case), independent_rows=True, fused_vjp=True)
    sol = tfd().odeint_adjoint(rac.module(case), y, t, rtol=case.rtol, atol=case.atol, method=case.method, options=opts,
                               adjoint_options=dict(opts, max_num_steps=limit))
    loss = (sol * torch.tensor(np.ascontiguousarray(w[idx].transpose(1, 0, 2)), device=DEV)).sum()
    with pytest.raises(AssertionError, match=r"max_num_steps exceeded \(%d>=%d\)" % (limit, limit)):
        loss.backward()
    status = tfd().adjoint.last_stats["backward"]["row_status"].cpu().numpy()
    assert np.array_equal(status != 0, fails[idx])
    assert np.all(status[status != 0] == 4)


def test_no_forward_calls_constant_launches_and_determinism():
    case = rac.ALL["lorenz-dopri5-f64-fwd-rows"]
    pool, w, _ = rac.pool_adjoints(case)
    idx = rac.rc.tile(len(pool), 4099)
    func = rac.module(case)
    calls = []
    h = func.register_forward_hook(lambda *a: calls.append(1))
    deltas = {}
    try:
        for T in (3, 11):
            c = case._replace(t=case.t[:T])
            y = torch.tensor(pool[idx], device=DEV, requires_grad=True)
            t = torch.tensor(c.t, dtype=torch.float64, device=DEV, requires_grad=True)
            sol = tfd().odeint_adjoint(func, y, t, rtol=c.rtol, atol=c.atol, method=c.method,
                                       options=dict(rac.options(c), independent_rows=True, fused_vjp=True))
            loss = (sol * torch.tensor(np.ascontiguousarray(w[idx][:, :T].transpose(1, 0, 2)), device=DEV)).sum()
            torch.cuda.synchronize()
            n0, before = len(calls), _launches()
            loss.backward()
            torch.cuda.synchronize()
            deltas[T] = _launches() - before
            assert len(calls) == n0
    finally:
        h.remove()
    assert deltas[3] == deltas[11] == 2, deltas
    runs = [rac.run(func, pool[idx], w[idx], case, DEV)[:2] for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    # T = 1: y0.grad is grad_output[0], t.grad zero, nothing launched
    y = torch.tensor(pool[idx], device=DEV, requires_grad=True)
    t = torch.tensor(case.t[:1], dtype=torch.float64, device=DEV, requires_grad=True)
    sol = tfd().odeint_adjoint(func, y, t, method="dopri5", options={"independent_rows": True, "fused_vjp": True})
    wt = torch.tensor(w[idx][:, :1].transpose(1, 0, 2).copy(), device=DEV)
    loss = (sol * wt).sum()
    before = _launches()
    loss.backward()
    assert _launches() == before
    assert torch.equal(y.grad, wt[0]) and torch.equal(t.grad, torch.zeros_like(t))


def test_refusals_raise_before_any_launch():
    from test_rows_adjoint_cpu import refusal_cases
    cases, t = refusal_cases(DEV)
    for name, func, y0, kw in cases:
        before = _launches()
        with pytest.raises(ValueError):
            tfd().odeint_adjoint(func, y0, t, **kw)
        torch.cuda.synchronize()
        assert _launches() == before, name
