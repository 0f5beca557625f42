"""GPU: options={'independent_rows': True} (k_rows_adaptive) -- every row solved as if it had been passed to odeint alone.

Under the exact schedule (tests/exact_schedule.py) every row must equal the oracle's solve of its pool row alone bit for bit,
with that solve's accepted / rejected counts and final step size (tests/rows_cases.py builds the pools;
tests/test_independent_rows_cpu.py checks their premises).  Right-hand sides that are not +, -, * only are compared with the
persistent kernel's solve of each row alone; the ordinary controller at the benchmark's size with the parity bars."""
import warnings

import numpy as np
import pytest
import torch

import exact_schedule as es
import rows_cases as rc
import np_ref
from golden_util import max_rel_err
from problems import PROBLEMS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _tdtype(dtype):
    return torch.float64 if dtype == "float64" else torch.float32


def _builtin(case):
    r = tfd().rhs
    if case.problem == "lorenz":
        return r.Lorenz()
    if case.problem == "lv":
        return r.LotkaVolterra()
    if case.problem == "kepler":
        return r.Kepler()
    g = torch.Generator().manual_seed(0)
    return r.CubicMLP(hidden=50, dtype=_tdtype(case.dtype), generator=g).to(DEV)


def _solve(func, y0, case, first_step=True, rows=True, **opts):
    """The engine on `case` (y0: numpy array); returns (numpy solution, last_stats)."""
    options = dict(es.OPTIONS, **opts)
    if rows:
        options["independent_rows"] = True
    if first_step:
        options["first_step"] = case.first_step
    sol = tfd().odeint(func, torch.tensor(y0, device=DEV), torch.tensor(case.t), rtol=case.rtol, atol=case.atol,
                       method=case.method, options=options)
    return sol.cpu().numpy(), dict(tfd().last_stats)


def _ratio_bar(dtype):
    return 1e-12 if dtype == "float64" else 2.0 ** -21


def _check_totals(st, case, rows):
    acc, rej = st["row_accepted"], st["row_rejected"]
    assert st["independent_rows"] and st["fused_rhs"] and st["rows"] == rows
    assert "dt_next" not in st and "error_ratio" not in st
    assert acc.dtype == rej.dtype == torch.int64 and st["row_status"].dtype == torch.int32
    assert st["row_dt_next"].dtype == st["row_error_ratio"].dtype == torch.float64
    assert st["n_accepted"] == int(acc.sum()) and st["n_rejected"] == int(rej.sum())
    n_k = es.N_K[case.method]
    per_row = 1 + (1 if case.first_step is None else 0)
    assert st["nfe"] == rows * per_row + (n_k - 1) * int((acc + rej).sum())
    assert int(st["row_status"].abs().sum()) == 0 and st["status"] == 0


def _batches(case):
    return rc.BATCHES + ((rc.BIG,) if case.method == "dopri5" and not case.reverse else ())


@pytest.mark.parametrize("name", [c.name for c in rc.CASES])
def test_rows_equal_the_oracle_row_by_row(name):
    case = rc.ALL[name]
    pool, solves = rc.pool_solves(case)
    want_sol = np.stack([s.sol[:, 0, :] for s in solves])                          # (pool, T, dim)
    want_acc = np.array([s.stats.n_acc for s in solves])
    want_rej = np.array([s.stats.n_rej for s in solves])
    want_dt = np.array([s.dt_next for s in solves])
    want_m = np.array([s.rec.m[-1] for s in solves])
    for n in _batches(case):
        idx = rc.tile(len(pool), n)
        with warnings.catch_warnings():
            warnings.simplefilter("error", RuntimeWarning)
            got, st = _solve(_builtin(case), pool[idx], case)
        assert got.dtype == want_sol.dtype and got.shape == (len(case.t), n, pool.shape[1])
        want = want_sol[idx].transpose(1, 0, 2)
        bad = got != want
        assert not bad.any(), "n=%d: %d of %d values differ from the oracle (first at %s)" % (
            n, int(bad.sum()), bad.size, np.argwhere(bad)[0])
        del want, bad
        assert np.array_equal(st["row_accepted"].cpu().numpy(), want_acc[idx]), n
        assert np.array_equal(st["row_rejected"].cpu().numpy(), want_rej[idx]), n
        assert np.array_equal(st["row_dt_next"].cpu().numpy(), want_dt[idx]), n
        m = st["row_error_ratio"].cpu().numpy()
        assert np.all(np.abs(m - want_m[idx]) <= _ratio_bar(case.dtype) * want_m[idx]), n
        _check_totals(st, case, n)


@pytest.mark.parametrize("name", [c.name for c in rc.INITIAL])
def test_initial_step_per_row_matches_the_oracle(name):
    """first_step=None: the heuristic on each row's own norms.  Under the exact schedule dt_next = h0 * 2**-n_rej, so
    dt_next * 2**n_rej is the row's initial step; it must match the oracle's within 1e-12 (fp64) / 1e-5 (fp32) -- pow and
    the sums' order differ from numpy in the last ulps.  In fp32 that difference can move a decision and so the whole
    schedule, so only fp64 counts must equal the oracle's; the solution is held to the parity bars in both."""
    case = rc.ALL[name]
    pool, solves = rc.pool_solves(case)
    for s in solves:
        assert s.dt_next == s.rec.dt[0] * 2.0 ** -s.stats.n_rej
    idx = rc.tile(len(pool), 4099)
    got, st = _solve(_builtin(case), pool[idx], case, first_step=False)
    acc, rej = st["row_accepted"].cpu().numpy(), st["row_rejected"].cpu().numpy()
    want_acc, want_rej = np.array([s.stats.n_acc for s in solves])[idx], np.array([s.stats.n_rej for s in solves])[idx]
    if case.dtype == "float64":
        assert np.array_equal(acc, want_acc) and np.array_equal(rej, want_rej)
    h0 = st["row_dt_next"].cpu().numpy() * 2.0 ** rej
    want_h0 = np.array([s.rec.dt[0] for s in solves])[idx]
    bar = 1e-12 if case.dtype == "float64" else 1e-5
    assert np.all(np.abs(h0 - want_h0) <= bar * want_h0)
    want = np.stack([s.sol[:, 0, :] for s in solves])[idx].transpose(1, 0, 2)
    assert max_rel_err(got, want) <= (1e-6 if case.dtype == "float64" else 1e-3)
    _check_totals(st, case, 4099)


NON_BASIC = [es._case("kepler", "dopri5", "float64", False, "r3")._replace(method="dopri8", name="kepler-dopri8-f64")] + [
    es._case("cubic", "dopri5", dt, False, "r9") for dt in es.DTYPES]


@pytest.mark.parametrize("k", range(len(NON_BASIC)))
def test_pow_and_tanh_rows_equal_the_persistent_kernel_alone(k):
    """Kepler (pow; a (3, 32) state is 24 rows of one orbit) and CubicMLP (tanh): each row of the batched solve equals the
    persistent kernel's solve of that row alone, bit for bit."""
    case = NON_BASIC[k]
    f = _builtin(case)
    y0 = es.initial_state(case, es.batch_size(case, 132))
    got, st = _solve(f, y0, case)
    dim = f.dim
    rows = y0.reshape(-1, dim)
    assert st["rows"] == len(rows)
    got_rows = got.reshape(len(case.t), -1, dim)
    for r in range(len(rows)):
        one, so = _solve(f, rows[r:r + 1], case, rows=False)
        assert so["fused_rhs"] and not so.get("independent_rows")
        assert np.array_equal(got_rows[:, r], one[:, 0]), r
        assert int(st["row_accepted"][r]) == so["n_accepted"] and int(st["row_rejected"][r]) == so["n_rejected"]
        assert float(st["row_dt_next"][r]) == so["dt_next"]


def test_ordinary_controller_at_benchmark_size():
    """65 536 Lorenz rows, fp64 dopri5, the benchmark's times and default tolerances: 64 random rows against the oracle's solve
    of each alone, within the parity bars (1e-6, counts +-2); the rows do not all take the same number of steps."""
    rng = np.random.default_rng(0)
    y0 = 1.0 + 0.1 * rng.standard_normal((65536, 3))
    t = np.arange(1000) * 0.01
    sol = tfd().odeint(tfd().rhs.Lorenz(), torch.tensor(y0, device=DEV), torch.tensor(t), method="dopri5",
                       options={"independent_rows": True})
    st = dict(tfd().last_stats)
    acc = st["row_accepted"].cpu().numpy()
    rej = st["row_rejected"].cpu().numpy()
    assert len(np.unique(acc)) > 1
    f = PROBLEMS["lorenz"](backend="numpy")
    for r in np.random.default_rng(1).choice(65536, 64, replace=False):
        s = np_ref.Stats()
        ref = np_ref.odeint(f, y0[r:r + 1], t, method="dopri5", stats=s)
        assert max_rel_err(sol[:, r:r + 1].cpu().numpy(), ref) <= 1e-6, r
        assert abs(int(acc[r]) - s.n_acc) <= 2 and abs(int(rej[r]) - s.n_rej) <= 2, (r, acc[r], rej[r], s.n_acc, s.n_rej)


def test_nan_in_one_row_fails_that_row_only():
    case = rc.ALL["lorenz-dopri5-f64-fwd-rows"]
    pool, _ = rc.pool_solves(case)
    y0 = pool[rc.tile(len(pool), 10000)].copy()
    y0[4321, 1] = np.nan
    with pytest.raises(AssertionError, match=r"non-finite values in state .*\[row 4321; 1 of 10000 rows failed\]"):
        _solve(_builtin(case), y0, case)
    st = tfd().last_stats
    bad = torch.nonzero(st["row_status"]).flatten().tolist()
    assert bad == [4321] and int(st["row_status"][4321]) & 2


def test_max_num_steps_marks_only_the_rows_that_exceed_it():
    """max_num_steps=40 is exceeded, in the oracle, by the pool's 100x rows alone (checked here)."""
    case = rc.ALL["lorenz-dopri5-f64-fwd-rows"]
    pool, solves = rc.pool_solves(case)
    f = es.numpy_rhs(case)
    fails = []
    for i, y in enumerate(pool):
        try:
            es.oracle_solve(f, y[None], case.t, case.method, case.rtol, case.atol,
                            dict(es.OPTIONS, first_step=case.first_step, max_num_steps=40))
        except AssertionError as e:
            assert "max_num_steps exceeded (40>=40)" in str(e)
            fails.append(i)
    hundred = [i for i in range(len(pool)) if np.allclose(pool[i], 100.0 * pool[i % rc.CLUSTER])]
    assert fails and fails == hundred
    idx = rc.tile(len(pool), 4099)
    with pytest.raises(AssertionError, match=r"max_num_steps exceeded \(40>=40\)"):
        _solve(_builtin(case), pool[idx], case, max_num_steps=40)
    status = tfd().last_stats["row_status"].cpu().numpy()
    assert np.array_equal(status != 0, np.isin(idx, fails))
    assert np.all(status[status != 0] == 4)


def _launches():
    from tfdiffeq_b200 import _lib
    return int(_lib.lib.b2ode_launch_count())


def test_unsupported_combinations_raise_before_any_launch():
    lorenz = tfd().rhs.Lorenz()
    y = torch.ones(4, 3, dtype=torch.float64, device=DEV)
    t = torch.linspace(0, 0.1, 3, dtype=torch.float64)
    on = {"independent_rows": True}
    calls = [
        lambda: tfd().odeint(PROBLEMS["lorenz"](backend="torch", device=DEV), y, t, method="dopri5", options=on),
        lambda: tfd().odeint(lorenz, (y, y), t, method="dopri5", options=on),
        lambda: tfd().odeint(lorenz, y, t, rtol=[1e-6, 1e-7], method="dopri5", options=on),
        lambda: tfd().odeint(lorenz, y, t, method="dopri5", options=dict(on, fused_rhs=False)),
        lambda: tfd().odeint(lorenz, y, t, method="dopri5", options=dict(on, fused_rhs="stages")),
        lambda: tfd().odeint(lorenz, y, t, method="dopri5", options=dict(on, shared_step_group=object())),
        lambda: tfd().odeint_adjoint(lorenz, y, t, method="dopri5", options=on),
        lambda: tfd().odeint_adjoint(lorenz, y, t, method="dopri5", adjoint_options=on),
    ] + [(lambda m: lambda: tfd().odeint(lorenz, y, t, method=m, options=on))(m)
         for m in ("tsit5", "adams", "fixed_adams", "explicit_adams")]
    for call in calls:
        before = _launches()
        with pytest.raises(ValueError):
            call()
        torch.cuda.synchronize()
        assert _launches() == before


@pytest.mark.parametrize("method", ["rk4", "euler"])
def test_fixed_grid_ignores_the_flag(method):
    y0 = torch.tensor(es.initial_state(rc.ALL["lorenz-dopri5-f64-fwd-rows"], 1000), device=DEV)
    t = torch.linspace(0, 0.5, 11, dtype=torch.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        a = tfd().odeint(tfd().rhs.Lorenz(), y0, t, method=method, options={"independent_rows": True})
    b = tfd().odeint(tfd().rhs.Lorenz(), y0, t, method=method)
    assert torch.equal(a, b)


def test_host_output_and_single_time():
    case = rc.ALL["lorenz-dopri5-f64-fwd-rows"]
    pool, _ = rc.pool_solves(case)
    y0 = pool[rc.tile(len(pool), 4099)]
    dev_sol, _ = _solve(_builtin(case), y0, case)
    host = torch.empty(dev_sol.shape, dtype=torch.float64).pin_memory()
    host.fill_(float("nan"))
    ret, st = _solve(_builtin(case), y0, case, host_output=host)
    assert np.array_equal(host.numpy(), dev_sol) and np.array_equal(ret, dev_sol)
    one = tfd().odeint(tfd().rhs.Lorenz(), torch.tensor(y0, device=DEV), torch.tensor([0.5], dtype=torch.float64),
                       method="dopri5", options={"independent_rows": True})
    assert one.shape == (1,) + y0.shape and np.array_equal(one[0].cpu().numpy(), y0)
    assert tfd().last_stats["n_accepted"] == 0 and tfd().last_stats["n_rejected"] == 0
