"""GPU: LatentODEFunc solves bit for bit against an oracle whose right-hand side is the device's own evaluation, on every
kernel family that evaluates it.

expm1, exp and the cuBLAS products of the module's forward are not restated by numpy, so ``b2ode_rhs_eval`` stands in,
as tests/test_exact_rhs_gpu.py does for CubicMLP: it is elementwise and deterministic, and a row's result depends on that
row alone.  The oracle (oracle/np_ref.py under the exact step schedule of tests/exact_schedule.py) keeps its own driver,
stage combines, error norm, controller and dense output on the CPU and fetches only f(t, y) from the device.
tests/test_latent_rhs_gpu.py pins those values to the 60-digit reference; this file pins the persistent kernel, the stage
kernels, the per-row kernel and the one-launch fixed grid to them, and asserts the path each solve took."""
import numpy as np
import pytest
import torch

import exact_schedule as es
import latent_cases as lc
import np_ref
from test_exact_rhs_gpu import dev_rhs
from test_exact_schedule_gpu import _assert_exact, _ratio_bar

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _engine(module, y0, t, method, rtol, atol, opts):
    kw = {} if rtol is None else dict(rtol=rtol, atol=atol)
    sol = tfd().odeint(module, torch.tensor(y0, device=DEV), torch.tensor(t), method=method, options=opts, **kw)
    return sol.cpu().numpy(), dict(tfd().last_stats)


@pytest.mark.parametrize("path", ["persistent", "stages"])
@pytest.mark.parametrize("method,dtype,reverse", lc.SOLVE_CASES)
def test_shared_step_solves_equal_the_oracle(method, dtype, reverse, path):
    module = lc.solve_module(dtype).to(DEV)
    y0, t, rtol, atol, opts = lc.solve_setup(method, dtype, reverse)
    s = es.oracle_solve(dev_rhs(module), y0, t, method, rtol, atol, opts)
    p = es.premises(s, opts["first_step"])
    assert p["dyadic"] and p["decisions_agree"] and p["n_rej"] >= 1 and p["margin"] > es.MARGIN[dtype], p
    extra = {} if path == "persistent" else dict(fused_rhs="stages")
    got, st = _engine(module, y0, t, method, rtol, atol, dict(opts, **extra))
    assert st["fused_rhs"] == (path == "persistent") and st["stage_rhs"] == (path == "stages"), st
    _assert_exact(got, st, s, dtype)


@pytest.mark.parametrize("method,dtype,reverse", lc.SOLVE_CASES)
def test_independent_rows_equal_the_oracle_row_by_row(method, dtype, reverse):
    module = lc.solve_module(dtype).to(DEV)
    y0, t, rtol, atol, opts = lc.solve_setup(method, dtype, reverse)
    y0 = y0[:24]
    got, st = _engine(module, y0, t, method, rtol, atol, dict(opts, independent_rows=True))
    assert st["independent_rows"] and st["fused_rhs"]
    f = dev_rhs(module)
    n_rej = 0
    for r in range(0, len(y0), 3):
        s = es.oracle_solve(f, y0[r:r + 1], t, method, rtol, atol, opts)
        p = es.premises(s, opts["first_step"])
        assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[dtype], p
        n_rej += p["n_rej"]
        assert np.array_equal(got[:, r], s.sol[:, 0]), r
        assert (int(st["row_accepted"][r]), int(st["row_rejected"][r])) == (s.stats.n_acc, s.stats.n_rej), r
        assert float(st["row_dt_next"][r]) == s.dt_next, r
        m = s.rec.m[-1]
        assert abs(float(st["row_error_ratio"][r]) - m) <= _ratio_bar(dtype) * m, r
    assert n_rej >= 1


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("reverse", [False, True])
def test_fixed_grid_rk4_equals_the_oracle(dtype, reverse):
    """k_fused_fixed on a step_size grid finer than the outputs: interpolated rows."""
    module = lc.solve_module(dtype).to(DEV)
    y0, t, opts = lc.fixed_setup(dtype, reverse)
    st_o = np_ref.Stats()
    want = np_ref.odeint(dev_rhs(module), y0, t, method="rk4", options=opts, stats=st_o)
    got, st = _engine(module, y0, t, "rk4", None, None, opts)
    assert st["fused_rhs"] and st["nfe"] == st_o.nfe
    assert got.dtype == want.dtype and np.array_equal(got, want), "%d values differ" % int((got != want).sum())
