"""GPU: adaptive solves under an exact step schedule (tests/exact_schedule.py) against the oracle, bit for bit.

With safety=0.5, ifactor=1, dfactor=0.5 and a power-of-two first step, every step size is first_step * 2**-k in the
oracle and in every engine path, so for Lorenz and Lotka-Volterra (+, -, * only) every stage, step end and dense output
is a chain of correctly rounded operations: the solution must equal the oracle's exactly, the counts must be equal, the
final step size must be the oracle's, and the reported error ratio must match an exactly summed value from the oracle's
last attempt.  tests/test_exact_schedule_cpu.py checks on the oracle that each case's decisions are robust and that the
case exercises rejections, long steps, steps without output and outputs on step ends; the checks that depend on the
device's SM count are repeated here at run time."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import exact_schedule as es
from golden_util import max_rel_err
from problems import PROBLEMS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _tdtype(dtype):
    return torch.float64 if dtype == "float64" else torch.float32


_ORACLE = {}


def _oracle(case, n):
    key = (case.name, n)
    if key not in _ORACLE:
        _ORACLE.clear()            # consecutive tests share at most the last solve; keep host memory flat
        _ORACLE[key] = es.solve_case(case, n=n)
    return _ORACLE[key]


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


def _solve(func, y0, case, first_step=True, **opts):
    """The engine on `case` (y0: numpy array or tuple of arrays); returns (numpy solution, last_stats)."""
    y = tuple(torch.tensor(a, device=DEV) for a in y0) if isinstance(y0, tuple) else torch.tensor(y0, device=DEV)
    options = dict(es.OPTIONS, **opts)
    if first_step:
        options["first_step"] = case.first_step
    sol = tfd().odeint(func, y, torch.tensor(case.t), rtol=case.rtol, atol=case.atol, method=case.method, options=options)
    st = dict(tfd().last_stats)
    got = tuple(s.cpu().numpy() for s in sol) if isinstance(sol, tuple) else sol.cpu().numpy()
    return got, st


def _check_premises(s, case):
    """The run-time half of the premises (the CPU test checks them at 132 SMs)."""
    p = es.premises(s, case.first_step)
    assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[case.dtype], p


def _ratio_bar(dtype):
    # fp64: the persistent kernel's tagged partials replace the last 4 mantissa bits of the sums (2^-48); fp32: m is rounded
    return 1e-12 if dtype == "float64" else 2.0 ** -21


def _assert_exact(got, st, s, dtype):
    want = s.sol
    for g, w in (zip(got, want) if isinstance(want, tuple) else ((got, want),)):
        assert g.dtype == w.dtype and g.shape == w.shape
        bad = g != w
        assert not bad.any(), "%d of %d values differ from the oracle, max |diff| %.3e (first at %s)" % (
            int(bad.sum()), bad.size, float(np.abs(g.astype(np.float64) - w).max()), np.argwhere(bad)[0])
    assert (st["n_accepted"], st["n_rejected"], st["nfe"]) == (s.stats.n_acc, s.stats.n_rej, s.stats.nfe), st
    assert st["dt_next"] == s.dt_next, (st["dt_next"], s.dt_next)
    m = s.rec.m[-1]
    assert abs(st["error_ratio"] - m) <= _ratio_bar(dtype) * m, (st["error_ratio"], m)


# --------------------------------------------------------------------------------------------------
# the persistent kernel (k_fused_adaptive)
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c.name for c in es.PERSISTENT])
def test_persistent_kernel_is_bit_exact(name):
    case = es.ALL[name]
    sms = _sms()
    n = es.batch_size(case, sms)
    g = es.fused_geometry(n, sms, case.method, case.dtype, es.DIM[case.problem])
    want = es.BATCH_FEATURES.get((case.batch, g.tpt))
    if want is not None:
        assert g.ncw == want["ncw"] and want["has"] <= g.features and not (want.get("not", set()) & g.features), g
    y0, s = _oracle(case, n)
    _check_premises(s, case)
    got, st = _solve(_builtin(case), y0, case)
    assert st["fused_rhs"] and not st["stage_rhs"]
    _assert_exact(got, st, s, case.dtype)


def _capacity(case):
    from tfdiffeq_b200 import _lib, solvers
    from tfdiffeq_b200.odeint import SOLVERS
    f = _builtin(case)
    y = torch.zeros(1, es.DIM[case.problem], dtype=_tdtype(case.dtype), device=DEV)
    desc = SOLVERS[case.method](f, (y,), rtol=case.rtol, atol=case.atol)._describe(solvers._Segments((y,)))
    return int(_lib.lib.b2ode_fused_capacity(C.byref(desc), f.kind))


@pytest.mark.parametrize("name", [c.name for c in es.CAPACITY])
def test_persistent_kernel_at_its_capacity(name):
    """The largest batch the instantiation keeps co-resident (b2ode_fused_capacity): the fullest blocks it launches."""
    case = next(c for c in es.CAPACITY if c.name == name)
    n = _capacity(case)
    assert n > 0
    y0, s = _oracle(case, n)
    _check_premises(s, case)
    assert s.stats.n_rej >= 1
    got, st = _solve(_builtin(case), y0, case)
    assert st["fused_rhs"], "the capacity batch did not take the persistent kernel"
    _assert_exact(got, st, s, case.dtype)


def _outlier_case(k):
    rows = es.OUTLIER_ROWS(_sms())
    return es.OUTLIER[0]._replace(outlier=rows[k], name="outlier-row%d" % rows[k])


@pytest.mark.parametrize("k", range(len(es.OUTLIER)))
def test_outlier_row_dominates_and_stays_exact(k):
    """One row with a 100x larger state carries most of the sum of err^2 and the max |y| that sets the tolerance: a
    trajectory warp, compute-warp slot or block whose share were dropped would change the error ratio and the schedule."""
    case = _outlier_case(k)
    y0, s = _oracle(case, es.batch_size(case, _sms()))
    _check_premises(s, case)
    ya, yb, err = s.rec.last
    e2 = (err[0].astype(np.float64) ** 2).sum(-1)
    assert e2[case.outlier] > 0.5 * e2.sum()
    assert np.argmax(np.abs(yb[0]).max(-1)) == case.outlier
    got, st = _solve(_builtin(case), y0, case)
    assert st["fused_rhs"]
    _assert_exact(got, st, s, case.dtype)


@pytest.mark.parametrize("k", range(len(es.OUTLIER)))
def test_nan_in_any_row_is_reported(k):
    case = _outlier_case(k)
    y0 = es.initial_state(case._replace(outlier=None), es.batch_size(case, _sms()))
    y0[case.outlier, 1] = np.nan
    with pytest.raises(AssertionError, match="non-finite values in state"):
        _solve(_builtin(case), y0, case)
    assert tfd().last_stats["fused_rhs"]


@pytest.mark.parametrize("name", [c.name for c in es.NON_BASIC])
def test_persistent_equals_stage_kernels_on_pow_and_tanh(name):
    """Kepler (pow; the fp64 dopri5 instance at one trajectory per thread) and CubicMLP (tanh): no IEEE-basic oracle, but the
    persistent kernel and the stage kernels run the same device code, so they must agree bit for bit."""
    case = es.ALL[name]
    y0, s = _oracle(case, es.batch_size(case, _sms()))
    _check_premises(s, case)
    f = _builtin(case)
    a, sa = _solve(f, y0, case)
    b, sb = _solve(f, y0, case, fused_rhs="stages")
    assert sa["fused_rhs"] and sb["stage_rhs"]
    assert np.array_equal(a, b)
    assert sa["dt_next"] == sb["dt_next"]
    assert abs(sa["error_ratio"] - sb["error_ratio"]) <= _ratio_bar(case.dtype) * sb["error_ratio"]
    for st in (sa, sb):
        assert (st["n_accepted"], st["n_rejected"], st["nfe"]) == (s.stats.n_acc, s.stats.n_rej, s.stats.nfe)
    assert max_rel_err(a, s.sol) <= (1e-6 if case.dtype == "float64" else 1e-3)


# --------------------------------------------------------------------------------------------------
# the generic (per-stage) path
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["func", "func_graph", "stages"])
@pytest.mark.parametrize("name", [c.name for c in es.GENERIC])
def test_generic_path_is_bit_exact(name, variant):
    """The torch right-hand side called as func (eager, and replayed from a CUDA graph) and the built-in one evaluated
    inside the stage kernels; tsit5 includes its own dense output (k_emit_tsit5)."""
    case = es.ALL[name]
    y0, s = _oracle(case, es.batch_size(case, _sms()))
    _check_premises(s, case)
    if variant == "stages":
        got, st = _solve(_builtin(case), y0, case, fused_rhs="stages")
        assert st["stage_rhs"]
    else:
        f = PROBLEMS[case.problem](backend="torch", device=DEV)
        got, st = _solve(f, y0, case, cuda_graph=variant == "func_graph")
        assert not st["stage_rhs"] and st["cuda_graph"] == (variant == "func_graph")
    assert not st["fused_rhs"]
    _assert_exact(got, st, s, case.dtype)


@pytest.mark.parametrize("dtype", es.DTYPES)
def test_tuple_state_with_odd_segments_is_bit_exact(dtype):
    """Three components of 12 297, 2 002 and 21 elements (scalar tails in every kernel) with per-component tolerances."""
    y0, func, rtol, atol, t, first_step = es.tuple_case(dtype)
    s = es.oracle_solve(func, y0, t, "dopri5", rtol, atol, dict(es.OPTIONS, first_step=first_step))
    lo, lv = PROBLEMS["lorenz"](backend="torch", device=DEV), PROBLEMS["lv"](backend="torch", device=DEV)
    case = es.Case("tuple", None, "dopri5", dtype, False, None, rtol, atol, first_step, t, None, None)
    got, st = _solve(lambda tt, y: (lo(tt, y[0]), lv(tt, y[1]), lo(tt, y[2])), y0, case)
    _assert_exact(got, st, s, dtype)


def test_host_output_on_long_steps_is_bit_exact():
    """options={'host_output': pinned}: rows of steps longer than the persistent kernel buffers are written by the compute
    warps after the decision and streamed to the host; the generic path copies at the end."""
    case = es.ALL["lorenz-dopri5-f64-fwd-ncw3_partial"]
    y0, s = _oracle(case, es.batch_size(case, _sms()))
    host = torch.empty(s.sol.shape, dtype=torch.float64).pin_memory()
    for func, fused in ((_builtin(case), True), (PROBLEMS["lorenz"](backend="torch", device=DEV), False)):
        host.fill_(float("nan"))
        got, st = _solve(func, y0, case, host_output=host)
        assert st["fused_rhs"] == fused
        _assert_exact(got, st, s, case.dtype)
        _assert_exact(host.numpy(), st, s, case.dtype)


# --------------------------------------------------------------------------------------------------
# first_step=None: the initial-step heuristic against the oracle's
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["persistent", "generic"])
@pytest.mark.parametrize("name", [c.name for c in es.INITIAL])
def test_initial_step_matches_oracle(name, path):
    """dt_next = h0 * 2**-n_rej under the exact schedule, so it pins the initial step (misc.py:183-247) of k_init_* and of
    the persistent kernel's two reductions; pow and the order of the norms' sums differ from numpy in the last ulps."""
    case = es.ALL[name]
    y0, s = _oracle(case, es.batch_size(case, _sms()))
    _check_premises(s, case)
    assert s.dt_next == s.rec.dt[0] * 2.0 ** -s.stats.n_rej
    f = _builtin(case) if path == "persistent" else PROBLEMS[case.problem](backend="torch", device=DEV)
    got, st = _solve(f, y0, case, first_step=False)
    assert st["fused_rhs"] == (path == "persistent")
    assert (st["n_accepted"], st["n_rejected"], st["nfe"]) == (s.stats.n_acc, s.stats.n_rej, s.stats.nfe)
    assert abs(st["dt_next"] - s.dt_next) <= (1e-12 if case.dtype == "float64" else 1e-5) * s.dt_next
    assert max_rel_err(got, s.sol) <= (1e-6 if case.dtype == "float64" else 1e-3)


# --------------------------------------------------------------------------------------------------
# the opt-in bulk-copy finalize kernel (B2ODE_FINALIZE_BULK=1, read once per process: a child process)
# --------------------------------------------------------------------------------------------------
def _bulk_child():
    """Runs in the child: every BULK case exactly against the oracle with the module called as func (fused_rhs=False),
    a profile showing that k_rk_finalize_bulk ran, and a NaN in the part of the state past the last whole tile."""
    from torch.profiler import ProfilerActivity, profile
    for case in es.BULK:
        n = es.batch_size(case, _sms())
        y0, s = es.solve_case(case, n=n)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            got, st = _solve(_builtin(case), y0, case, fused_rhs=False)
        names = {e.key for e in prof.key_averages()}
        assert any("k_rk_finalize_bulk" in k for k in names), sorted(names)
        assert not st["fused_rhs"] and not st["stage_rhs"]
        _assert_exact(got, st, s, case.dtype)
        if n * 3 % 512:
            bad = y0.copy()
            flat = bad.reshape(-1)
            flat[(n * 3 // 512) * 512 + 4] = np.nan                # in the remainder the bulk kernel reads directly
            try:
                _solve(_builtin(case), bad, case, fused_rhs=False)
            except AssertionError as e:
                assert "non-finite values in state" in str(e)
            else:
                raise AssertionError("a NaN in the remainder was not reported")
        print("bulk ok:", case.name, n, flush=True)


def test_bulk_finalize_is_bit_exact():
    env = dict(os.environ, B2ODE_FINALIZE_BULK="1",
               PYTHONPATH=os.pathsep.join([ROOT, HERE, os.path.join(ROOT, "oracle")] +
                                          ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--bulk-child"], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("bulk ok:") == len(es.BULK), r.stdout


if __name__ == "__main__" and sys.argv[1:] == ["--bulk-child"]:
    _bulk_child()
