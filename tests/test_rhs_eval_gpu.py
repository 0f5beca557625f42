"""GPU: every built-in right-hand side one evaluation at a time (``b2ode_rhs_eval``, i.e. k_rk_stage_rhs with no stage terms)
against the high-precision references and bounds of tests/rhs_cases.py: non-default parameters, non-zero biases, every
hidden width, saturated tanh, and the underflow / overflow / NaN / inf rows by class.  Lorenz and Lotka-Volterra must equal
their numpy restatement bit for bit.  The stage kernels with stage terms, the persistent, per-row and fixed-grid kernels
evaluate the same ``eval``; tests/test_exact_rhs_gpu.py pins them to this entry point bit for bit."""
import numpy as np
import pytest
import torch

import rhs_cases as rc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _bits(a):
    return a.view(np.int64 if a.dtype == np.float64 else np.int32)


def _same_bits(a, b):
    """Equal bit for bit, NaNs equal to NaNs whatever their payload."""
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(_bits(a)[~nan], _bits(b)[~nan])


def _eval(ev, y=None, **kw):
    y = ev.y if y is None else y
    return rc.device_eval(ev.module.to(DEV), torch.tensor(y, device=DEV), **kw).cpu().numpy()


@pytest.mark.parametrize("name", [c.name for c in rc.EVAL_CASES])
def test_evaluation_is_within_the_bound_of_the_reference(name):
    ev = rc.evaluation(name)
    with np.errstate(all="ignore"):
        got = _eval(ev)
    assert got.dtype == ev.y.dtype and got.shape == ev.y.shape
    ok, diff = rc.within_bound(got, ev)
    assert ok.all(), "%d values outside the bound, worst %.3e over a bound of %.3e" % (
        int((~ok).sum()), float(diff[~ok].max()), float(ev.bound[ev.regular][~ok].max()))
    if ev.exact is not None:
        assert np.array_equal(_bits(got), _bits(ev.exact))
    # class by class where no bound applies; for Kepler everywhere (the sign of a zero acceleration is determined)
    rows = np.ones(len(ev.y), dtype=bool) if rc.EVAL[name].kind == "kepler" else ~ev.regular
    assert np.array_equal(rc.classes(got[rows]), rc.classes(ev.class_ref[rows])), np.argwhere(
        rc.classes(got[rows]) != rc.classes(ev.class_ref[rows]))[:5]
    # the reversed system -f(-t, y): the exact negation, -0 included
    with np.errstate(all="ignore"):
        neg = _eval(ev, time_sign=-1.0)
    assert _same_bits(neg, -got)


@pytest.mark.parametrize("name", ["lorenz-a-32", "lv-b-64", "kepler-32", "kepler-64", "mlp-h127-cube-std3-32",
                                  "mlp-h128-lin-std3-64", "mlp-h1-lin-std0.1-64"])
def test_row_counts_and_misaligned_buffers(name):
    """1, 31, 33 and 257 rows (one partial block, one full block and a partial one), a batch beyond one pass of the
    evaluation kernel's grid (8 blocks of 256 rows per SM, one row more than a whole number of passes), and y / k_out one
    element into their allocations (4 or 8 bytes off a 16-byte boundary).  Rows are independent, so every row must equal
    bit for bit the table's evaluation of the same input, which the test above pins to the reference."""
    ev = rc.evaluation(name)
    with np.errstate(all="ignore"):
        base = _eval(ev)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    rng = np.random.default_rng(5)
    for n in (1, 31, 33, 257, 2 * 8 * 256 * sms + 1):
        idx = rng.integers(0, len(ev.y), n)
        for offset in (0, 1):
            with np.errstate(all="ignore"):
                got = _eval(ev, ev.y[idx], offset=offset)
            assert _same_bits(got, base[idx]), (n, offset)


@pytest.mark.parametrize("name", [c.name for c in rc.EVAL_CASES])
def test_evaluation_against_the_modules_cuda_forward(name):
    """rhs.py's claim about ``forward``: Lorenz, Lotka-Volterra and Kepler evaluate the same IEEE operations as the torch
    expressions, bit for bit (for Kepler that rests on torch's CUDA ``pow(x, 1.5)`` and the library's ``::pow`` being the
    same routine); CubicMLP's two products go through cuBLAS in ``forward``, so there both sides are held to the
    reference's bound instead."""
    ev = rc.evaluation(name)
    c = rc.EVAL[name]
    mod = (rc.mlp_as(ev.module, c.dtype) if c.kind == "mlp" else ev.module).to(DEV)
    with torch.no_grad(), np.errstate(all="ignore"):
        fwd = mod(torch.zeros((), device=DEV), torch.tensor(ev.y, device=DEV)).cpu().numpy()
        got = _eval(ev)
    if c.kind == "mlp":
        ok, diff = rc.within_bound(fwd, ev)
        assert ok.all(), float(diff[~ok].max())
        r = ev.regular
        assert np.all(np.abs(got[r].astype(np.float64) - fwd[r]) <= 2 * ev.bound[r] + np.spacing(np.abs(ev.ref[r])))
    else:
        assert _same_bits(got, fwd), "%d values differ from forward" % int((_bits(got) != _bits(fwd)).sum())
