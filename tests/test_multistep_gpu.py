"""GPU: the multistep solvers (SURVEY 8f-4) -- b2ode_lincomb / b2ode_reduce against numpy, and fixed_adams /
explicit_adams / adams against the oracle at sizes beyond the golden fixtures (those run in test_parity_gpu.py)."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import np_ref
from problems import PROBLEMS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _ops(y0):
    from tfdiffeq_b200 import multistep, solvers
    seg = solvers._Segments(y0)
    return seg, multistep._Ops(seg)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("shapes", [[(1000, 3)], [(7,), (1031, 5), (2, 3, 4)], [(1 << 20,)]])
def test_lincomb_is_bit_exact(dtype, shapes):
    g = torch.Generator().manual_seed(sum(int(np.prod(s)) for s in shapes))
    y0 = tuple(torch.randn(*s, generator=g, dtype=dtype).to(DEV) for s in shapes)
    seg, ops = _ops(y0)
    npdt = np.float32 if dtype == torch.float32 else np.float64
    base = seg.new(); seg.fill(base, y0)
    terms = []
    for j in range(5):
        f = seg.new()
        seg.fill(f, tuple(torch.randn(*s, generator=g, dtype=dtype).to(DEV) for s in shapes))
        terms.append(f)
    coefs = [55 / 24, -59 / 24, 37 / 24, -9 / 24, 0.123456789]
    out = seg.new()
    ops.lincomb(out, base, 0.0371, terms, coefs)
    torch.cuda.synchronize()
    for s in range(seg.nseg):
        acc = None
        for c, tm in zip(coefs, terms):
            term = npdt(c) * seg.views(tm)[s].cpu().numpy()
            acc = term if acc is None else acc + term
        want = seg.views(base)[s].cpu().numpy() + npdt(0.0371) * acc
        assert np.array_equal(seg.views(out)[s].cpu().numpy(), want)
    # no base, unit scale, a single term with coefficient 1: a copy; a - b through coefficient -1
    ops.lincomb(out, None, 1.0, [terms[0]], [1.0])
    assert torch.equal(out, terms[0]) or all(torch.equal(a, b) for a, b in zip(seg.views(out), seg.views(terms[0])))
    ops.lincomb(out, terms[1], 1.0, [terms[2]], [-1.0])
    for a, b, c in zip(seg.views(out), seg.views(terms[1]), seg.views(terms[2])):
        assert torch.equal(a, b - c)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_reductions_match_numpy(dtype):
    from tfdiffeq_b200 import _lib
    g = torch.Generator().manual_seed(3)
    shapes = [(5,), (100003,), (64, 33)]
    y0 = tuple(torch.randn(*s, generator=g, dtype=dtype).to(DEV) for s in shapes)
    seg, ops = _ops(y0)
    npdt = np.float32 if dtype == torch.float32 else np.float64
    A, B = seg.new(), seg.new()
    seg.fill(A, y0)
    seg.fill(B, tuple(a + 1e-3 * torch.randn_like(a) for a in y0))
    r = ops.reduce(_lib.RED_ABSMAX2, A, B)
    for s in range(seg.nseg):
        assert r[s, 0] == float(seg.views(A)[s].abs().max()) and r[s, 1] == float(seg.views(B)[s].abs().max())
    for rep in range(3):                                              # the workspace cleans itself up between launches
        r = ops.reduce(_lib.RED_RATIO_SUMSQ, A, None, [0.37] * 3, [0.011, 0.5, 2.0])
        for s, tol in enumerate([0.011, 0.5, 2.0]):
            a = seg.views(A)[s].cpu().numpy()
            ratio = (npdt(0.37) * a) / npdt(tol)
            want = float(np.sum((ratio * ratio).astype(np.float64)))
            assert abs(r[s, 0] - want) <= 1e-12 * want
    r = ops.reduce(_lib.RED_NOT_CONVERGED, A, B, [1e-3] * 3, [1e-4] * 3)
    for s in range(seg.nseg):
        a, b = seg.views(A)[s].cpu().numpy(), seg.views(B)[s].cpu().numpy()
        want = int(np.sum(~(np.abs(a - b) < npdt(1e-4) + npdt(1e-3) * np.maximum(np.abs(a), np.abs(b)))))
        assert int(r[s, 0]) == want
    # NaN propagates through the maxima and fails the convergence test
    seg.views(A)[1].view(-1)[777] = float("nan")
    r = ops.reduce(_lib.RED_ABSMAX2, A, B)
    assert np.isnan(r[1, 0]) and not np.isnan(r[0, 0]) and not np.isnan(r[1, 1])
    r = ops.reduce(_lib.RED_NOT_CONVERGED, A, B, [1e-3] * 3, [10.0] * 3)
    assert int(r[1, 0]) == 1 and int(r[0, 0]) == 0


def _both(problem, y0, t, dtype="float64", pkw=None, **kw):
    pkw = pkw or {}
    fn = PROBLEMS[problem](backend="numpy", dtype=dtype, **pkw)
    ft = PROBLEMS[problem](backend="torch", dtype=dtype, device=DEV, **pkw)
    st = np_ref.Stats()
    ref = np_ref.odeint(fn, y0, t, stats=st, **kw)
    got = tfd().odeint(ft, torch.tensor(y0, device=DEV), torch.tensor(t), **kw)
    return ref, got.cpu().numpy(), st, dict(tfd().last_stats)


def _lorenz_y0(batch, dtype=np.float64):
    rng = np.random.default_rng(0)
    return (np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((batch, 3))).astype(dtype)


@pytest.mark.parametrize("method,options", [("explicit_adams", dict(max_order=5)), ("fixed_adams", None),
                                            ("fixed_adams", dict(max_order=6, max_iters=2))])
def test_fixed_adams_lorenz_4096_vs_oracle(method, options):
    t = np.arange(201) * 0.005
    kw = dict(method=method, rtol=1e-6, atol=1e-8)
    if options:
        kw["options"] = options
    ref, got, st, stats = _both("lorenz", _lorenz_y0(4096), t, **kw)
    assert stats["nfe"] == st.nfe
    assert np.max(np.abs(got - ref)) <= 1e-9 * np.max(np.abs(ref))


@pytest.mark.parametrize("method,options,dtype", [("explicit_adams", dict(max_order=5), "float64"),
                                                  ("fixed_adams", None, "float64"), ("fixed_adams", None, "float32")])
def test_fixed_adams_is_bit_exact_over_several_grid_passes(method, options, dtype):
    """fixed_adams / explicit_adams issue np_ref.FixedAdams's operations in its order: k_lincomb sums its terms left to
    right with the oracle's python-float coefficients, the start-up steps are k_fixed's 3/8-rule combines and the
    convergence test compares the same bits.  So at a size where k_lincomb and k_reduce loop over their grid (Lorenz,
    600 001 x 3 fp64 / 750 001 x 3 fp32: 3-4 vector passes and a scalar tail) the solution must equal the oracle's."""
    import exact_stream as xs
    rows = xs.LORENZ_ROWS[dtype]
    assert xs.build_geom([3 * rows], dtype, torch.cuda.get_device_properties(DEV).multi_processor_count).segs[0].passes >= 3
    kw = dict(method=method, rtol=1e-6, atol=1e-8) if dtype == "float64" else dict(method=method, rtol=1e-4, atol=1e-6)
    if options:
        kw["options"] = options
    ref, got, st, stats = _both("lorenz", xs.fixed_y0("lorenz", dtype, rows), xs.MULTISTEP_T, dtype=dtype, **kw)
    assert stats["nfe"] == st.nfe and stats.get("not_converged", 0) == getattr(st, "not_converged", 0)
    assert got.dtype == ref.dtype and np.array_equal(got, ref), np.max(np.abs(got - ref))


def test_fixed_adams_fp32_and_interior_outputs():
    # a grid coarser than t (step_size option): outputs inside a cell are linearly interpolated (solvers.py:106-115)
    t = np.linspace(0.0, 1.0, 38)
    ref, got, st, stats = _both("lorenz", _lorenz_y0(512, np.float32), t, dtype="float32", method="fixed_adams",
                                rtol=1e-4, atol=1e-6, options=dict(step_size=0.01))
    assert stats["nfe"] == st.nfe
    assert np.max(np.abs(got - ref)) <= 2e-4 * np.max(np.abs(ref))


def test_fixed_adams_reports_non_convergence_like_the_reference(capfd):
    # one functional iteration with a tolerance it cannot meet: the reference prints a warning per step and carries on
    t = np.linspace(0.0, 0.5, 26)
    ref, got, st, stats = _both("lorenz", _lorenz_y0(64), t, method="fixed_adams", rtol=1e-14, atol=1e-16,
                                options=dict(max_iters=1))
    err = capfd.readouterr().err
    assert "Functional iteration did not converge" in err
    assert stats["not_converged"] == st.not_converged > 0 and stats["nfe"] == st.nfe
    assert np.max(np.abs(got - ref)) <= 1e-9 * np.max(np.abs(ref))


@pytest.mark.parametrize("rtol,atol,options", [(1e-6, 1e-8, None), (1e-5, 1e-7, dict(max_order=5)), (1e-4, 1e-6, dict(max_order=2))])
def test_adams_lorenz_1024_vs_oracle(rtol, atol, options):
    t = np.arange(41) * 0.025
    kw = dict(method="adams", rtol=rtol, atol=atol)
    if options:
        kw["options"] = options
    ref, got, st, stats = _both("lorenz", _lorenz_y0(1024), t, **kw)
    # (identical step sequences; near the noise floor, rtol <~ 1e-8 on this chaotic system, the order-selection comparisons
    #  of adams.py:195-202 are decided by the last bits of the error norms and the sequences part ways -- not tested)
    assert (stats["n_accepted"], stats["n_rejected"], stats["nfe"]) == (st.n_acc, st.n_rej, st.nfe)
    assert np.max(np.abs(got - ref)) <= 1e-7 * np.max(np.abs(ref))


def test_adams_fp32_tuple_state_and_reverse_time():
    T = tfd()
    f = lambda t, y: (-y[0], -0.5 * y[1] * y[1])                      # noqa: E731
    y0 = (torch.linspace(1, 2, 300, device=DEV), torch.linspace(0.5, 1.5, 77, device=DEV).reshape(7, 11))
    t = torch.linspace(0.0, 1.0, 6)
    out = T.odeint(f, y0, t, method="adams", rtol=1e-5, atol=1e-7)
    ex0 = y0[0][None] * torch.exp(-t.to(DEV))[:, None]
    ex1 = y0[1][None] / (1 + 0.5 * y0[1][None] * t.to(DEV)[:, None, None])
    assert out[0].dtype == torch.float32 and out[0].shape == (6, 300) and out[1].shape == (6, 7, 11)
    # sanity only (parity is tested against the oracle above): the reference's scheme carries the PREDICTOR forward
    # (adams.py:211), so its global error sits well above the requested tolerance
    assert float((out[0] - ex0).abs().max()) < 5e-3 and float((out[1] - ex1).abs().max()) < 5e-3
    back = T.odeint(f, (out[0][-1], out[1][-1]), t.flip(0), method="adams", rtol=1e-5, atol=1e-7)
    assert float((back[0][-1] - y0[0]).abs().max()) < 2e-2
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        T.odeint(f, y0, t[:2], method="adams", options=dict(bogus=2))
    assert any("VariableCoefficientAdamsBashforth: Unexpected arguments {'bogus': 2}" in str(x.message) for x in w)


def test_adams_nonfinite_raises_instead_of_spinning():
    f = lambda t, y: y / (t - t)                                      # noqa: E731  inf / nan right away
    with pytest.raises(AssertionError):
        tfd().odeint(f, torch.ones(8, device=DEV, dtype=torch.float64), torch.tensor([0.0, 1.0]), method="adams")
