"""CPU: the references, bounds and tables of tests/rhs_cases.py, checked on themselves.

The torch modules' ``forward`` on the CPU must lie within each case's bound of the high-precision reference (a wrong
reference or a bound that is too tight fails here, without a GPU), the numpy restatements of Lorenz and Lotka-Volterra
must equal ``forward`` bit for bit, the tables must reach every edge they claim, and every solve case of
tests/test_exact_rhs_gpu.py must have rejections and decision margins on a numpy stand-in of its oracle."""
import numpy as np
import pytest

import exact_schedule as es
import np_ref
import rhs_cases as rc


def _bits(a):
    return a.view(np.int64 if a.dtype == np.float64 else np.int32)


@pytest.mark.parametrize("name", [c.name for c in rc.EVAL_CASES])
def test_forward_is_within_the_bound_of_the_reference(name):
    ev = rc.evaluation(name)
    ok, diff = rc.within_bound(ev.forward, ev)
    assert ev.regular.any() and ok.all(), "%d values outside the bound, worst %.3e over a bound of %.3e" % (
        int((~ok).sum()), float(diff[~ok].max()), float(ev.bound[ev.regular][~ok].max()))
    assert np.all(np.isfinite(ev.ref[ev.regular])) and np.all(np.isfinite(ev.forward[ev.regular]))
    if ev.exact is not None:
        assert np.array_equal(_bits(ev.exact), _bits(ev.forward))


@pytest.mark.parametrize("dtype", rc.DTYPES)
def test_bounds_are_a_few_ulps_not_a_tolerance(dtype):
    """The Kepler bound is 6 ulp (fp32) / 4 ulp (fp64) of the result; the CubicMLP bound at H = 50, std 0.1 stays below
    H + 10 ulps of the largest term: a kernel wrong by a few hundred ulps cannot pass."""
    eps = float(np.finfo(dtype).eps)
    ev = rc.evaluation("kepler-%s" % dtype[-2:])
    r = ev.regular
    acc = np.abs(ev.ref[r][:, 2:])
    assert np.all(ev.bound[r][:, 2:] <= (2 + rc.MATH_ULPS[dtype]["pow"]) * 1.01 * eps * acc)
    ev = rc.evaluation("mlp-h50-cube-std0.1-%s" % dtype[-2:])
    W2, b2 = rc.mlp_weights(ev.module, dtype)[2:]
    scale = np.abs(W2).sum(0) + np.abs(b2)
    assert np.all(ev.bound[ev.regular] <= 60 * eps * scale)


def test_parameter_sets_are_distinct_and_not_trivial():
    for p in [v for k, v in rc.LORENZ_PARAMS.items() if k != "default"] + list(rc.LV_PARAMS.values()):
        assert len(set(p)) == len(p)
        for v in p:
            assert v != 0 and abs(v) != 1 and np.log2(abs(v)) != round(np.log2(abs(v)))
            assert float(np.float32(v)) != v                       # the cast to a fp32 state changes it
    assert float(np.float32(rc.LORENZ_PARAMS["default"][1])) != rc.LORENZ_PARAMS["default"][1]
    assert len(rc.LORENZ_PARAMS) >= 3 and len(rc.LV_PARAMS) >= 2


@pytest.mark.parametrize("dtype", rc.DTYPES)
def test_kepler_table_reaches_its_edges(dtype):
    ev = rc.evaluation("kepler-%s" % dtype[-2:])
    y, f = ev.y, ev.forward
    tiny = np.finfo(dtype).tiny
    with np.errstate(all="ignore"):
        r2 = y[:, 0] * y[:, 0] + y[:, 1] * y[:, 1]
        r = np.sqrt(r2.astype(np.float64))
    reg = ev.regular
    assert reg[:136].all() and r[reg].min() < 2e-3 and r[reg].max() > 5e2
    for sx in (1, -1):
        for sy in (1, -1):
            assert np.any(reg & (sx * y[:, 0] > 0) & (sy * y[:, 1] > 0))
    assert np.any(reg & (y[:, 0] == 0) & (y[:, 1] != 0)) and np.any(reg & (y[:, 1] == 0) & (y[:, 0] != 0))
    assert np.any((r2 > 0) & (r2 < tiny)), "no subnormal r^2"
    assert np.any((r2 == 0) & ((y[:, 0] != 0) | (y[:, 1] != 0))), "no r^2 flushed to zero"
    assert np.any(np.isinf(r2) & np.isfinite(y).all(1)), "no overflowing r^2"
    cl = rc.classes(f[:, 2:])
    for code in range(7):
        assert np.any(cl == code), "class %d never occurs" % code
    origin = (y[:, 0] == 0) & (y[:, 1] == 0)
    assert origin.sum() == 4 and np.all(cl[origin] == 0)
    assert np.any(np.isnan(y)) and np.any(np.isinf(y))
    # a zero coordinate gives a zero of the opposite sign
    on_axis = reg & (y[:, 0] == 0)
    assert np.array_equal(np.signbit(f[on_axis, 2]), ~np.signbit(y[on_axis, 0]))


def test_mlp_tables_reach_their_edges():
    widths = {rc.EVAL[n].args[0] for n in rc.EVAL if rc.EVAL[n].kind == "mlp"}
    assert widths == set(rc.MLP_WIDTHS)
    for h in rc.MLP_WIDTHS:
        mine = [c.args for c in rc.EVAL_CASES if c.kind == "mlp" and c.args[0] == h]
        assert {a[1] for a in mine} == {True, False} and {a[2] for a in mine} == {0.1, 3.0}
    sat = nan32 = 0
    for c in rc.EVAL_CASES:
        if c.kind != "mlp":
            continue
        ev = rc.evaluation(c.name)
        W1, b1, W2, b2 = rc.mlp_weights(ev.module, c.dtype)
        assert np.all(b1 != 0) and np.all(b2 != 0) and W1.dtype == np.dtype(c.dtype)
        assert ev.regular[:32].all()
        sat += int(ev.saturated.sum())
        if c.dtype == "float32":
            assert ev.regular[36:].all() != c.args[1] and ev.regular[36:].any() != c.args[1]     # 1e13^3 = inf in fp32
            nan32 += int(np.isnan(ev.class_ref).any(1).sum())
            # the elementwise class reference is the same function: within the bound wherever a bound applies
            assert rc.within_bound(ev.class_ref, ev)[0].all()
        else:
            assert ev.regular.all()
        if c.args[2] == 3.0:
            assert ev.saturated.any(), c.name
    assert sat > 0 and nan32 > 0
    # the cross-dtype cases use the cast weights: a fp64-built module's fp32 image differs from it
    ev = rc.evaluation("mlp-h50-built-64-state-32")
    assert ev.module.W1.dtype.is_floating_point and str(ev.module.W1.dtype) == "torch.float64"
    w32 = rc.mlp_weights(ev.module, "float32")[0]
    assert np.any(w32.astype(np.float64) != ev.module.W1.detach().numpy())


# --------------------------------------------------------------------------------------------------
# the solve cases: premises on the numpy stand-in (exact for Lorenz and Lotka-Volterra)
# --------------------------------------------------------------------------------------------------
_ADAPTIVE = sorted({(c.system, c.method, c.dtype, c.reverse) for c in rc.SOLVE_CASES if c.path not in ("fixed", "rows")})


@pytest.mark.parametrize("system,method,dtype,reverse", _ADAPTIVE)
def test_solve_cases_have_rejections_and_margins(system, method, dtype, reverse):
    case = rc._sc(system, method, dtype, reverse, "persistent")
    y0, t, rtol, atol, opts = rc.solve_setup(case)
    s = es.oracle_solve(rc.numpy_rhs(case, rc.solve_module(case)), y0, t, method, rtol, atol, opts)
    p = es.premises(s, opts["first_step"])
    assert p["dyadic"] and p["decisions_agree"] and p["n_rej"] >= 1 and p["attempts"] <= es.MAX_ATTEMPTS, p
    assert p["margin"] > 10 * es.MARGIN[dtype], p


def test_solve_cases_cover_the_paths():
    kinds = {}
    for c in rc.SOLVE_CASES:
        kinds.setdefault((rc.solve_kind(c), c.path), set()).add((c.method, c.dtype, c.reverse))
    for kind in ("kepler", "mlp"):
        for dt in rc.DTYPES:
            for rev in (False, True):
                methods = [m for m in es.METHODS if (kind, m) != ("kepler", "bosh3")]
                assert {(m, dt, rev) for m in methods} <= kinds[kind, "persistent"]
                assert {(m, dt, rev) for m in methods + ["tsit5"]} <= kinds[kind, "stages"]
                assert {(m, dt, rev) for m in rc.FIXED_METHODS} <= kinds[kind, "fixed"]
                assert {(m, dt, rev) for m in ("dopri5", "dopri8")} <= kinds[kind, "rows"]
        assert kinds[kind, "stages_graph"]
    assert ("dopri8", "float64", False) in kinds["kepler", "stages_graph"]
    assert rc.SOLVE["mlp-h50-cube-rk4-32-fwd-fixed"]                     # BASELINE config 3's path
    for kind in ("lorenz", "lv"):
        assert {p for k, p in kinds if k == kind} == {"persistent", "stages", "rows", "fixed"}
    # the fixed grid interpolates: FIXED_STEP does not divide the output spacing
    y0, t, _, _, opts = rc.solve_setup(rc.SOLVE["kepler-rk4-64-fwd-fixed"])
    assert (t[1] - t[0]) / opts["step_size"] != round((t[1] - t[0]) / opts["step_size"])
    st = np_ref.Stats()
    np_ref.odeint(rc.numpy_rhs(rc.SOLVE["kepler-rk4-64-fwd-fixed"], None), y0, t, method="rk4", options=opts, stats=st)
    assert st.nfe > 4 * (len(t) - 1)
