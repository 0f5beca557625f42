"""CPU checks of tests/exact_backprop.py: the restated reverse sweep is the derivative of the oracle's solve, the cases'
schedules and sizes reach what tests/test_exact_backprop_gpu.py claims to test, the engine's recompute reproduces the
forward's stage inputs, and every wrong variant of the sweep is told apart from the real one."""
import numpy as np
import pytest
import torch

import exact_adjoint as ea
import exact_backprop as eb
import exact_schedule as es
import exact_stream as xs
import np_ref

# largest relative difference measured between the restatement and autograd through np_ref over all small cases:
# 1.8e-15 (fp64), 1.1e-6 (fp32); the bounds are 4x those
BOUND = {"float64": 7e-15, "float32": 4e-6}
SMALL = [c for c in eb.ALL.values() if c not in eb.LARGE]


def _autograd(case):
    """y0 and parameter gradients by autograd through np_ref.odeint on torch-CPU tensors (schedule held constant)."""
    module = eb.make_module(case)
    y0 = eb.initial_state(case)
    w = ea.loss_weights(case, y0)
    tdt = eb.TDT[case.dtype]
    ys0 = tuple(torch.tensor(v).requires_grad_(True) for v in y0)
    call = ea.tuple_call(module, eb.tensor_input(case))
    sol = np_ref.odeint(lambda t, y: call(torch.tensor(float(t), dtype=tdt), y), ys0, np.asarray(case.t, dtype=np.float64),
                        rtol=case.rtol, atol=case.atol, method=case.method, options=eb.options(case))
    loss = sum((s * torch.from_numpy(g)).sum() for s, g in zip(sol, w) if g is not None)
    ps = [p for p in module.parameters() if p.requires_grad]
    gs = torch.autograd.grad(loss, list(ys0) + ps, allow_unused=True)
    return gs[:len(ys0)], gs[len(ys0):]


def _rel(a, b):
    b = np.asarray(b)
    return float(np.max(np.abs(np.asarray(a) - b)) / max(float(np.max(np.abs(b))), 1e-300))


@pytest.mark.parametrize("name", sorted(c.name for c in SMALL))
def test_restatement_is_the_derivative(name):
    case = eb.small(eb.ALL[name])
    _, _, _, fwd, got = eb.solve_case(case)
    want_y, want_p = _autograd(case)
    assert len(got.params) == len(want_p)
    errs = [_rel(a, b.numpy()) for a, b in zip(got.y0, want_y)]
    errs += [_rel(a.numpy(), b.numpy()) for a, b in zip(got.params, want_p) if b is not None]
    assert max(errs) <= BOUND[case.dtype], (name, errs)


_FWD = {}


def _forward(name):
    if name not in _FWD:
        _FWD.clear()
        case = eb.ALL[name]
        module = eb.make_module(case)
        y0 = eb.initial_state(case)
        f = ea.numpy_func(module, case.dtype, eb.tensor_input(case))
        _FWD[name] = eb.forward(f, y0, case.t, case.method, case.rtol, case.atol, eb.options(case))
    return _FWD[name]


@pytest.mark.parametrize("name", sorted(c.name for c in SMALL))
def test_schedule_premises(name):
    """What a bit-exact comparison of the case proves: the exact schedule holds with margin, and the outputs fall inside
    steps, on step ends and leave steps without any (the large cases are checked by the GPU test on the same oracle)."""
    check_premises(eb.ALL[name], _forward(name))


def check_premises(case, fwd):
    if case.method in eb.ADAPTIVE:
        p = es.premises(fwd.solve, case.first_step)
        assert p["dyadic"] and p["decisions_agree"], p
        assert p["margin"] > es.MARGIN[case.dtype], p
        assert p["n_rej"] >= 1 and p["max_rows"] >= 1 and p["empty_steps"] >= 1 and p["rows_on_step_end"] >= 1, p
        assert p["others_non_dyadic"], p
    else:
        assert any(s.ends for s in fwd.steps), "no output on a step end"
        assert any(s.j1 - s.j0 > int(s.ends) for s in fwd.steps), "no output inside a step"
    if case in eb.GROWTH:
        # past 2 x 16 slots: the record is regrown twice, each time behind record launches already enqueued
        assert fwd.n_acc > 2 * eb.RECORD_SLOTS and fwd.n_rej >= 1, (fwd.n_acc, fwd.n_rej)


def check_recompute(case, fwd):
    """The backward pass's recompute of every stage input from y_n and the forward's k's equals the forward's Y_i."""
    T = np.dtype(case.dtype).type
    tab = eb.tableau(case.method)
    for st in fwd.steps:
        for i in range(1, tab.n_k):
            Y = eb.recompute(tab, case.method, st.y, st.k, i, st.dt, T)
            for a, b in zip(Y, st.Y[i]):
                assert np.array_equal(a.view(np.uint8), np.asarray(b).view(np.uint8)), (case.name, i)


@pytest.mark.parametrize("name", sorted(c.name for c in SMALL))
def test_recompute_reproduces_the_forward_stage_inputs(name):
    check_recompute(eb.ALL[name], _forward(name))


def test_rk4_combine_order_does_not_reproduce_the_forward():
    """The defect the rk4 fix removes, on the CPU alone: rk4's stage inputs formed by the combine of _FIXED_TAB (the
    backward's recompute before the fix) differ from the forward's in many elements, in both dtypes."""
    for dtype in es.DTYPES:
        case = eb.ALL["lorenz_forced-rk4-%s-fwd-4099" % ("f64" if dtype == "float64" else "f32")]
        fwd = _forward(case.name)
        T = np.dtype(dtype).type
        tab = eb.tableau("rk4")
        differ = [0, 0, 0]
        for st in fwd.steps:
            for i in range(1, 4):
                Y = eb.recompute(tab, "rk4", st.y, st.k, i, st.dt, T, rk4_combine=True)
                differ[i - 1] += int(np.sum(Y[0] != st.Y[i][0]))
        assert all(d > 0 for d in differ), differ


def test_geometry_at_132_sms():
    sms = xs.H100_SMS
    # k_bp_combine's vector path over 2+ grid-stride passes with a scalar tail: Lorenz at 600 001 rows (fp64) and
    # 750 001 (fp32), 3 n elements, odd
    for dt, rows in xs.LORENZ_ROWS.items():
        seg = xs.build_geom([3 * rows], dt, sms).segs[0]
        assert seg.vector and seg.passes >= 2 and seg.tail > 0, seg
    # ExactLinear at 4 300 x 128 = 550 400 fp64 elements: two vector passes over the grid
    seg = xs.build_geom([eb.LINEAR_ROWS * eb.LINEAR_DIM], "float64", sms).segs[0]
    assert seg.passes >= 2, seg
    # Tuple5: every component at a 16-byte aligned offset, odd lengths; the (1,) component has no whole 16-byte pack, so
    # it runs entirely on the scalar tail, and the (n, 3) components leave a tail of one element
    for dt in es.DTYPES:
        lens = [3 * eb.ROWS, 3 * eb.ROWS, 2 * ea.TUPLE_M, 2 * ea.TUPLE_M, 1]
        g = xs.build_geom(lens, dt, sms)
        assert g.segs[4].n // xs.vector_width(dt) == 0 and g.segs[4].tail == 1
        assert g.segs[0].tail > 0
    # k_bp_rhs: one thread per row over min(ceil(rows / 256), 8 SMs) blocks, two passes with a partial last one
    g = xs.row_grid(eb.BUILTIN_ROWS, sms)
    assert g.passes >= 2 and g.partial, g


@pytest.mark.parametrize("variant,name", [
    ("rk4_combine", "lorenz_forced-rk4-f64-fwd-4099"), ("rk4_combine", "lorenz_forced-rk4-f32-rev-4099"),
    ("tau_t0", "lorenz_forced-dopri5-f64-fwd-4099"), ("tau_t0", "lorenz_forced-rk4-f32-fwd-4099"),
    ("dt_f32", "lorenz_forced-rk4-f64-fwd-4099"), ("dt_f32", "lorenz_forced-euler-f64-rev-4099"),
    ("no_f1", "lorenz_forced-dopri5-f64-fwd-4099"), ("no_f1", "lorenz_forced-bosh3-f32-rev-4099")])
def test_negative_controls_differ_in_bits(variant, name):
    """Each wrong restatement differs from the real one, so the GPU test's equality can tell them apart."""
    case = eb.ALL[name]
    module = eb.make_module(case)
    y0 = eb.initial_state(case)
    w = ea.loss_weights(case, y0)
    fwd = _forward(name)
    real = eb.reverse_sweep(fwd, case.method, module, y0, w, eb.tensor_input(case), case.reverse)
    bad = eb.reverse_sweep(fwd, case.method, module, y0, w, eb.tensor_input(case), case.reverse, variant)
    same = all(np.array_equal(a, b) for a, b in zip(real.y0, bad.y0))
    same = same and all(torch.equal(a, b) for a, b in zip(real.params, bad.params))
    assert not same, (variant, name)
