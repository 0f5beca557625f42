"""CPU (no GPU needed): the premises of odeint_adjoint's fused_vjp option.

* The vector-Jacobian products of b2ode_rhs.cuh (``vjp`` of each built-in right-hand side), restated here in NumPy in the
  kernel's operation order, equal torch-CPU autograd of the module's ``forward`` bit for bit: Lorenz, Lotka-Volterra and
  Kepler, fp32 and fp64, non-default parameters, cotangents with exact zeros.  Kepler's restatement takes ``r^3`` and
  ``r2 ** 0.5`` from torch: torch's CPU ``pow`` is not correctly rounded, while its CUDA ``pow`` computes the exponent 0.5
  as the correctly rounded sqrt the kernel uses (the GPU test checks the kernel against CUDA autograd).
* CubicMLP's restated products (row by row, parameter cotangents summed over all rows) agree with fp64 autograd.
* The adjoint entry points reject malformed augmented layouts with one code and message, before any CUDA call.
* odeint_adjoint refuses every unsupported combination with ValueError before the forward solve.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import tfdiffeq_b200 as tfd
from tfdiffeq_b200 import _lib, tableaus

NP = {torch.float32: np.float32, torch.float64: np.float64}


def _autograd(mod, y, a):
    """(f, (-a)^T df/dy) from torch autograd of the module, as odeint_adjoint's default backward takes them."""
    y_ = y.clone().requires_grad_(True)
    f = mod(torch.zeros((), dtype=y.dtype), y_)
    g, = torch.autograd.grad(f, y_, -a)
    return f.detach().numpy(), g.numpy()


def vjp_lorenz(m, y, g, T):
    s, b, r = T(m.sigma), T(m.beta), T(m.rho)
    x, yy, z = y[:, 0], y[:, 1], y[:, 2]
    g0s = g[:, 0] * s
    gx = ((g[:, 2] * yy + g[:, 1] * (r - z)) + -g0s) + T(0)
    gy = ((g[:, 2] * x + -g[:, 1]) + g0s) + T(0)
    gz = ((-g[:, 2]) * b + -(g[:, 1] * x)) + T(0)
    return np.stack([gx, gy, gz], 1)


def vjp_lotka_volterra(m, y, g, T):
    a, b, c, d = T(m.a), T(m.b), T(m.c), T(m.d)
    x, z = y[:, 0], y[:, 1]
    gx = (((g[:, 1] * z) * d + ((-g[:, 0]) * z) * b) + g[:, 0] * a) + T(0)
    gz = ((g[:, 1] * (d * x) + g[:, 1] * (-c)) + (-g[:, 0]) * (b * x)) + T(0)
    return np.stack([gx, gz], 1)


def vjp_kepler(y, g, T, r3, sqrt_r2):
    x, yy = y[:, 0], y[:, 1]
    f2, f3 = (-x) / r3, (-yy) / r3
    g_r3 = (-g[:, 3]) * (f3 / r3) + (-g[:, 2]) * (f2 / r3)
    g_r2 = g_r3 * (T(1.5) * sqrt_r2)
    gx = ((-(g[:, 2] / r3) + g_r2 * x) + g_r2 * x) + T(0)
    gy = ((-(g[:, 3] / r3) + g_r2 * yy) + g_r2 * yy) + T(0)
    return np.stack([gx, gy, g[:, 0] + T(0), g[:, 1] + T(0)], 1)


def _rows(kind, n, dtype, seed):
    """Rows and cotangents: about one cotangent component in six, and whole rows, exactly zero."""
    rng = np.random.default_rng(seed)
    D = {"lorenz": 3, "lotka_volterra": 2, "kepler": 4}[kind]
    y = rng.standard_normal((n, D)) * 3.0
    if kind == "kepler":
        y[::97, :2] = [0.5, -0.25]
    a = rng.standard_normal((n, D)) * (rng.random((n, D)) >= 1.0 / 6)
    a[::11] = 0.0
    return torch.tensor(y, dtype=dtype), torch.tensor(a, dtype=dtype)


MODULES = {"lorenz": lambda: tfd.rhs.Lorenz(9.5, 2.5, 27.25),
           "lotka_volterra": lambda: tfd.rhs.LotkaVolterra(1.3, 0.7, 2.9, 1.1),
           "kepler": lambda: tfd.rhs.Kepler()}


def _bits(x):
    return x.view(np.uint32 if x.dtype == np.float32 else np.uint64)


@pytest.mark.parametrize("kind", ["lorenz", "lotka_volterra", "kepler"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_restated_vjp_equals_cpu_autograd_bit_for_bit(kind, dtype):
    T = NP[dtype]
    mod = MODULES[kind]()
    y, a = _rows(kind, 50000, dtype, 7)
    f, want = _autograd(mod, y, a)
    yn, g = y.numpy(), -a.numpy()
    with np.errstate(all="ignore"):
        if kind == "lorenz":
            got = vjp_lorenz(mod, yn, g, T)
        elif kind == "lotka_volterra":
            got = vjp_lotka_volterra(mod, yn, g, T)
        else:
            r2 = y[:, 0] * y[:, 0] + y[:, 1] * y[:, 1]
            got = vjp_kepler(yn, g, T, (r2 ** 1.5).numpy(), (r2 ** 0.5).numpy())
    assert got.dtype == T
    assert np.array_equal(_bits(got), _bits(want))
    assert (want == 0).any() and np.signbit(got[got == 0]).sum() == 0        # zeros come out +0, as autograd's do


def cubic_mlp_vjp(W1, b1, W2, b2, y, a, cube):
    """The kernel's CubicMLP products in fp64: per row f and g^T df/dy, g = -a; the parameter cotangents summed over rows
    (W1, b1, W2, b2 flattened)."""
    g = -a
    u = y ** 3 if cube else y
    z = np.tanh(u @ W1 + b1)
    delta = (g @ W2.T) * (1.0 - z * z)
    f = z @ W2 + b2
    gy = delta @ W1.T
    if cube:
        gy = gy * (3.0 * y * y)
    dparams = np.concatenate([(u.T @ delta).ravel(), delta.sum(0), (z.T @ g).ravel(), g.sum(0)])
    return f, gy, dparams


@pytest.mark.parametrize("hidden", [1, 50, 128])
@pytest.mark.parametrize("cube", [True, False])
def test_cubic_mlp_restatement_agrees_with_fp64_autograd(hidden, cube):
    gen = torch.Generator().manual_seed(hidden)
    mod = tfd.rhs.CubicMLP(hidden, cube=cube, std=0.5, dtype=torch.float64, generator=gen)
    with torch.no_grad():
        mod.b1.copy_(0.1 * torch.randn(hidden, generator=gen, dtype=torch.float64))
        mod.b2.copy_(torch.tensor([0.25, -0.5], dtype=torch.float64))
    rng = np.random.default_rng(hidden)
    y = torch.tensor(rng.standard_normal((4099, 2)))
    a = torch.tensor(rng.standard_normal((4099, 2)))
    y_ = y.clone().requires_grad_(True)
    fw = mod(0.0, y_)
    params = list(mod.parameters())
    grads = torch.autograd.grad(fw, [y_] + params, -a)
    want_p = torch.cat([p.reshape(-1) for p in grads[1:]]).numpy()
    W = [p.detach().numpy() for p in (mod.W1, mod.b1, mod.W2, mod.b2)]
    f, gy, dp = cubic_mlp_vjp(*W, y.numpy(), a.numpy(), cube)
    assert dp.shape == (5 * hidden + 2,)
    # fp64 rounding of sums over <= 4099 rows and <= 128 units
    np.testing.assert_allclose(f, fw.detach().numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(gy, grads[0].numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(dp, want_p, rtol=1e-11, atol=1e-11)


# --------------------------------------------------------------------------------------------------
# C ABI: one validation for both adjoint entry points
# --------------------------------------------------------------------------------------------------
BUF = [C.c_void_p(0x1000 * (i + 1)) for i in range(16)]


def _rhs(kind, params=(), data=BUF[0]):
    return _lib.RhsDesc(kind=kind, n_params=len(params), params=(C.c_double * 8)(*params), data=data, time_sign=-1.0)


def _adaptive_desc(lens):
    tab = tableaus.DOPRI5
    d = _lib.AdaptiveDesc()
    d.dtype, d.nseg, d.n_k, d.fsal = _lib.F64, len(lens), tab.n_k, 1
    for i, n in enumerate(lens):
        d.seg_len[i] = n
    for i, row in enumerate(tab.beta):
        for j, v in enumerate(row):
            d.beta[i][j] = v
    return d


def _both(rd, lens, ws_bytes=1 << 24):
    """(code, message) of b2ode_adjoint_rhs_eval and of b2ode_rk_stage_adjoint_rhs on a solver bound to fake buffers
    (nothing is dereferenced: every check runs before the first CUDA call)."""
    lib = _lib.lib
    ptrs = _lib.PtrArray(*[b.value for b in BUF[:_lib.MAXSEG]])
    la = _lib.LenArray(*(list(lens) + [0] * (_lib.MAXSEG - len(lens))))
    got = [(lib.b2ode_adjoint_rhs_eval(_lib.F64, C.byref(rd), BUF[1], la, ptrs, ptrs, BUF[2], ws_bytes, 132, None),
            lib.b2ode_last_error())]
    h = C.c_void_p()
    d = _adaptive_desc(lens)
    assert lib.b2ode_adaptive_create(C.byref(h), C.byref(d)) == 0
    try:
        b = _lib.AdaptiveBuffers()
        b.state, b.workspace, b.workspace_bytes, b.tstage, b.t_out, b.n_out = BUF[3].value, BUF[4].value, 1 << 30, \
            BUF[5].value, BUF[6].value, 2
        for i in range(len(lens)):
            b.y0[i], b.f0[i], b.ystage[i], b.out[i] = BUF[7].value, BUF[8].value, BUF[9].value, BUF[10].value
        assert lib.b2ode_adaptive_bind(h, C.byref(b), None) == 0
        got.append((lib.b2ode_rk_stage_adjoint_rhs(h, 1, ptrs, C.byref(rd), ptrs, BUF[2], ws_bytes), lib.b2ode_last_error()))
    finally:
        lib.b2ode_adaptive_destroy(h)
    return got


def test_adjoint_layout_validation_is_shared():
    lorenz = _rhs(_lib.RHS_LORENZ, (10.0, 8.0 / 3.0, 28.0))
    mlp = _rhs(_lib.RHS_CUBIC_MLP, (50.0, 1.0))
    cases = [(lorenz, (12, 12, 1), b"4 segments"),
             (lorenz, (12, 12, 1, 1, 1), b"4 segments"),
             (lorenz, (10, 10, 1, 1), b"state length 10 is not a multiple of the row size 3"),
             (lorenz, (12, 15, 1, 1), b"adj_y has 15 elements and y 12"),
             (lorenz, (12, 12, 2, 1), b"adj_t has 2 elements, not 1"),
             (lorenz, (12, 12, 1, 3), b"no trainable parameters"),
             (mlp, (12, 12, 1, 251), b"hidden width 50 takes 1 (frozen weights) or 252"),
             (_rhs(_lib.RHS_CUBIC_MLP, (50.0, 1.0), data=None), (12, 12, 1, 252), b"cubic-MLP"),
             (_rhs(9), (12, 12, 1, 1), b"unknown built-in right-hand side 9")]
    for rd, lens, text in cases:
        got = _both(rd, lens)
        if len(lens) != 4:
            got = got[1:]          # b2ode_adjoint_rhs_eval takes four lengths: only a solver can hold another count
        assert got == [(-1, got[0][1])] * len(got), (lens, got)
        assert text in got[0][1], (lens, got)
        la = _lib.LenArray(*(list(lens) + [0] * (_lib.MAXSEG - len(lens))))
        if len(lens) == 4:
            assert _lib.lib.b2ode_adjoint_rhs_workspace_bytes(C.byref(rd), la, 132) == 0


def test_adjoint_workspace_size_and_check():
    lib = _lib.lib
    mlp = _rhs(_lib.RHS_CUBIC_MLP, (50.0, 1.0))
    rows = 131072
    la = _lib.LenArray(2 * rows, 2 * rows, 1, 252)
    need = lib.b2ode_adjoint_rhs_workspace_bytes(C.byref(mlp), la, 132)
    assert need == 16 + 512 * 252 * 8                      # one row of P doubles per block; 512 blocks < 8 per SM
    la_big = _lib.LenArray(2 * 10 ** 6, 2 * 10 ** 6, 1, 252)
    assert lib.b2ode_adjoint_rhs_workspace_bytes(C.byref(mlp), la_big, 132) == 16 + 132 * 8 * 252 * 8
    la0 = _lib.LenArray(2 * rows, 2 * rows, 1, 1)
    assert lib.b2ode_adjoint_rhs_workspace_bytes(C.byref(mlp), la0, 132) == 16     # frozen weights: the ticket only
    got = _both(mlp, (2 * rows, 2 * rows, 1, 252), ws_bytes=need - 1)
    assert got == [(-3, got[0][1])] * 2 and b"workspace too small" in got[0][1], got


# --------------------------------------------------------------------------------------------------
# refusals: ValueError before the forward solve (CPU tensors: nothing could launch anyway)
# --------------------------------------------------------------------------------------------------
def refusal_cases(dev):
    y3 = torch.ones(4, 3, dtype=torch.float64, device=dev)
    y2 = torch.ones(4, 2, dtype=torch.float64, device=dev)
    t = torch.tensor([0.0, 0.1], device=dev)
    on = {"fused_vjp": True}
    lin = tfd.rhs.LinearODE(torch.eye(3, dtype=torch.float64)).to(dev)
    mlp_part = tfd.rhs.CubicMLP(8, dtype=torch.float64).to(dev)
    mlp_part.b2.requires_grad_(False)

    class MLPExtra(tfd.rhs.CubicMLP):
        def __init__(self):
            super(MLPExtra, self).__init__(8, dtype=torch.float64)
            self.extra = torch.nn.Parameter(torch.zeros(1, dtype=torch.float64))

    class LorenzTrainable(tfd.rhs.Lorenz):
        def __init__(self):
            super(LorenzTrainable, self).__init__()
            self.w = torch.nn.Parameter(torch.zeros(1, dtype=torch.float64))

    lor = tfd.rhs.Lorenz()
    return [("not a built-in", lin, y3, {}, dict(adjoint_options=on)),
            ("tuple state", lor, (y3,), {}, dict(adjoint_options=on)),
            ("partial rows", lor, torch.ones(4, 4, dtype=torch.float64, device=dev), {}, dict(adjoint_options=on)),
            ("fixed grid", lor, y3, {}, dict(adjoint_method="rk4", adjoint_options=on)),
            ("multistep", lor, y3, {}, dict(adjoint_method="adams", adjoint_options=on)),
            ("forward method inherited", lor, y3, dict(method="euler"), dict(adjoint_options=on)),
            ("fused_rhs False", lor, y3, {}, dict(adjoint_options=dict(on, fused_rhs=False))),
            ("fused_rhs stages", lor, y3, dict(method="dopri5"), dict(options=dict(on, fused_rhs="stages"))),
            ("shared_step_group", lor, y3, {}, dict(adjoint_options=dict(on, shared_step_group=object()))),
            ("independent_rows", lor, y3, {}, dict(adjoint_options=dict(on, independent_rows=True))),
            ("partially frozen", mlp_part, y2, {}, dict(adjoint_options=on)),
            ("extra parameters", MLPExtra().to(dev), y2, {}, dict(adjoint_options=on)),
            ("trainable built-in", LorenzTrainable().to(dev), y3, {}, dict(adjoint_options=on))], t


def test_fused_vjp_refusals_raise_before_the_forward_solve():
    cases, t = refusal_cases("cpu")
    for name, func, y0, fwd, kw in cases:
        if "options" in kw and "method" not in fwd:
            fwd = dict(fwd, method="dopri5")
        with pytest.raises(ValueError):
            tfd.odeint_adjoint(func, y0, t, **fwd, **kw)
    # a supported call passes the checks and reaches the solver, which has no CPU path
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        tfd.odeint_adjoint(tfd.rhs.Lorenz(), torch.ones(4, 3, dtype=torch.float64), t, adjoint_options={"fused_vjp": True})
