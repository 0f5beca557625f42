"""CPU: the refusals of odeint(..., options={'backprop': True}), the ctypes mirrors of the b2ode_bp_* ABI and its
argument checks (which run before any CUDA call), and a torch-CPU restatement of one reverse step -- stage sweep plus
dense-output VJP, the formulas of k_bp_combine / k_bp_dense -- against autograd through np_ref.runge_kutta_step and the
quartic interpolant."""
import ctypes as C
import re

import numpy as np
import pytest
import torch
import torch.nn as nn


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


class Lin(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Parameter(torch.tensor(0.5, dtype=torch.float64))

    def forward(self, t, y):
        return -self.a * y


@pytest.mark.parametrize("method,opts", [("tsit5", {}), ("adams", {}), ("fixed_adams", {}), ("explicit_adams", {}),
                                         ("dopri5", {"independent_rows": True}), ("dopri5", {"shared_step_group": object()}),
                                         ("dopri5", {"cuda_graph": True}), ("rk4", {"host_output": object()})])
def test_refusals_raise_before_anything_runs(method, opts):
    y0 = torch.ones(3, dtype=torch.float64, requires_grad=True)       # CPU tensors: any launch would fail differently
    t = torch.linspace(0, 1, 3, dtype=torch.float64)
    with pytest.raises(ValueError):
        tfd().odeint(Lin(), y0, t, method=method, options=dict(opts, backprop=True))


def test_time_gradients_are_refused():
    y0 = torch.ones(3, dtype=torch.float64, requires_grad=True)
    t = torch.linspace(0, 1, 3, dtype=torch.float64, requires_grad=True)
    with pytest.raises(ValueError):
        tfd().odeint(Lin(), y0, t, method="dopri5", options={"backprop": True})


def test_odeint_adjoint_refuses_the_key():
    y0 = torch.ones(3, dtype=torch.float64)
    t = torch.linspace(0, 1, 3, dtype=torch.float64)
    for kw in (dict(options={"backprop": True}), dict(adjoint_options={"backprop": True})):
        with pytest.raises(ValueError):
            tfd().odeint_adjoint(Lin(), y0, t, method="dopri5", **kw)


def _header():
    import os
    here = os.path.dirname(os.path.abspath(__file__))
    return open(os.path.join(os.path.dirname(here), "include", "b2ode.h")).read()


@pytest.mark.parametrize("name,cls", [("b2ode_bp_step", "BpStep"), ("b2ode_bp_record_desc", "BpRecordDesc"),
                                      ("b2ode_bp_combine_desc", "BpCombineDesc"), ("b2ode_bp_dense_desc", "BpDenseDesc"),
                                      ("b2ode_bp_rhs_desc", "BpRhsDesc")])
def test_ctypes_mirrors_follow_the_header(name, cls):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), _header(), re.S).group(1)
    fields = []
    for decl in re.sub(r"/\*.*?\*/", "", body, flags=re.S).split(";"):
        decl = decl.strip()
        if not decl:
            continue
        names = decl.split(None, 1)[1] if not decl.startswith("const") else decl.split(None, 2)[2]
        names = re.sub(r"\[[^]]*\]", "", names)
        for n in names.split(","):
            fields.append(re.match(r"\**\s*(\w+)", n.strip()).group(1))
    lib = tfd()._lib
    assert [f[0] for f in getattr(lib, cls)._fields_] == fields
    assert C.sizeof(lib.BpStep) == 40
    assert int(re.search(r"#define B2ODE_BP_MAXTERMS (\d+)", _header()).group(1)) == lib.BP_MAXTERMS


def test_bad_descriptors_are_rejected_without_the_device():
    lib = tfd()._lib
    d = lib.BpCombineDesc()
    assert lib.lib.b2ode_bp_combine(None) == -1
    d.dtype, d.nseg, d.nterms = 7, 1, 1
    assert lib.lib.b2ode_bp_combine(C.byref(d)) == -1 and b"dtype" in lib.lib.b2ode_last_error()
    d.dtype, d.nterms = 1, 0
    assert lib.lib.b2ode_bp_combine(C.byref(d)) == -1 and b"nterms" in lib.lib.b2ode_last_error()
    d.nterms, d.seg_len[0] = 1, 8
    assert lib.lib.b2ode_bp_combine(C.byref(d)) == -1 and b"null" in lib.lib.b2ode_last_error()
    e = lib.BpDenseDesc()
    e.dtype, e.nseg, e.kind, e.n_k = 1, 1, 5, 7
    assert lib.lib.b2ode_bp_dense(C.byref(e)) == -1 and b"kind" in lib.lib.b2ode_last_error()
    e.kind = 0
    assert lib.lib.b2ode_bp_dense(C.byref(e)) == -1 and b"required" in lib.lib.b2ode_last_error()
    e.step, e.t_out, e.k_mask = 8, 8, 1 << 9
    assert lib.lib.b2ode_bp_dense(C.byref(e)) == -1 and b"k_mask" in lib.lib.b2ode_last_error()
    assert lib.lib.b2ode_bp_record(None, C.byref(lib.BpRecordDesc())) != 0
    r = lib.BpRhsDesc()
    assert lib.lib.b2ode_bp_rhs(None) == -1
    r.dtype, r.rhs.kind, r.n = 1, 9, 6
    assert lib.lib.b2ode_bp_rhs(C.byref(r)) == -1 and b"unknown built-in" in lib.lib.b2ode_last_error()
    r.rhs.kind, r.rhs.n_params, r.n = lib.RHS_LORENZ, 3, 7
    assert lib.lib.b2ode_bp_rhs(C.byref(r)) == -1 and b"multiple" in lib.lib.b2ode_last_error()
    r.n, r.n_params = 6, 4
    assert lib.lib.b2ode_bp_rhs(C.byref(r)) == -1 and b"n_params" in lib.lib.b2ode_last_error()
    r.n_params, r.mode = 0, 3
    assert lib.lib.b2ode_bp_rhs(C.byref(r)) == -1 and b"mode" in lib.lib.b2ode_last_error()
    r.mode = lib.BP_VJP
    assert lib.lib.b2ode_bp_rhs(C.byref(r)) == -1 and b"required" in lib.lib.b2ode_last_error()
    r.step, r.t_scalar, r.y, r.out = 8, 8, 8, 8
    assert lib.lib.b2ode_bp_rhs(C.byref(r)) == -1 and b"cotangent" in lib.lib.b2ode_last_error()


def test_bp_rhs_workspace_bytes():
    lib = tfd()._lib
    rd = lib.RhsDesc(kind=lib.RHS_CUBIC_MLP, n_params=2, data=8)
    rd.params[0], rd.params[1] = 50, 1
    P = 5 * 50 + 2
    for rows, sm in ((1, 132), (3000, 132), (10 ** 6, 132), (10 ** 6, 0)):
        grid = min(max((rows + 255) // 256, 1), (sm or 132) * 8)
        assert lib.lib.b2ode_bp_rhs_workspace_bytes(C.byref(rd), 2 * rows, P, sm) == 16 + grid * P * 8
    assert lib.lib.b2ode_bp_rhs_workspace_bytes(C.byref(rd), 2 * 10, 7, 132) == 0          # not 0 or 5 H + 2
    lz = lib.RhsDesc(kind=lib.RHS_LORENZ, n_params=3)
    assert lib.lib.b2ode_bp_rhs_workspace_bytes(C.byref(lz), 30, 0, 132) == 16
    assert lib.lib.b2ode_bp_rhs_workspace_bytes(C.byref(lz), 31, 0, 132) == 0


def test_partially_frozen_builtins_are_refused():
    m = tfd().rhs.CubicMLP(8, dtype=torch.float64)
    m.b2.requires_grad_(False)
    y0 = torch.ones(4, 2, dtype=torch.float64, requires_grad=True)
    t = torch.linspace(0, 1, 3, dtype=torch.float64)
    with pytest.raises(ValueError):
        tfd().odeint(m, y0, t, method="dopri5", options={"backprop": True})
    lz = tfd().rhs.Lorenz()
    lz.extra = nn.Parameter(torch.ones(2, dtype=torch.float64))
    with pytest.raises(ValueError):
        tfd().odeint(lz, torch.ones(4, 3, dtype=torch.float64), t, method="dopri5", options={"backprop": True})


def _restated_reverse_step(tab, f, t0, dt, y0, gy1, outs):
    """One reverse step as the engine forms it, f0 an input: returns (lambda_n, mu_0).  mu_0 is what the engine applies
    J^T to at y_n (FSAL) or carries into the previous step's last k (adaptive Heun)."""
    s = tab.n_k
    # lambda (the cotangent of y1) enters k_j through y1's weights: for FSAL y1 is the last stage input (row s - 2 of
    # beta), otherwise y1 = y0 + sum dt b_j k_j
    lam_coef = tab.beta[s - 2] if tab.fsal else tab.c_sol
    k = [None] * s
    k[0] = outs["f0"]
    Y, calls = [], []
    for i in range(s - 1):
        yi = y0 + sum(dt * tab.beta[i][j] * k[j] for j in range(i + 1))
        leaf = yi.detach().requires_grad_(True)
        with torch.enable_grad():
            ki = f(t0 + tab.alpha[i] * dt, leaf)
        k[i + 1] = ki.detach()
        calls.append((leaf, ki))
    # dense VJP (k_bp_dense): outputs at x, cotangents g
    GA = sum(g * x ** 4 for x, g in outs["gx"])
    GB = sum(g * x ** 3 for x, g in outs["gx"])
    GC = sum(g * x ** 2 for x, g in outs["gx"])
    GD = sum(g * x for x, g in outs["gx"])
    G1 = sum(g for x, g in outs["gx"])
    gmid = 16 * GA - 32 * GB + 16 * GC
    g0 = 18 * GB - 8 * GA - 11 * GC + G1 + gmid
    lam = gy1 + (14 * GB - 8 * GA - 5 * GC)
    mu = [dt * tab.c_mid[j] * gmid for j in range(s)]
    mu[0] = mu[0] + dt * (5 * GB - 2 * GA + GD - 4 * GC)
    mu[s - 1] = mu[s - 1] + dt * (2 * GA - 3 * GB + GC)
    # stage sweep (k_bp_combine + J^T)
    nu = [None] * (s - 1)
    for i in range(s - 2, -1, -1):
        j = i + 1
        m = mu[j] + sum(dt * tab.beta[l][j] * nu[l] for l in range(j, s - 1))
        if j < len(lam_coef):
            m = m + dt * lam_coef[j] * lam
        leaf, ki = calls[i]
        nu[i] = torch.autograd.grad(ki, leaf, m)[0]
    mu0 = mu[0] + sum(dt * tab.beta[l][0] * nu[l] for l in range(s - 1)) + dt * lam_coef[0] * lam
    return g0 + sum(nu) + lam, mu0


@pytest.mark.parametrize("name", ["dopri5", "bosh3", "dopri8", "adaptive_heun"])
def test_restated_reverse_step_equals_autograd_through_the_oracle(name):
    import np_ref
    tab = tfd().tableaus.TABLEAUS[name]
    ntab = np_ref.ADAPTIVE[name]
    assert tab.fsal == (name != "adaptive_heun")
    A = torch.tensor([[-0.3, 1.1, 0.2], [-0.9, -0.1, 0.4], [0.3, -0.5, -0.2]], dtype=torch.float64)

    def f(t, y):
        return torch.tanh(y @ A) * (1.0 + 0.3 * float(t))
    y0 = torch.tensor([0.4, -0.7, 1.2], dtype=torch.float64, requires_grad=True)
    f0 = f(0.1, y0).detach().requires_grad_(True)
    t0, dt = 0.1, 0.37
    xs = [0.25, 0.8, 1.0]
    g = torch.Generator().manual_seed(3)
    gs = [torch.randn(3, generator=g, dtype=torch.float64) for _ in xs]
    gy1 = torch.randn(3, generator=g, dtype=torch.float64)
    # autograd through the oracle's step and interpolant
    with torch.enable_grad():
        y1, f1, _, k = np_ref.runge_kutta_step(lambda t, y: (f(t, y[0]),), (y0,), (f0,), t0, dt, ntab)
        coeffs = np_ref.interp_fit_rk((y0,), y1, k, dt, ntab)
        loss = (y1[0] * gy1).sum()
        for x, gg in zip(xs, gs):
            loss = loss + (np_ref.interp_evaluate(coeffs, t0, t0 + dt, t0 + x * dt)[0] * gg).sum()
        want_y0, want_f0 = torch.autograd.grad(loss, (y0, f0))
    got_y0, got_mu0 = _restated_reverse_step(tab, f, t0, dt, y0.detach(), gy1,
                                             dict(f0=f0.detach(), gx=list(zip(xs, gs))))
    assert torch.allclose(got_y0, want_y0, rtol=1e-12, atol=1e-12)
    assert torch.allclose(got_mu0, want_f0, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("ends", [False, True])
def test_restated_fixed_grid_step_equals_autograd(ends):
    """One fixed-grid rk4 step (3/8 rule, rk_common.py:73-81) with outputs by linear interpolation (solvers.py:106-115):
    the linear rule of k_bp_dense plus the stage sweep with f0 an evaluation at y_n, against autograd."""
    from tfdiffeq_b200.backprop import _FIXED_TAB
    beta, c_sol = _FIXED_TAB["rk4"]
    A = torch.tensor([[-0.3, 1.1], [-0.9, -0.1]], dtype=torch.float64)

    def f(t, y):
        return torch.tanh(y @ A) * (1.0 + 0.3 * t)
    t0, dt = 0.2, 0.3
    taus = [t0, t0 + dt / 3, t0 + 2 * dt / 3, t0 + dt]
    y0 = torch.tensor([0.4, -0.7], dtype=torch.float64, requires_grad=True)
    g = torch.Generator().manual_seed(5)
    ts = [t0 + 0.1, t0 + 0.25] + ([t0 + dt] if ends else [])
    gs = [torch.randn(2, generator=g, dtype=torch.float64) for _ in ts]
    gy1 = torch.randn(2, generator=g, dtype=torch.float64)
    with torch.enable_grad():
        k1 = f(taus[0], y0)
        k2 = f(taus[1], y0 + dt * k1 / 3)
        k3 = f(taus[2], y0 + dt * (-k1 / 3 + k2))
        k4 = f(taus[3], y0 + dt * (k1 - k2 + k3))
        y1 = y0 + (k1 + 3 * k2 + 3 * k3 + k4) * (dt / 8)
        loss = (y1 * gy1).sum()
        for i, (tj, gj) in enumerate(zip(ts, gs)):
            out = y1 if (ends and i == len(ts) - 1) else y0 + ((y1 - y0) / dt) * (tj - t0)
            loss = loss + (out * gj).sum()
        (want,) = torch.autograd.grad(loss, y0)
    # the engine's formulas: linear dense rule, then the sweep with every k_j an evaluation
    yd = y0.detach()
    a0, lam = torch.zeros(2, dtype=torch.float64), gy1.clone()
    for i, (tj, gj) in enumerate(zip(ts, gs)):
        if ends and i == len(ts) - 1:
            lam = lam + gj
            continue
        q = (tj - t0) / dt
        lam, a0 = lam + gj * q, a0 + gj * (1 - q)
    # the stage inputs as the forward forms them (fixed_eval's B2ODE_OP_RK4_S2..S4), which the recompute reproduces
    stage = (lambda k: yd, lambda k: yd + dt * k[0] / 3, lambda k: yd + dt * (k[0] / -3 + k[1]),
             lambda k: yd + dt * ((k[0] - k[1]) + k[2]))
    ks, calls = [], []
    for i in range(4):
        Y = stage[i](ks)
        leaf = Y.clone().requires_grad_(True)
        with torch.enable_grad():
            kk = f(taus[i], leaf)
        ks.append(kk.detach())
        calls.append((leaf, kk))
    nu = [None] * 4
    for j in range(3, -1, -1):
        m = dt * c_sol[j] * lam + sum(dt * beta[l - 1][j] * nu[l] for l in range(j + 1, 4))
        leaf, kk = calls[j]
        nu[j] = torch.autograd.grad(kk, leaf, m)[0]
    got = a0 + sum(nu) + lam
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
