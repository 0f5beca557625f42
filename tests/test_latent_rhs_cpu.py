"""CPU: rhs.LatentODEFunc (examples/latent_ode.py's network as a built-in right-hand side) without a GPU.

The constructor's refusals, the packed weight layout, the ABI constant, the library's description checks and workspace
sizes for B2ODE_RHS_LATENT_MLP (all of which run before any CUDA call), the refusals of partly frozen weights, and the
60-digit reference with its error bound (tests/latent_cases.py), checked against torch-CPU forward and autograd."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import latent_cases as lc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tfd():
    import tfdiffeq_b200
    import tfdiffeq_b200.backprop  # noqa: F401  (imported on first use by odeint)
    return tfdiffeq_b200


def _desc(H, data=8, n_params=1):
    lib = tfd()._lib
    rd = lib.RhsDesc(kind=lib.RHS_LATENT_MLP, n_params=n_params, data=data)
    rd.params[0] = H
    return rd


def test_constructor_refusals():
    L = tfd().rhs.LatentODEFunc
    for kw in (dict(latent_dim=3), dict(latent_dim=8), dict(hidden=0), dict(hidden=33), dict(hidden=-1)):
        with pytest.raises(ValueError):
            L(**kw)
    m = L(hidden=1)
    assert m.hidden == 1 and m.rhs_params() == [1.0]
    assert L(hidden=32).rhs_params() == [32.0]


def test_default_init_is_seeded_and_within_fan_in_bounds():
    L = tfd().rhs.LatentODEFunc
    a = L(hidden=20, generator=torch.Generator().manual_seed(3))
    b = L(hidden=20, generator=torch.Generator().manual_seed(3))
    c = L(hidden=20, generator=torch.Generator().manual_seed(4))
    for pa, pb, pc in zip(a.parameters(), b.parameters(), c.parameters()):
        assert torch.equal(pa, pb) and not torch.equal(pa, pc)
    for fc in (a.fc1, a.fc2, a.fc3):
        lim = 1.0 / np.sqrt(fc.in_features)
        for p in (fc.weight.detach(), fc.bias.detach()):
            assert float(p.abs().max()) <= lim and float(p.abs().max()) > 0.5 * lim
    assert isinstance(a.fc1, torch.nn.Linear) and a.fc1.weight.shape == (20, 4) and a.fc3.weight.shape == (4, 20)
    assert a.fc1.weight.dtype == torch.float32
    assert L(dtype=torch.float64).fc2.bias.dtype == torch.float64


def test_rhs_data_layout():
    m = tfd().rhs.LatentODEFunc(hidden=7, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    d = m.rhs_data(torch.float64, "cpu")
    H = 7
    assert d.numel() == H * H + 10 * H + 4 and d.is_contiguous()
    off = 0
    for p in (m.fc1.weight, m.fc1.bias, m.fc2.weight, m.fc2.bias, m.fc3.weight, m.fc3.bias):
        assert torch.equal(d[off:off + p.numel()], p.detach().reshape(-1))
        off += p.numel()
    # the flattened parameter order the kernels use for the gradients is the module's own
    assert [n for n, _ in m.named_parameters()] == list(m.trainable_weights[1])
    assert m.rhs_data(torch.float32, "cpu").dtype == torch.float32


def test_forward_takes_stacked_rows():
    m = tfd().rhs.LatentODEFunc(hidden=5, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    y = torch.randn(3, 8, dtype=torch.float64)
    f = m(torch.tensor(0.0), y)
    assert f.shape == y.shape
    # row by row the same function (BLAS may block the two shapes differently: equal to rounding)
    assert torch.allclose(f[:, 4:], m(torch.tensor(0.0), y[:, 4:].contiguous()), rtol=1e-14, atol=1e-14)


def test_abi_constant_matches_header():
    with open(os.path.join(ROOT, "include", "b2ode.h")) as fh:
        h = fh.read()
    assert int(re.search(r"#define B2ODE_RHS_LATENT_MLP (\d+)", h).group(1)) == tfd()._lib.RHS_LATENT_MLP == 4
    assert len({tfd()._lib.RHS_LORENZ, tfd()._lib.RHS_LOTKA_VOLTERRA, tfd()._lib.RHS_CUBIC_MLP, tfd()._lib.RHS_KEPLER,
                tfd()._lib.RHS_LATENT_MLP}) == 5


@pytest.mark.parametrize("H", [1, 20, 32])
def test_workspace_sizes_and_parameter_count(H):
    lib = tfd()._lib
    L = lib.lib
    P = H * H + 10 * H + 4
    rd = _desc(H)
    rows = 131072
    la = lib.LenArray(4 * rows, 4 * rows, 1, P)
    assert L.b2ode_adjoint_rhs_workspace_bytes(C.byref(rd), la, 132) == 16 + 512 * P * 8
    assert L.b2ode_adjoint_rhs_workspace_bytes(C.byref(rd), lib.LenArray(4 * rows, 4 * rows, 1, 1), 132) == 16
    assert L.b2ode_adjoint_rhs_workspace_bytes(C.byref(rd), lib.LenArray(4 * rows, 4 * rows, 1, P - 1), 132) == 0
    assert b"latent-MLP of hidden width %d takes 1 (frozen weights) or %d" % (H, P) in L.b2ode_last_error()
    assert L.b2ode_bp_rhs_workspace_bytes(C.byref(rd), 4 * rows, P, 132) > 16
    assert L.b2ode_bp_rhs_workspace_bytes(C.byref(rd), 4 * rows, 5 * H + 2, 132) == 0
    for n_rows, sm in ((1, 132), (3000, 132), (10 ** 6, 132)):
        grid = min(max((n_rows + 127) // 128, 1), sm * 8)
        assert L.b2ode_rows_bp_workspace_bytes(C.byref(rd), n_rows, P, sm) == 16 + grid * P * 8
        assert L.b2ode_rows_bp_workspace_bytes(C.byref(rd), n_rows, 0, sm) == 16
    assert L.b2ode_rows_bp_workspace_bytes(C.byref(rd), 10, P + 1, 132) == 0
    # rows of 4: a state that is not whole rows is refused
    assert L.b2ode_bp_rhs_workspace_bytes(C.byref(rd), 4 * 10 + 2, 0, 132) == 0
    assert b"multiple of the row size 4" in L.b2ode_last_error()


def test_description_refusals():
    lib = tfd()._lib
    L = lib.lib
    la = lib.LenArray(40, 40, 1, 1)
    for rd in (_desc(0), _desc(33), _desc(20, data=None), _desc(20, n_params=0), _desc(float("nan"))):
        assert L.b2ode_adjoint_rhs_workspace_bytes(C.byref(rd), la, 132) == 0
        assert b"latent-MLP right-hand side needs {H in [1, 32]} and its weights" in L.b2ode_last_error()
        assert L.b2ode_rows_bp_workspace_bytes(C.byref(rd), 10, 0, 132) == 0
        assert L.b2ode_bp_rhs_workspace_bytes(C.byref(rd), 40, 0, 132) == 0
    for H in (1, 32):
        assert L.b2ode_adjoint_rhs_workspace_bytes(C.byref(_desc(H)), la, 132) == 16


def _partly_frozen(which):
    m = tfd().rhs.LatentODEFunc(hidden=4)
    getattr(getattr(m, which[0]), which[1]).requires_grad_(False)
    return m


@pytest.mark.parametrize("which", [("fc1", "weight"), ("fc2", "bias"), ("fc3", "bias")])
def test_partly_frozen_weights_are_refused(which):
    t = tfd()
    m = _partly_frozen(which)
    y0 = torch.zeros(8, 4)
    msg = r"LatentODEFunc whose six weights \(fc1.weight, fc1.bias, fc2.weight, fc2.bias, fc3.weight, fc3.bias\) are all " \
          r"trainable or all frozen"
    with pytest.raises(ValueError, match="fused_vjp supports a " + msg):
        t.adjoint._check_fused_vjp(m, y0, None, {})
    with pytest.raises(ValueError, match="backprop differentiates a " + msg):
        t.backprop.check_builtin(m, {})
    t.backprop.check_builtin(m, {"fused_rhs": False})          # the generic path takes any parameters


def test_extra_parameters_are_refused_and_whole_sets_accepted():
    t = tfd()
    m = t.rhs.LatentODEFunc(hidden=4)
    y0 = torch.zeros(8, 4)
    t.adjoint._check_fused_vjp(m, y0, None, {})
    t.backprop.check_builtin(m, {})
    for p in m.parameters():
        p.requires_grad_(False)
    t.adjoint._check_fused_vjp(m, y0, None, {})
    t.backprop.check_builtin(m, {})
    m.extra = torch.nn.Parameter(torch.zeros(1))
    with pytest.raises(ValueError, match="six weights"):
        t.adjoint._check_fused_vjp(m, y0, None, {})
    with pytest.raises(ValueError, match="six weights"):
        t.backprop.check_builtin(m, {})


def test_a_weight_replaced_by_a_buffer_is_refused():
    t = tfd()
    for m in (t.rhs.LatentODEFunc(hidden=4), t.rhs.CubicMLP(4)):
        name = m.trainable_weights[1][0].split(".")
        owner = m if len(name) == 1 else getattr(m, name[0])
        w = getattr(owner, name[-1]).detach().clone()
        delattr(owner, name[-1])
        owner.register_buffer(name[-1], w)
        assert not t.rhs.weights_all_or_none(m)
        with pytest.raises(ValueError, match="all trainable or all frozen"):
            t.adjoint._check_fused_vjp(m, torch.zeros(8, m.dim), None, {})
        with pytest.raises(ValueError, match="all trainable or all frozen"):
            t.backprop.check_builtin(m, {})


def test_fused_vjp_message_names_the_class():
    t = tfd()
    with pytest.raises(ValueError, match="CubicMLP or LatentODEFunc"):
        t.adjoint._check_fused_vjp(torch.nn.Linear(4, 4), torch.zeros(8, 4), None, {})


def test_trainable_per_row_adjoint_is_refused():
    t = tfd()
    m = t.rhs.LatentODEFunc(hidden=4)
    with pytest.raises(ValueError, match="frozen parameters"):
        t.adjoint._check_independent_rows(m, "dopri5", "dopri5", 1e-7, 1e-9)


@pytest.mark.parametrize("H,std,dtype", [(1, 0.1, "float64"), (20, 0.1, "float32"), (20, 3.0, "float64"),
                                         (32, 3.0, "float32"), (32, 0.1, "float64")])
def test_reference_bound_holds_for_torch_cpu(H, std, dtype):
    tdt = torch.float64 if dtype == "float64" else torch.float32
    mod = lc.module(H, std, tdt, seed=H)
    y, g = lc.rows(24, std, seed=7 * H, dtype=np.dtype(dtype))
    ref = lc.reference(mod, y, g)
    bf, bg = lc.bound(mod, y, g, ref, dtype)
    f, gy = lc.torch_eval(mod, y, g, dtype=tdt)
    assert np.all(np.abs(f - ref["f"]) <= bf), float(np.max(np.abs(f - ref["f"]) / bf))
    assert np.all(np.abs(gy - ref["gy"]) <= bg), float(np.max(np.abs(gy - ref["gy"]) / bg))
    # both elu branches occur in both layers (in the wide networks), and the bound is a few ulps of the sums, not a tolerance
    assert (ref["a1"] > 0).any() and (ref["a1"] < 0).any()
    if H > 1:
        assert (ref["a2"] > 0).any() and (ref["a2"] < 0).any()
    eps = float(np.finfo(dtype).eps)
    W3 = np.abs(lc.weights(mod)[4])
    assert np.all(bf <= 20 * (H + 10) * eps * (np.abs(ref["z2"]) @ W3.T + np.abs(lc.weights(mod)[5]) + 1))


@pytest.mark.parametrize("method,dtype,reverse", lc.SOLVE_CASES)
def test_exact_solve_cases_have_rejections_and_margins(method, dtype, reverse):
    """Every exact-schedule case of tests/test_latent_exact_gpu.py, on the torch-CPU stand-in of its oracle: power-of-two
    steps, at least one rejection and a margin on every accept decision (the GPU test re-checks them on the device-
    evaluated oracle itself)."""
    import exact_schedule as es
    y0, t, rtol, atol, opts = lc.solve_setup(method, dtype, reverse)
    s = es.oracle_solve(lc.torch_rhs(lc.solve_module(dtype)), y0, t, method, rtol, atol, opts)
    p = es.premises(s, opts["first_step"])
    assert p["dyadic"] and p["decisions_agree"] and p["n_rej"] >= 1 and p["margin"] > es.MARGIN[dtype], p
