"""GPU: rhs.LatentODEFunc, examples/latent_ode.py's network, as a built-in right-hand side.

* Per evaluation, ``b2ode_rhs_eval`` (f) and ``b2ode_adjoint_rhs_eval`` (g^T df/dy) within the error bound of the 60-digit
  reference of tests/latent_cases.py, at H = 1, 20, 32, fp32 and fp64, weights at std 0.1 and 3; non-finite rows by
  class; the reversed system as the exact negation; a batch past one pass of the evaluation grid.
* Solves: the persistent kernel, the stage kernels (``fused_rhs='stages'``), ``independent_rows`` and the fixed grid
  against the module's own forward on the generic path (``fused_rhs=False``).  (tsit5 is left out: on this network its
  controller drives dt to about 1e-8 on the generic path and in the kernels alike, and the solve does not finish.)
* Gradients with trainable weights: ``fused_vjp`` against the default autograd adjoint, ``backprop`` against
  ``fused_rhs=False``, ``independent_rows`` + ``backprop`` against single-row solves, each also run twice for equal bits,
  and a 271 337-row batch, where the parameter-sum tiles loop, run to run."""
import numpy as np
import pytest
import torch

import latent_cases as lc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    import tfdiffeq_b200.backprop  # noqa: F401  (imported on first use by odeint)
    return tfdiffeq_b200


def _bits_equal(a, b):
    it = torch.int64 if a.dtype == torch.float64 else torch.int32
    return a.shape == b.shape and torch.equal(a.contiguous().view(it), b.contiguous().view(it))


def _device_f(mod, y, time_sign=1.0):
    import rhs_cases as rc
    return rc.device_eval(mod, y, time_sign=time_sign)


def _device_vjp(mod, y, g, time_sign=1.0):
    """g^T df/dy through the stage kernels' augmented dynamics: b2ode_adjoint_rhs_eval at (y, a = -g), frozen weights."""
    from test_fused_vjp_gpu import fused_eval
    dt = y.dtype
    comps = (y, -g, torch.zeros((), dtype=dt, device=DEV), torch.zeros((), dtype=dt, device=DEV))
    run, weights = fused_eval(mod, comps, 0.0, time_sign)
    out = run()
    torch.cuda.synchronize()
    del weights
    return out[0], out[1]


CASES = [(H, std, dt) for H in (1, 20, 32) for std in (0.1, 3.0) for dt in ("float32", "float64")]


@pytest.mark.parametrize("H,std,dtype", CASES)
def test_eval_and_vjp_within_the_bound(H, std, dtype):
    tdt = torch.float64 if dtype == "float64" else torch.float32
    mod = lc.module(H, std, tdt, seed=100 + H).to(DEV)
    for p in mod.parameters():
        p.requires_grad_(False)
    y, g = lc.rows(48, std, seed=H + (7 if std > 1 else 0), dtype=np.dtype(dtype))
    ref = lc.reference(mod.cpu(), y, g)
    mod.to(DEV)
    bf, bg = lc.bound(mod.cpu(), y, g, ref, dtype)
    mod.to(DEV)
    yt, gt = torch.tensor(y, device=DEV), torch.tensor(g, device=DEV)
    f = _device_f(mod, yt).double().cpu().numpy()
    f2, gy = _device_vjp(mod, yt, gt)
    assert np.all(np.abs(f - ref["f"]) <= bf), float(np.max(np.abs(f - ref["f"]) / bf))
    gy = gy.double().cpu().numpy()
    assert np.all(np.abs(gy - ref["gy"]) <= bg), float(np.max(np.abs(gy - ref["gy"]) / bg))
    assert (ref["a1"] > 0).any() and (ref["a1"] <= 0).any()
    if H > 1:
        assert (ref["a2"] > 0).any() and (ref["a2"] <= 0).any()
    # the vjp's f is eval's, bit for bit, and the reversed system is the exact negation
    assert _bits_equal(f2, _device_f(mod, yt))
    assert _bits_equal(_device_f(mod, yt, -1.0), -_device_f(mod, yt))
    fn, gn = _device_vjp(mod, yt, gt, -1.0)
    assert _bits_equal(fn, -f2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_non_finite_rows_and_grid_passes(dtype):
    mod = lc.module(20, 0.5, dtype, seed=3).to(DEV)
    sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    n = 8 * 256 * sm + 1                                          # one row past a whole pass of the evaluation grid
    gen = torch.Generator(device=DEV).manual_seed(5)
    y = torch.randn(n, 4, dtype=dtype, device=DEV, generator=gen)
    y[7, 2] = float("nan")
    y[9, 0] = float("inf")
    y[11, 1] = -float("inf")
    f = _device_f(mod, y)
    want = mod(torch.zeros((), dtype=dtype, device=DEV), y).detach()
    bad = ~torch.isfinite(want)
    assert torch.equal(bad, ~torch.isfinite(f)) and torch.equal(torch.isnan(want), torch.isnan(f))
    fin = ~bad.any(1)
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    assert float((f[fin] - want[fin]).abs().max()) <= tol * max(1.0, float(want[fin].abs().max()))
    # rows are independent: a row evaluated in the big batch equals the same row alone
    for r in (0, 7, n // 2, n - 1):
        assert _bits_equal(f[r:r + 1][~torch.isnan(f[r:r + 1])], _device_f(mod, y[r:r + 1].clone())[~torch.isnan(f[r:r + 1])])


def _spiral_latent(n, dtype, seed=0):
    """latent_ode.py's initial states are a recognition network's samples: here z0 ~ N(0, 1) rows of 4."""
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(n, 4, dtype=dtype, generator=gen).to(DEV)


def _samp_ts(n=100, dtype=torch.float64):
    # generate_spiral2d's grid (latent_ode.py:31-32): 100 samples of linspace(0, 6 pi, 1000) from the start
    return torch.linspace(0.0, 6.0 * np.pi, 1000, dtype=dtype)[:n].to(DEV)


@pytest.mark.parametrize("method,opts", [("dopri5", {}), ("dopri8", {}), ("dopri5", {"fused_rhs": "stages"}),
                                         ("dopri8", {"fused_rhs": "stages"}), ("dopri5", {"independent_rows": True}),
                                         ("rk4", {"step_size": 0.05})])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("reverse", [False, True])
def test_solves_against_the_generic_path(method, opts, dtype, reverse):
    mod = tfd().rhs.LatentODEFunc(hidden=20, dtype=dtype, generator=torch.Generator().manual_seed(1)).to(DEV)
    for p in mod.parameters():
        p.requires_grad_(False)
    y0 = _spiral_latent(1000, dtype)
    t = _samp_ts(11, dtype)
    t = -t if reverse else t
    rtol, atol = (1e-9, 1e-11) if dtype == torch.float64 else (1e-5, 1e-7)
    got = tfd().odeint(mod, y0, t, rtol=rtol, atol=atol, method=method, options=dict(opts) or None)
    st = dict(tfd().last_stats)
    if method == "rk4" or "independent_rows" in opts:
        assert st["fused_rhs"] and st.get("independent_rows", False) == ("independent_rows" in opts), st
    else:
        assert st["fused_rhs"] == (opts.get("fused_rhs") != "stages") and st["stage_rhs"] == (opts.get("fused_rhs") == "stages"), st
    shared = {k: v for k, v in opts.items() if k not in ("independent_rows", "fused_rhs")}
    want = tfd().odeint(mod, y0, t, rtol=rtol, atol=atol, method=method, options=dict(shared, fused_rhs=False))
    # the same steps up to rounding; with independent rows every row takes its own steps (both within the tolerance)
    tol = (1e-7 if dtype == torch.float64 else 2e-3) * (100 if "independent_rows" in opts else 1)
    assert float((got - want).abs().max()) <= tol * max(1.0, float(want.abs().max()))


def _loss_weights(t, n, dtype, seed=2):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(len(t), n, 4, dtype=dtype, generator=gen).to(DEV)


def _grads(mod, y0, t, w, odeint, with_solution=False, **kw):
    y = y0.clone().requires_grad_(True)
    sol = odeint(mod, y, t, **kw)
    (sol * w).sum().backward()
    gp = [p.grad.clone() for p in mod.parameters()]
    for p in mod.parameters():
        p.grad = None
    return ([y.grad] + gp, sol.detach()) if with_solution else [y.grad] + gp


def _rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-300)


def test_fused_vjp_against_the_autograd_adjoint():
    mod = tfd().rhs.LatentODEFunc(hidden=20, dtype=torch.float64, generator=torch.Generator().manual_seed(2)).to(DEV)
    y0 = _spiral_latent(1000, torch.float64)
    t = _samp_ts(11)
    w = _loss_weights(t, 1000, torch.float64)
    kw = dict(rtol=1e-7, atol=1e-9, method="dopri5")
    on = _grads(mod, y0, t, w, tfd().odeint_adjoint, adjoint_options={"fused_vjp": True}, **kw)
    off = _grads(mod, y0, t, w, tfd().odeint_adjoint, **kw)
    assert len(on) == 7
    for a, b in zip(on, off):
        assert _rel(a, b) <= 1e-10, _rel(a, b)
    again = _grads(mod, y0, t, w, tfd().odeint_adjoint, adjoint_options={"fused_vjp": True}, **kw)
    assert all(_bits_equal(a, b) for a, b in zip(on, again))


@pytest.mark.parametrize("method", ["dopri5", "adaptive_heun", "rk4"])
def test_backprop_against_the_generic_path(method):
    mod = tfd().rhs.LatentODEFunc(hidden=20, dtype=torch.float64, generator=torch.Generator().manual_seed(3)).to(DEV)
    y0 = _spiral_latent(1000, torch.float64)
    t = _samp_ts(11)
    w = _loss_weights(t, 1000, torch.float64)
    kw = dict(rtol=1e-7, atol=1e-9, method=method)
    extra = {"step_size": 0.1} if method == "rk4" else {}
    on = _grads(mod, y0, t, w, tfd().odeint, options=dict(extra, backprop=True), **kw)
    assert tfd().backprop.last_stats["func_calls"] == 0
    off = _grads(mod, y0, t, w, tfd().odeint, options=dict(extra, backprop=True, fused_rhs=False), **kw)
    for a, b in zip(on, off):
        assert _rel(a, b) <= 1e-10, _rel(a, b)
    again = _grads(mod, y0, t, w, tfd().odeint, options=dict(extra, backprop=True), **kw)
    assert all(_bits_equal(a, b) for a, b in zip(on, again))


def test_rows_backprop_against_single_row_solves():
    mod = tfd().rhs.LatentODEFunc(hidden=20, dtype=torch.float64, generator=torch.Generator().manual_seed(4)).to(DEV)
    n = 24
    y0 = _spiral_latent(n, torch.float64, seed=5)
    t = _samp_ts(6)
    w = _loss_weights(t, n, torch.float64, seed=6)
    kw = dict(rtol=1e-7, atol=1e-9, method="dopri5")
    rows, sol_rows = _grads(mod, y0, t, w, tfd().odeint, with_solution=True,
                            options={"independent_rows": True, "backprop": True}, **kw)
    psum = [torch.zeros_like(p) for p in mod.parameters()]
    same = 0
    for r in range(n):
        # the shared-step forward (stage kernels) and the rows kernel add up a row's error norm in different orders, so
        # their step sizes can differ by a rounding: bit-equality is required where the two forward solutions agree
        one, sol_one = _grads(mod, y0[r:r + 1], t, w[:, r:r + 1], tfd().odeint, with_solution=True,
                              options={"backprop": True}, **kw)
        if torch.equal(sol_one, sol_rows[:, r:r + 1]):
            same += 1
            assert _bits_equal(rows[0][r:r + 1], one[0]), r
        else:
            assert _rel(rows[0][r:r + 1], one[0]) <= 1e-10, r
        for s, g in zip(psum, one[1:]):
            s += g
    assert same >= n // 2, same
    for a, b in zip(rows[1:], psum):
        assert _rel(a, b) <= 1e-10, _rel(a, b)
    again = _grads(mod, y0, t, w, tfd().odeint, options={"independent_rows": True, "backprop": True}, **kw)
    assert all(_bits_equal(a, b) for a, b in zip(rows, again))


def test_rows_fused_vjp_adjoint_with_frozen_weights():
    mod = tfd().rhs.LatentODEFunc(hidden=20, dtype=torch.float64, generator=torch.Generator().manual_seed(7)).to(DEV)
    for p in mod.parameters():
        p.requires_grad_(False)
    n = 64
    y0 = _spiral_latent(n, torch.float64, seed=8)
    t = _samp_ts(6)
    w = _loss_weights(t, n, torch.float64, seed=9)
    kw = dict(rtol=1e-7, atol=1e-9, method="dopri5")
    opts = {"independent_rows": True, "fused_vjp": True}
    y = y0.clone().requires_grad_(True)
    (tfd().odeint_adjoint(mod, y, t, options=opts, adjoint_options=opts, **kw) * w).sum().backward()
    for r in (0, 17, 63):
        yr = y0[r:r + 1].clone().requires_grad_(True)
        (tfd().odeint_adjoint(mod, yr, t, adjoint_options={"fused_vjp": True}, **kw) * w[:, r:r + 1]).sum().backward()
        assert _rel(y.grad[r:r + 1], yr.grad) <= 1e-8, r


def test_large_batch_is_deterministic():
    """271 337 rows: several tiles per block in every parameter-sum kernel."""
    mod = tfd().rhs.LatentODEFunc(hidden=20, dtype=torch.float32, generator=torch.Generator().manual_seed(10)).to(DEV)
    n = 271337
    y0 = _spiral_latent(n, torch.float32, seed=11)
    t = _samp_ts(3, torch.float32) * 0.1
    w = _loss_weights(t, n, torch.float32, seed=12)
    kw = dict(rtol=1e-5, atol=1e-7, method="dopri5")
    for odeint, extra in ((tfd().odeint_adjoint, dict(adjoint_options={"fused_vjp": True})),
                          (tfd().odeint, dict(options={"backprop": True})),
                          (tfd().odeint, dict(options={"backprop": True, "independent_rows": True}))):
        a = _grads(mod, y0, t, w, odeint, **extra, **kw)
        b = _grads(mod, y0, t, w, odeint, **extra, **kw)
        assert all(_bits_equal(x, z) for x, z in zip(a, b))
        assert all(bool(torch.isfinite(x).all()) and float(x.abs().max()) > 0 for x in a)
