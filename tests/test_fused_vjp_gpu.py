"""GPU: odeint_adjoint's backward pass for built-in right-hand sides in the stage kernels (adjoint_options fused_vjp).

* Per evaluation, b2ode_adjoint_rhs_eval against the default path's augmented dynamics (torch autograd of the module's
  forward) on the same device tensors, both time signs, fp32 and fp64, at row counts where the grid strides: Lorenz,
  Lotka-Volterra and Kepler bit for bit in every segment; CubicMLP within a bound of fp64 CPU autograd, and bit-identical
  between two calls and under CUDA-graph replay.
* Whole odeint_adjoint, flag on against flag off: same forward solution, gradients, backward step counts and dt_next for
  the bit-exact systems; CubicMLP to rounding.
* No forward call per evaluation, and the refusals raise before any launch.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_adjoint as ea
from problems import PROBLEMS
from test_fused_vjp_cpu import refusal_cases

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _state(kind, rows, dtype, seed):
    rng = np.random.default_rng(seed)
    D = {"lorenz": 3, "lotka_volterra": 2, "kepler": 4, "cubic_mlp": 2}[kind]
    y = rng.standard_normal((rows, D)) * (3.0 if kind != "cubic_mlp" else 1.0)
    a = rng.standard_normal((rows, D)) * (rng.random((rows, D)) >= 1.0 / 6)
    a[::11] = 0.0
    return torch.tensor(y, dtype=dtype, device=DEV), torch.tensor(a, dtype=dtype, device=DEV)


def _module(kind, dtype):
    if kind == "lorenz":
        return tfd().rhs.Lorenz(9.5, 2.5, 27.25)
    if kind == "lotka_volterra":
        return tfd().rhs.LotkaVolterra(1.3, 0.7, 2.9, 1.1)
    if kind == "kepler":
        return tfd().rhs.Kepler()
    gen = torch.Generator().manual_seed(5)
    m = tfd().rhs.CubicMLP(50, std=0.5, dtype=torch.float64, generator=gen)
    with torch.no_grad():
        m.b1.copy_(0.1 * torch.randn(50, generator=gen, dtype=torch.float64))
        m.b2.copy_(torch.tensor([0.25, -0.5], dtype=torch.float64))
    return m.to(device=DEV, dtype=dtype)


def fused_eval(mod, comps, t, sign):
    """The four k components of b2ode_adjoint_rhs_eval at the augmented state `comps`, in the engine's layout."""
    from tfdiffeq_b200 import _lib, solvers
    lib = _lib.lib
    seg = solvers._Segments(comps)
    Y, K = seg.new(), seg.new()
    seg.fill(Y, comps)
    dtype = comps[0].dtype
    rd, weights = mod.rhs_desc(dtype, DEV, sign)
    lens = _lib.LenArray(*seg.lens)
    sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    nb = int(lib.b2ode_adjoint_rhs_workspace_bytes(C.byref(rd), lens, sm))
    ws = torch.zeros(nb, dtype=torch.uint8, device=DEV)
    tt = torch.tensor(t, dtype=dtype, device=DEV)

    def run():
        _lib.check(lib.b2ode_adjoint_rhs_eval(solvers._DT[dtype], C.byref(rd), C.c_void_p(tt.data_ptr()), lens,
                                              solvers._ptr_array(seg.ptrs(Y)), solvers._ptr_array(seg.ptrs(K)),
                                              C.c_void_p(ws.data_ptr()), nb, sm,
                                              C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)))
        return tuple(v.clone() for v in seg.views(K))
    return run, weights


def default_eval(mod, comps, t, sign):
    """odeint_adjoint's default augmented dynamics on the same tensors, behind the reverse-time wrapper for sign -1."""
    from tfdiffeq_b200 import adjoint
    func = adjoint._TupleFunc(mod)
    f_params = tuple(p for p in func.parameters() if p.requires_grad)
    dyn = adjoint._augmented_dynamics(func, 1, f_params, comps[0].dtype, DEV, None)
    tt = torch.tensor(t, dtype=comps[0].dtype, device=DEV)
    if sign < 0:
        return tuple(-x for x in dyn(-tt, comps))
    return dyn(tt, comps)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int64 if a.dtype == torch.float64 else torch.int32),
                                              b.contiguous().view(torch.int64 if b.dtype == torch.float64 else torch.int32))


@pytest.mark.parametrize("kind", ["lorenz", "lotka_volterra", "kepler"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_eval_equals_autograd_bit_for_bit(kind, dtype, sign):
    """600 001 rows: more than two passes of the 8-blocks-per-SM grid."""
    mod = _module(kind, dtype)
    y, a = _state(kind, 600001, dtype, 11)
    comps = (y, a, torch.tensor(0.375, dtype=dtype, device=DEV), torch.zeros((), dtype=dtype, device=DEV))
    run, weights = fused_eval(mod, comps, 0.5, sign)      # `weights` backs the descriptor: keep it referenced
    got = run()
    want = default_eval(mod, comps, 0.5, sign)
    for s, (g, w) in enumerate(zip(got, want)):
        assert _bits_equal(g, w.reshape(g.shape)), (s, float((g - w.reshape(g.shape)).abs().max()))
    assert bool(torch.signbit(got[2])) == (sign < 0)                 # -0 behind the reverse-time wrapper, as torch gives


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("cube", [True, False])
def test_cubic_mlp_eval_bound_determinism_and_graph_replay(dtype, sign, cube):
    mod = _module("cubic_mlp", dtype)
    mod.cube = cube
    y, a = _state("cubic_mlp", 300001, dtype, 12)
    P = 5 * 50 + 2
    comps = (y, a, torch.tensor(0.375, dtype=dtype, device=DEV), torch.full((P,), 0.5, dtype=dtype, device=DEV))
    run, weights = fused_eval(mod, comps, 0.5, sign)      # `weights` backs the descriptor: keep it referenced
    got = run()
    again = run()
    assert all(_bits_equal(g, h) for g, h in zip(got, again))
    # fp64 CPU autograd of the same weights at the same (rounded) inputs
    ref_mod = _module("cubic_mlp", torch.float64).cpu()
    ref_mod.cube = cube
    want = default_eval_cpu(ref_mod, tuple(c.double().cpu() for c in comps), 0.5, sign)
    tol = 1e-10 if dtype == torch.float64 else 2e-5
    for s, (g, w) in enumerate(zip(got, want)):
        g = g.double().cpu().reshape(w.shape)
        scale = max(float(w.abs().max()), 1e-30)
        assert float((g - w).abs().max()) <= tol * scale, (s, float((g - w).abs().max()) / scale)
    # CUDA-graph replay of the launch: the ticket is left at zero, so every replay sums the partials the same way
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        graph.capture_begin()
        captured = run()
        graph.capture_end()
    torch.cuda.current_stream(DEV).wait_stream(side)
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        assert all(_bits_equal(g, h) for g, h in zip(got, captured))


def default_eval_cpu(mod, comps, t, sign):
    from tfdiffeq_b200 import adjoint
    func = adjoint._TupleFunc(mod)
    f_params = tuple(p for p in func.parameters() if p.requires_grad)
    dyn = adjoint._augmented_dynamics(func, 1, f_params, torch.float64, torch.device("cpu"), None)
    tt = torch.tensor(t, dtype=torch.float64)
    out = dyn(-tt, comps) if sign < 0 else dyn(tt, comps)
    return tuple(-x for x in out) if sign < 0 else out


# --------------------------------------------------------------------------------------------------
# whole odeint_adjoint, flag on against flag off
# --------------------------------------------------------------------------------------------------
def _run(mod, y0, t, w, on, **kw):
    y = y0.clone().requires_grad_(True)
    tt = t.clone().requires_grad_(True)
    opts = dict(kw.pop("options", {}) or {})
    if on:
        kw["adjoint_options"] = dict(opts, fused_vjp=True)
    sol = tfd().odeint_adjoint(mod, y, tt, options=opts or None, **kw)
    (sol * w).sum().backward()
    st = tfd().adjoint.last_stats
    grads = [p.grad.clone() if p.grad is not None else None for p in mod.parameters()]
    for p in mod.parameters():
        p.grad = None
    return sol.detach(), y.grad, tt.grad, grads, dict(st["forward"]), [dict(b) for b in st["backward"]]


def _counts(b):
    return (b["n_accepted"], b["n_rejected"], b["nfe"], b["dt_next"])


def _compare_exact(mod, y0, t, w, **kw):
    off = _run(mod, y0, t, w, False, **dict(kw))
    on = _run(mod, y0, t, w, True, **dict(kw))
    assert torch.equal(on[0], off[0])
    assert torch.equal(on[1], off[1])
    assert torch.equal(on[2], off[2])
    assert _counts(on[4]) == _counts(off[4])
    assert len(on[5]) == len(off[5]) == len(t) - 1
    assert [_counts(b) for b in on[5]] == [_counts(b) for b in off[5]]
    assert all(b.get("fused_vjp") is True for b in on[5]) and not any("fused_vjp" in b for b in off[5])


@pytest.mark.parametrize("name,reverse", [("builtin_lorenz-dopri5-f64-fwd-12627", False),
                                          ("builtin_lorenz-dopri5-f64-fwd-12627", True),
                                          ("builtin_lorenz-tsit5-f64-fwd-12627", False)])
def test_odeint_adjoint_lorenz_flag_on_equals_flag_off(name, reverse):
    """The 12 627-row inputs of tests/exact_adjoint.py; reversed output times make the backward solves run forward."""
    case = ea.ALL[name]
    y0 = ea.initial_state(case)[0]
    w = ea.loss_weights(case, (y0,))[0]
    t = -case.t if reverse else case.t
    _compare_exact(tfd().rhs.Lorenz(), torch.tensor(y0, device=DEV), torch.tensor(t, device=DEV),
                   torch.tensor(w, device=DEV), rtol=case.rtol, atol=case.atol, method=case.method,
                   options=ea.options(case))


def test_odeint_adjoint_lotka_volterra_bosh3_flag_on_equals_flag_off():
    rng = np.random.default_rng(21)
    y0 = torch.tensor(1.0 + rng.random((5003, 2)), device=DEV)
    w = torch.tensor(rng.standard_normal((4, 5003, 2)), device=DEV)
    t = torch.tensor([0.0, 0.2, 0.35, 0.5], device=DEV)
    _compare_exact(tfd().rhs.LotkaVolterra(1.3, 0.7, 2.9, 1.1), y0, t, w, rtol=1e-6, atol=1e-8, method="bosh3")


def test_odeint_adjoint_kepler_dopri8_flag_on_equals_flag_off():
    k_np = PROBLEMS["kepler"](backend="numpy")
    y0 = torch.tensor(k_np.y0(64, seed=3), device=DEV)
    rng = np.random.default_rng(22)
    w = torch.tensor(rng.standard_normal((3,) + tuple(y0.shape)), device=DEV)
    t = torch.tensor([0.0, 0.3, 0.6], device=DEV)
    _compare_exact(tfd().rhs.Kepler(), y0, t, w, rtol=1e-9, atol=1e-9, method="dopri8")


def _spiral(n, dtype):
    """ode_demo's spiral: initial states along r = 2 exp(-theta / 4), slightly perturbed."""
    rng = np.random.default_rng(23)
    th = rng.uniform(0.0, 6.0, n)
    r = 2.0 * np.exp(-th / 4.0) * (1.0 + 0.05 * rng.standard_normal(n))
    return torch.tensor(np.stack([r * np.cos(th), r * np.sin(th)], 1), dtype=dtype, device=DEV)


def test_odeint_adjoint_cubic_mlp_flag_on_against_flag_off():
    n = 8192
    t = torch.tensor([0.0, 0.2, 0.5, 1.0], device=DEV)
    rng = np.random.default_rng(24)
    w = torch.tensor(rng.standard_normal((4, n, 2)), device=DEV)
    y0 = _spiral(n, torch.float64)
    mod = tfd().rhs.CubicMLP(50, dtype=torch.float64, generator=torch.Generator().manual_seed(0)).to(DEV)
    kw = dict(rtol=1e-7, atol=1e-9, method="dopri5")
    off = _run(mod, y0, t, w, False, **kw)
    on = _run(mod, y0, t, w, True, **kw)
    assert torch.equal(on[0], off[0])                                  # the forward solve is the same persistent kernel
    assert [_counts(b)[:3] for b in on[5]] == [_counts(b)[:3] for b in off[5]]

    def rel(a, b):
        return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-300)
    assert rel(on[1], off[1]) <= 1e-9 and rel(on[2], off[2]) <= 1e-9
    for g_on, g_off in zip(on[3], off[3]):
        assert rel(g_on, g_off) <= 1e-9
    # fp32 with the flag against the fp64 default path
    mod32 = tfd().rhs.CubicMLP(50, dtype=torch.float64, generator=torch.Generator().manual_seed(0)).to(DEV, torch.float32)
    on32 = _run(mod32, y0.float(), t.float(), w.float(), True, rtol=1e-5, atol=1e-7, method="dopri5")
    assert rel(on32[1].double(), off[1]) <= 1e-3
    for g32, g64 in zip(on32[3], off[3]):
        assert rel(g32.double(), g64) <= 1e-3


def test_no_forward_call_per_evaluation():
    mod = tfd().rhs.CubicMLP(50, dtype=torch.float64, generator=torch.Generator().manual_seed(0)).to(DEV)
    calls = [0]
    mod.register_forward_hook(lambda *a: calls.__setitem__(0, calls[0] + 1))
    t = torch.tensor([0.0, 0.2, 0.5, 1.0], device=DEV)
    y0 = _spiral(4096, torch.float64)
    for on, check in ((True, lambda c: c == len(t) - 1), (False, lambda c: c > 10 * len(t))):
        sol = tfd().odeint_adjoint(mod, y0, t, rtol=1e-7, atol=1e-9, method="dopri5",
                                   adjoint_options={"fused_vjp": True} if on else None)
        calls[0] = 0
        sol.pow(2).sum().backward()
        assert check(calls[0]), (on, calls[0])                        # with the flag: the dL/dt_i terms only
        assert all(b.get("fused_vjp", False) == on for b in tfd().adjoint.last_stats["backward"])


def test_refusals_before_any_launch():
    from tfdiffeq_b200 import _lib
    cases, t = refusal_cases(DEV)
    for name, func, y0, fwd, kw in cases:
        if "options" in kw and "method" not in fwd:
            fwd = dict(fwd, method="dopri5")
        before = _lib.lib.b2ode_launch_count()
        with pytest.raises(ValueError):
            tfd().odeint_adjoint(func, y0, t, **fwd, **kw)
        assert _lib.lib.b2ode_launch_count() == before, name
