"""GPU: odeint(..., options={'backprop': True}) -- reverse-mode gradients through the accepted steps, checked against
autograd through the oracle's own discrete solver (oracle/np_ref.py on torch-CPU tensors, the schedule held constant by
its .item() reads) and against the bp_g_* fixtures of tests/golden/grad_*.npz."""
import gc
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TDT = {"float32": torch.float32, "float64": torch.float64}
ADAPTIVE = ["dopri5", "bosh3", "adaptive_heun", "dopri8"]
FIXED = ["euler", "midpoint", "rk4", "heun"]


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(1e-300, float(np.max(np.abs(b)))))


def _grad_case_module(case, tdt):
    from grad_cases import build_params, rhs_torch
    params = build_params(case, tdt, device=DEV)

    class F(nn.Module):
        def __init__(self):
            super().__init__()
            self.ps = nn.ParameterDict({n: nn.Parameter(p.detach().clone()) for n, p in params.items()})

        def forward(self, t, y):
            return rhs_torch(case, self.ps, t, y)
    return F().to(DEV)


def _oracle_counts(case):
    import np_ref
    from grad_cases import build_params, rhs_torch
    tdt = TDT[case["dtype"]]
    params = build_params(case, tdt)
    st = np_ref.Stats()
    y0 = tuple(torch.tensor(np.asarray(v), dtype=tdt) for v in case["y0"])
    with torch.no_grad():
        np_ref.odeint(lambda t, y: rhs_torch(case, params, torch.tensor(float(t), dtype=tdt), y),
                      y0[0] if len(y0) == 1 else y0, np.asarray(case["t"]), rtol=case["rtol"], atol=case["atol"],
                      method=case["method"], stats=st)
    return st.n_acc, st.n_rej


@pytest.mark.parametrize("name", ["spiral3_dopri5", "spiral3_dopri8", "spiral3_rk4", "mlp_tanh_dopri5", "mlp_tanh_f32",
                                  "timedep_dopri5", "tuple2_dopri5"])
def test_backprop_matches_golden_discrete_gradients(name, golden_dir):
    from grad_cases import GRAD_CASES
    case = GRAD_CASES[name]
    g = np.load(os.path.join(golden_dir, "grad_" + name + ".npz"))
    tdt = TDT[case["dtype"]]
    m = _grad_case_module(case, tdt)
    y0 = tuple(torch.tensor(v, dtype=tdt, device=DEV, requires_grad=True) for v in case["y0"])
    t = torch.tensor(case["t"], dtype=torch.float64, device=DEV)
    w = tuple(torch.tensor(v, dtype=tdt, device=DEV) for v in case["w"])
    ys = tfd().odeint(m, y0[0] if len(y0) == 1 else y0, t, rtol=case["rtol"], atol=case["atol"], method=case["method"],
                      options={"backprop": True})
    stats = dict(tfd().solvers.last_stats)
    ys = (ys,) if isinstance(ys, torch.Tensor) else ys
    assert all(y.grad_fn is not None for y in ys)
    sum((s * w_).sum() for s, w_ in zip(ys, w)).backward()
    tol = 1e-9 if case["dtype"] == "float64" else 1e-3
    for i, v in enumerate(y0):
        assert _rel(v.grad.cpu().numpy(), g["bp_g_y0_%d" % i]) <= tol, ("y0", i)
    for n, p in m.ps.items():
        assert _rel(p.grad.cpu().numpy(), g["bp_g_param_" + n]) <= tol, n
    if case["method"] in ADAPTIVE:
        assert (stats["n_accepted"], stats["n_rejected"]) == _oracle_counts(case)


class Net(nn.Module):
    """A small time-dependent field with trainable weights: y' = W2 tanh(W1 y + b cos t) - c y."""

    def __init__(self, d, dtype, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.W1 = nn.Parameter(0.6 * torch.randn(d, 6, generator=g, dtype=dtype))
        self.W2 = nn.Parameter(0.6 * torch.randn(6, d, generator=g, dtype=dtype))
        self.b = nn.Parameter(0.3 * torch.randn(6, generator=g, dtype=dtype))
        self.c = nn.Parameter(torch.tensor(0.1, dtype=dtype))

    def forward(self, t, y):
        return torch.tanh(y @ self.W1 + self.b * torch.cos(t)) @ self.W2 - self.c * y


def _oracle_backprop(net, y0, t, method, rtol, atol, w, options=None):
    """Autograd through np_ref on torch-CPU copies: (y0 grads, param grads, (n_acc, n_rej))."""
    import np_ref
    cpu = Net(y0[0].shape[-1], y0[0].dtype)
    cpu.load_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()})
    ys0 = tuple(v.detach().cpu().clone().requires_grad_(True) for v in y0)
    tdt = y0[0].dtype
    st = np_ref.Stats()

    def f(tt, y):
        tt = torch.tensor(float(tt), dtype=tdt)
        if isinstance(y, tuple):
            return tuple(cpu(tt, v) for v in y)
        return cpu(tt, y)
    sol = np_ref.odeint(f, ys0[0] if len(ys0) == 1 else ys0, np.asarray(t, dtype=np.float64), rtol=rtol, atol=atol,
                        method=method, options=options, stats=st)
    sol = (sol,) if len(ys0) == 1 else sol
    loss = sum((s * w_).sum() for s, w_ in zip(sol, w))
    ps = list(cpu.parameters())
    gs = torch.autograd.grad(loss, list(ys0) + ps)
    return gs[:len(ys0)], gs[len(ys0):], (st.n_acc, st.n_rej)


def _engine_backprop(net, y0, t, method, rtol, atol, w, options=None):
    y0d = tuple(v.detach().to(DEV).requires_grad_(True) for v in y0)
    for p in net.parameters():
        p.grad = None
    opts = dict(options or {}, backprop=True)
    func = net if len(y0d) == 1 else _TupleNet(net)
    ys = tfd().odeint(func, y0d[0] if len(y0d) == 1 else y0d, torch.tensor(t, dtype=torch.float64), rtol=rtol, atol=atol,
                      method=method, options=opts)
    st = dict(tfd().solvers.last_stats)
    ys = (ys,) if len(y0d) == 1 else ys
    sum((s * w_.to(DEV)).sum() for s, w_ in zip(ys, w)).backward()
    return [v.grad.cpu() for v in y0d], [p.grad.cpu() for p in net.parameters()], (st["n_accepted"], st["n_rejected"])


class _TupleNet(nn.Module):
    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, t, y):
        return tuple(self.net(t, v) for v in y)


def _check(method, dtype, t, tuple_state=False, seed=0, options=None):
    tdt = TDT[dtype]
    net = Net(3, tdt, seed).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    y0 = (torch.randn(4, 3, generator=g, dtype=tdt),)
    if tuple_state:
        y0 = y0 + (torch.randn(2, 3, generator=g, dtype=tdt),)
    w = tuple(torch.randn((len(t),) + v.shape, generator=g, dtype=tdt) for v in y0)
    rtol, atol = (1e-7, 1e-9) if dtype == "float64" else (1e-4, 1e-6)
    a = _oracle_backprop(net, y0, t, method, rtol, atol, w, options)
    b = _engine_backprop(net, y0, t, method, rtol, atol, w, options)
    tol = 1e-9 if dtype == "float64" else 1e-3
    if method in ADAPTIVE:
        assert a[2] == b[2], (a[2], b[2])
    for x, y in zip(list(a[0]) + list(a[1]), list(b[0]) + list(b[1])):
        assert _rel(y.numpy(), x.numpy()) <= tol, _rel(y.numpy(), x.numpy())


# dopri8 is left out of the Net matrix: its embedded error is a cancellation of ~1e-7 out of O(1) k's, so the ulp-level
# differences between CPU and GPU tanh/matmul move the oracle's own dt values by ~1e-9 relative (and, in fp32, can move a
# decision).  The oracle would then differentiate a different schedule.  dopri8 is checked on y**3 @ A below, where both
# sides evaluate the field bit for bit alike, and on the golden spiral3_dopri8 fixture.
@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("method", ["dopri5", "bosh3", "adaptive_heun"] + FIXED)
def test_backprop_matches_oracle(method, reverse, dtype):
    t = np.array([0.0, 0.13, 0.5, 0.51, 1.2, 1.6])
    if reverse:
        t = 1.0 - t
    options = {"step_size": 0.1} if method in FIXED else None
    _check(method, dtype, t, options=options)


class Cubic(nn.Module):
    def __init__(self, dtype, sign=1.0):
        super().__init__()
        # sign -1 for reverse time keeps the spiral decaying in the direction of integration
        self.A = nn.Parameter(sign * torch.tensor([[-0.1, 2.0], [-2.0, -0.1]], dtype=dtype))

    def forward(self, t, y):
        return (y ** 3) @ self.A


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("reverse", [False, True])
def test_backprop_dopri8_matches_oracle(reverse, dtype):
    import np_ref
    tdt = TDT[dtype]
    t = np.array([0.0, 0.3, 0.31, 0.9, 1.5])
    if reverse:
        t = 1.5 - t
    y0 = torch.tensor([[2.0, 0.0], [1.0, 0.5], [-0.7, 0.3]], dtype=tdt)
    w = torch.randn((len(t),) + y0.shape, generator=torch.Generator().manual_seed(4), dtype=tdt)
    rtol, atol = (1e-8, 1e-10) if dtype == "float64" else (1e-5, 1e-6)
    cpu = Cubic(tdt, -1.0 if reverse else 1.0)
    y0c = y0.clone().requires_grad_(True)
    st = np_ref.Stats()
    sol = np_ref.odeint(lambda tt, y: cpu(tt, y), y0c, t, rtol=rtol, atol=atol, method="dopri8", stats=st)
    want = torch.autograd.grad((sol * w).sum(), (y0c, cpu.A))
    m = Cubic(tdt, -1.0 if reverse else 1.0).to(DEV)
    y0d = y0.to(DEV).requires_grad_(True)
    ys = tfd().odeint(m, y0d, torch.tensor(t), rtol=rtol, atol=atol, method="dopri8", options={"backprop": True})
    assert (tfd().solvers.last_stats["n_accepted"], tfd().solvers.last_stats["n_rejected"]) == (st.n_acc, st.n_rej)
    (ys * w.to(DEV)).sum().backward()
    tol = 1e-9 if dtype == "float64" else 1e-3
    assert _rel(y0d.grad.cpu().numpy(), want[0].numpy()) <= tol
    assert _rel(m.A.grad.cpu().numpy(), want[1].numpy()) <= tol


@pytest.mark.parametrize("method", ["dopri5", "adaptive_heun", "rk4"])
def test_backprop_tuple_state(method):
    _check(method, "float64", np.array([0.0, 0.7, 1.5]), tuple_state=True,
           options={"step_size": 0.25} if method == "rk4" else None)


def test_backprop_outputs_inside_one_step_and_at_a_step_end():
    # many outputs inside few large steps; on the fixed grid an output on a grid point is the step's end state
    _check("dopri5", "float64", np.linspace(0.0, 0.05, 9))
    _check("midpoint", "float64", np.array([0.0, 0.05, 0.1, 0.2, 0.23]), options={"step_size": 0.1})


def test_backprop_single_output_launches_nothing():
    net = Net(3, torch.float64).to(DEV)
    y0 = torch.randn(4, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    ys = tfd().odeint(net, y0, torch.tensor([0.3], dtype=torch.float64), method="dopri5", options={"backprop": True})
    w = torch.randn_like(ys)
    n0 = tfd()._lib.lib.b2ode_launch_count()
    (ys * w).sum().backward()
    assert tfd()._lib.lib.b2ode_launch_count() == n0
    assert torch.equal(y0.grad, w[0])
    assert all(p.grad is None or float(p.grad.abs().max()) == 0.0 for p in net.parameters())


@pytest.mark.parametrize("method", FIXED)
def test_backprop_gradcheck_fixed_grid(method):
    net = Net(2, torch.float64).to(DEV)
    y0 = torch.randn(3, 2, dtype=torch.float64, device=DEV, requires_grad=True)
    t = torch.tensor([0.0, 0.25, 0.6], dtype=torch.float64)

    def fn(y, W1, c):
        net.W1.data.copy_(W1.detach())
        net.c.data.copy_(c.detach())
        return tfd().odeint(lambda tt, v: net(tt, v), y, t, method=method, options={"backprop": True, "step_size": 0.1})
    # a plain callable gets y0 gradients only: check those with gradcheck, the parameter route in the oracle tests
    assert torch.autograd.gradcheck(lambda y: fn(y, net.W1, net.c), (y0,), eps=1e-6, atol=1e-7, rtol=1e-6)


@pytest.mark.parametrize("method", ["dopri5", "bosh3", "adaptive_heun", "dopri8"])
def test_backprop_gradcheck_adaptive_on_an_exact_schedule(method):
    """tests/exact_schedule.py's controller options keep dt a power-of-two multiple of first_step that only a rejection
    changes, so the discrete solve is a smooth function of y0 while no decision moves: gradcheck applies, and the counts
    must be the same for every perturbed solve."""
    from exact_schedule import MARGIN, OPTIONS
    lz = tfd().rhs.Lorenz()
    y0 = (torch.tensor([[1.0, 2.0, 20.0], [-3.0, 0.5, 25.0]], dtype=torch.float64)).to(DEV).requires_grad_(True)
    t = torch.tensor([0.0, 0.011, 0.05, 0.0625], dtype=torch.float64)
    kw = dict(rtol=1e-6, atol=1e-8, method=method, options=dict(OPTIONS, first_step=2.0 ** -7, backprop=True))
    seen = set()

    def fn(y):
        out = tfd().odeint(lz, y, t, **kw)
        st = tfd().solvers.last_stats
        seen.add((st["n_accepted"], st["n_rejected"]))
        assert abs(st["error_ratio"] - 1.0) > MARGIN["float64"]
        return out
    assert torch.autograd.gradcheck(fn, (y0,), eps=1e-6, atol=1e-6, rtol=1e-5)
    assert len(seen) == 1, seen


def test_backprop_double_backward_fails_loudly():
    net = Net(3, torch.float64).to(DEV)
    y0 = torch.randn(4, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    ys = tfd().odeint(net, y0, torch.linspace(0, 1, 3, dtype=torch.float64), method="rk4",
                      options={"backprop": True, "step_size": 0.25})
    (g,) = torch.autograd.grad(ys.sum(), y0, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()


def test_backprop_flag_without_grad_is_the_plain_solve():
    net = Net(3, torch.float64).to(DEV)
    for p in net.parameters():
        p.requires_grad_(False)
    y0 = torch.randn(64, 3, dtype=torch.float64, device=DEV)
    t = torch.linspace(0, 1, 5, dtype=torch.float64)
    lib = tfd()._lib.lib
    n0 = lib.b2ode_launch_count()
    a = tfd().odeint(net, y0, t, method="dopri5")
    n1 = lib.b2ode_launch_count()
    b = tfd().odeint(net, y0, t, method="dopri5", options={"backprop": True})
    n2 = lib.b2ode_launch_count()
    assert torch.equal(a, b) and n1 - n0 == n2 - n1 and b.grad_fn is None
    with torch.no_grad():
        net.c.requires_grad_(True)
        c = tfd().odeint(net, y0, t, method="dopri5", options={"backprop": True})
    assert torch.equal(a, c) and c.grad_fn is None
    # without the flag, as before: no graph even with trainable weights
    net.c.requires_grad_(True)
    assert tfd().odeint(net, y0, t, method="dopri5").grad_fn is None


def _count_forward(mod):
    calls = [0]
    mod.register_forward_hook(lambda *a: calls.__setitem__(0, calls[0] + 1))
    return calls


@pytest.mark.parametrize("method", ["dopri5", "bosh3", "dopri8", "adaptive_heun", "rk4"])
@pytest.mark.parametrize("name", ["lorenz", "lv", "kepler"])
def test_backprop_builtin_is_bit_identical_to_unfused(name, method):
    """RHS::vjp equals CUDA autograd bit for bit and both paths share the combine and dense kernels: y0.grad of the
    built-in module (b2ode_bp_rhs, no forward call in the backward pass) equals the fused_rhs=False path (torch forward
    and autograd) bit for bit."""
    rhs = tfd().rhs
    torch.manual_seed(0)
    if name == "lorenz":
        mod, y0 = rhs.Lorenz(), torch.randn(96, 3, dtype=torch.float64) + torch.tensor([0.0, 0.0, 20.0], dtype=torch.float64)
        t = torch.linspace(0, 0.3, 5, dtype=torch.float64)
    elif name == "lv":
        mod, y0 = rhs.LotkaVolterra(), 1.0 + 0.2 * torch.rand(64, 2, dtype=torch.float64)
        t = torch.linspace(0, 2.0, 5, dtype=torch.float64)
    else:
        mod = rhs.Kepler()
        th = torch.rand(32, dtype=torch.float64) * 6.0
        y0 = torch.stack([torch.cos(th), torch.sin(th), -0.9 * torch.sin(th), 0.9 * torch.cos(th)], 1).reshape(8, 16)
        t = torch.linspace(0, 1.0, 5, dtype=torch.float64)
    y0 = y0.to(DEV)
    w = torch.randn((5,) + tuple(y0.shape), dtype=torch.float64).to(DEV)
    opts = {"backprop": True, "step_size": 0.05} if method == "rk4" else {"backprop": True}
    calls = _count_forward(mod)
    grads, counts = [], []
    for extra in ({}, {"fused_rhs": False}):
        y = y0.clone().requires_grad_(True)
        ys = tfd().odeint(mod, y, t, rtol=1e-8, atol=1e-10, method=method, options=dict(opts, **extra))
        counts.append(tfd().solvers.last_stats["n_accepted"])
        before = calls[0]
        (ys * w).sum().backward()
        if not extra:
            # the adaptive forward runs in the stage kernels too; the fixed grid's recorded forward calls the module
            assert calls[0] == before and (before == 0 or method == "rk4"), "the built-in backward called forward"
        else:
            assert calls[0] > before
        grads.append(y.grad)
    assert counts[0] == counts[1]
    assert torch.equal(grads[0], grads[1])


def test_backprop_trainable_cubic_mlp_against_unfused_and_deterministic():
    """Parameter cotangents summed in fp64 in a fixed order (b2ode_bp_rhs) against torch autograd of the module: within
    1e-10 relative in fp64 (the unfused path sums per call in fp64 as well, in another order); two runs give equal bits."""
    rhs = tfd().rhs
    mod = rhs.CubicMLP(50, dtype=torch.float64, generator=torch.Generator().manual_seed(0)).to(DEV)
    with torch.no_grad():
        mod.b1.normal_(0, 0.1)
        mod.b2.normal_(0, 0.1)
    g = torch.Generator().manual_seed(1)
    y0 = (torch.randn(3000, 2, generator=g, dtype=torch.float64)).to(DEV)
    t = torch.linspace(0, 0.5, 4, dtype=torch.float64)
    w = torch.randn((4, 3000, 2), generator=g, dtype=torch.float64).to(DEV)
    calls = _count_forward(mod)
    res = []
    for extra in ({}, {}, {"fused_rhs": False}):
        for p in mod.parameters():
            p.grad = None
        y = y0.clone().requires_grad_(True)
        ys = tfd().odeint(mod, y, t, rtol=1e-8, atol=1e-10, method="dopri5", options=dict(extra, backprop=True))
        before = calls[0]
        (ys * w).sum().backward()
        if not extra:
            assert calls[0] == before == 0
        res.append([y.grad] + [p.grad.clone() for p in mod.parameters()])
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)
    for a, b in zip(res[0], res[2]):
        assert _rel(a.cpu().numpy(), b.cpu().numpy()) <= 1e-10


def _expected_launches(method, steps, builtin):
    """2s + 1 per step (generic) or 2s + 2 (built-in: s evaluations, s - 1 + 1 fused VJPs), less the combines whose every
    term has a zero coefficient; adaptive Heun: its f0 is carried, not evaluated (one combine instead of one call)."""
    from tfdiffeq_b200 import tableaus as tb
    from tfdiffeq_b200.backprop import _FIXED_TAB
    if method in ("dopri5", "bosh3", "dopri8", "adaptive_heun"):
        tab = tb.TABLEAUS[method]
        beta, c_sol, fsal, s = tab.beta, tab.c_sol, tab.fsal, tab.n_k
        mask = {0, s - 1} | {j for j in range(s) if tab.c_mid[j] != 0.0}
    else:
        beta, c_sol = _FIXED_TAB[method]
        fsal, s, mask = False, len(c_sol), set()
    lc = beta[s - 2] if fsal else c_sol
    live = [any(beta[l][j] != 0.0 for l in range(j, s - 1)) or (j < len(lc) and lc[j] != 0.0) for j in range(s)]
    carry = method == "adaptive_heun"
    total = 0
    for n in range(steps):
        fresh = not carry or n == 0
        per = 2                                                # dense VJP, lambda_n
        if builtin:
            per += s if fresh else s - 1                       # evaluations (b2ode_bp_rhs, mode EVAL)
            per += sum(1 for j in range(1, s) if live[j] or j in mask)     # fused VJPs
            per += (1 if live[0] or 0 in mask else 0) if fresh else (1 if live[0] else 0)   # f0: VJP, or the carry
        else:
            per += s - 1                                       # stage inputs (every row has a non-zero weight)
            per += sum(1 for j in range(s) if live[j])         # reverse combines
        if carry and n < steps - 1:
            per += 1                                           # the carry added into mu_{s-1}
        total += per
    return total


@pytest.mark.parametrize("method,calls_per_step,extra", [("dopri5", 7, 0), ("bosh3", 4, 0), ("dopri8", 14, 0),
                                                          ("adaptive_heun", 1, 1), ("rk4", 4, 0), ("euler", 1, 0),
                                                          ("midpoint", 2, 0)])
def test_backprop_launches_and_func_calls(method, calls_per_step, extra):
    net = Net(3, torch.float64).to(DEV)
    y0 = torch.randn(8, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    t = torch.linspace(0, 1, 4, dtype=torch.float64)
    opts = {"backprop": True, "step_size": 0.1} if method in FIXED else {"backprop": True}
    ys = tfd().odeint(net, y0, t, method=method, options=opts)
    steps = tfd().solvers.last_stats["n_accepted"]
    ys.sum().backward()
    st = tfd().backprop.last_stats
    assert st["steps"] == steps
    assert st["func_calls"] == calls_per_step * steps + extra
    assert st["launches"] == _expected_launches(method, steps, False)
    # a built-in right-hand side: no func call, the documented launches
    lz = tfd().rhs.Lorenz()
    y1 = (torch.randn(8, 3, dtype=torch.float64) + 5.0).to(DEV).requires_grad_(True)
    ys = tfd().odeint(lz, y1, torch.linspace(0, 0.2, 4, dtype=torch.float64), method=method,
                      options=dict(opts, step_size=0.02) if method in FIXED else opts)
    steps = tfd().solvers.last_stats["n_accepted"]
    ys.sum().backward()
    st = tfd().backprop.last_stats
    assert st["func_calls"] == 0
    assert st["launches"] == _expected_launches(method, steps, True)


def test_backprop_memory_returns_to_baseline():
    net = Net(3, torch.float64).to(DEV)
    y0 = torch.randn(20000, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    t = torch.linspace(0, 2, 5, dtype=torch.float64)
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    ys = tfd().odeint(net, y0, t, method="dopri5", options={"backprop": True})
    held = torch.cuda.memory_allocated(DEV)
    steps = tfd().solvers.last_stats["n_accepted"]
    assert held - base >= steps * y0.numel() * 8
    ys.sum().backward()
    del ys
    y0.grad = None
    for p in net.parameters():
        p.grad = None
    gc.collect()
    torch.cuda.synchronize()
    # the checkpoints are released with the graph (allocations made before `base` may have gone too)
    assert torch.cuda.memory_allocated(DEV) <= base


def test_backprop_refusals_on_gpu_tensors():
    net = Net(3, torch.float64).to(DEV)
    y0 = torch.randn(4, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    t = torch.linspace(0, 1, 3, dtype=torch.float64)
    for method, opts in (("tsit5", {}), ("adams", {}), ("dopri5", {"cuda_graph": True})):
        with pytest.raises(ValueError):
            tfd().odeint(net, y0, t, method=method, options=dict(opts, backprop=True))
