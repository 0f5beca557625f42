"""GPU: odeint(..., options={'independent_rows': True, 'backprop': True}) -- every row's accepted steps reversed in one
launch of k_rows_bp.  Row r's y0 gradient must equal, bit for bit, the shared-step backprop path (stage kernels) run on
that row alone, and the oracle's discrete gradient (autograd through np_ref with the schedule held constant) within
1e-9 (fp64) / 1e-3 (fp32) relative; the forward is the plain rows solve, bit for bit.  A trainable CubicMLP's weight
gradients are the sum over rows of the single-row ones."""
import copy
import gc

import numpy as np
import pytest
import torch

import exact_schedule as es
import rows_cases as rc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TDT = {"float32": torch.float32, "float64": torch.float64}


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(1e-300, float(np.max(np.abs(b)))))


def _builtin(problem):
    r = tfd().rhs
    return {"lorenz": r.Lorenz, "lv": r.LotkaVolterra, "kepler": r.Kepler}[problem]()


def _launches():
    return tfd()._lib.lib.b2ode_launch_count()


def _rows_backprop(func, y0, t, method, rtol, atol, w, **opts):
    """(solution, y0.grad, parameter grads, forward last_stats, backprop last_stats, launches of the backward pass)."""
    y = y0.detach().clone().requires_grad_(True)
    for p in func.parameters():
        p.grad = None
    ys = tfd().odeint(func, y, t, rtol=rtol, atol=atol, method=method,
                      options=dict(opts, independent_rows=True, backprop=True))
    st = dict(tfd().solvers.last_stats)
    n0 = _launches()
    (ys * w).sum().backward()
    n = _launches() - n0
    return (ys.detach(), y.grad, [None if p.grad is None else p.grad.clone() for p in func.parameters()], st,
            dict(tfd().backprop.last_stats), n)


def _single_row(func, y_row, t, method, rtol, atol, w_row, with_sol=False, **opts):
    """The shared-step backprop path on one row alone: (y0.grad, parameter grads, n_accepted[, solution])."""
    y = y_row.detach().clone().requires_grad_(True)
    for p in func.parameters():
        p.grad = None
    ys = tfd().odeint(func, y, t, rtol=rtol, atol=atol, method=method, options=dict(opts, backprop=True))
    acc = tfd().solvers.last_stats["n_accepted"]
    (ys * w_row).sum().backward()
    res = (y.grad, [None if p.grad is None else p.grad.clone() for p in func.parameters()], acc)
    return res + (ys.detach(),) if with_sol else res


def _oracle(func, y_row, t, method, rtol, atol, w_row, options):
    """Autograd through np_ref on torch-CPU copies of func and the row: (y0 grad, parameter grads)."""
    import np_ref
    cpu = copy.deepcopy(func).cpu()
    y = y_row.detach().cpu().clone().requires_grad_(True)
    tdt = y.dtype

    def f(tt, v):
        return cpu(torch.tensor(float(tt), dtype=tdt), v)
    sol = np_ref.odeint(f, y, np.asarray(t, dtype=np.float64), rtol=rtol, atol=atol, method=method, options=options)
    ps = [p for p in cpu.parameters() if p.requires_grad]
    gs = torch.autograd.grad((sol * w_row.cpu()).sum(), [y] + ps)
    return gs[0], list(gs[1:])


def _oracle_counts(func, y_row, t, method, rtol, atol, options):
    import np_ref
    cpu = copy.deepcopy(func).cpu()
    st = np_ref.Stats()
    with torch.no_grad():
        np_ref.odeint(lambda tt, v: cpu(torch.tensor(float(tt), dtype=v.dtype), v), y_row.detach().cpu(),
                      np.asarray(t, dtype=np.float64), rtol=rtol, atol=atol, method=method, options=options, stats=st)
    return st.n_acc


def _case_opts(case):
    return dict(es.OPTIONS, first_step=case.first_step)


@pytest.mark.parametrize("name", [c.name for c in rc.CASES])
def test_rows_backprop_equals_the_single_row_path_and_the_oracle(name):
    case = rc.ALL[name]
    pool, _ = rc.pool_solves(case)
    tdt = TDT[case.dtype]
    t = torch.tensor(case.t)
    func = _builtin(case.problem)
    opts = _case_opts(case)
    g = torch.Generator().manual_seed(5)
    w_pool = torch.randn((len(case.t), len(pool), pool.shape[1]), generator=g, dtype=tdt)
    pool_t = torch.tensor(pool)
    single = []
    for p in range(len(pool)):
        gy, _, _ = _single_row(func, pool_t[p:p + 1].to(DEV), t, case.method, case.rtol, case.atol,
                               w_pool[:, p:p + 1].to(DEV), **opts)
        single.append(gy[0].cpu())
    single = torch.stack(single)
    # the oracle's discrete gradient for two pool rows (the first and a scaled one)
    tol = 1e-9 if case.dtype == "float64" else 1e-3
    for p in (0, len(pool) - 1):
        og, _ = _oracle(func, pool_t[p:p + 1], case.t, case.method, case.rtol, case.atol, w_pool[:, p:p + 1], opts)
        assert _rel(single[p].numpy(), og[0].numpy()) <= tol, (p, _rel(single[p].numpy(), og[0].numpy()))
    for n in rc.BATCHES:
        idx = rc.tile(len(pool), n)
        y0 = pool_t[idx].to(DEV)
        w = w_pool[:, idx].to(DEV)
        sol, gy, _, st, bst, launches = _rows_backprop(func, y0, t, case.method, case.rtol, case.atol, w, **opts)
        assert launches == 1 and bst["launches"] == 1 and bst["func_calls"] == 0 and bst["rows"] == n
        bad = (gy.cpu() != single[idx])
        assert not bad.any(), "n=%d: %d of %d gradient values differ (first at %s)" % (
            n, int(bad.sum()), bad.numel(), np.argwhere(bad.numpy())[0])
        plain = tfd().odeint(func, y0, t, rtol=case.rtol, atol=case.atol, method=case.method,
                             options=dict(opts, independent_rows=True))
        pst = tfd().solvers.last_stats
        assert torch.equal(sol, plain)
        for k in ("row_accepted", "row_rejected", "row_status"):
            assert torch.equal(st[k], pst[k]), k
        assert bst["steps"] == int(pst["row_accepted"].sum())


def _kepler_rows(n, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    th = torch.rand(n, generator=g, dtype=torch.float64) * 6.0
    e = 0.5 + 0.5 * torch.rand(n, generator=g, dtype=torch.float64)
    y = torch.stack([torch.cos(th), torch.sin(th), -e * torch.sin(th), e * torch.cos(th)], 1)
    return y.to(dtype)


def _mlp_rows(n, dtype, seed=0):
    # rows of very different scale: different step counts side by side in one block
    g = torch.Generator().manual_seed(seed)
    s = torch.tensor([0.1, 1.0, 3.0, 6.0], dtype=torch.float64)[torch.arange(n) % 4]
    return (s[:, None] * torch.randn(n, 2, generator=g, dtype=torch.float64)).to(dtype)


def _check_rows_against_single(func, y0, t, method, rtol, atol, seed=1, distinct=False, **opts):
    """Every row against the single-row backprop path.  The rows kernel steps like the persistent kernel, the single-row
    path like the stage kernels; their error sums can differ in the last bit, and under the ordinary controller so would
    every later dt.  Under the exact schedule (es.OPTIONS) the steps agree, so the forward solutions -- and then the
    gradients -- must agree bit for bit; a row whose forward differs (an attempt whose step factor is not a power of two)
    is held to 1e-10 (fp64) / 1e-5 (fp32) relative instead, and most rows must be bit-exact."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn((len(t),) + tuple(y0.shape), generator=g, dtype=y0.dtype)
    opts = dict(es.OPTIONS, **opts)
    sol, gy, pg, st, bst, launches = _rows_backprop(func, y0.to(DEV), t, method, rtol, atol, w.to(DEV), **opts)
    assert launches == 1 and bst["func_calls"] == 0
    acc = st["row_accepted"].cpu()
    if distinct:
        assert int(acc.min()) != int(acc.max()), "the rows should take different step counts"
    tol = 1e-10 if y0.dtype == torch.float64 else 1e-5
    sums, exact, per_row = None, 0, []
    for r in range(y0.shape[0]):
        sg, spg, sacc, ssol = _single_row(func, y0[r:r + 1].to(DEV), t, method, rtol, atol, w[:, r:r + 1].to(DEV),
                                          with_sol=True, **opts)
        assert sacc == int(acc[r])
        if torch.equal(sol[:, r:r + 1], ssol):
            assert torch.equal(gy[r:r + 1], sg), r
            exact += 1
        else:
            assert _rel(gy[r:r + 1].cpu().numpy(), sg.cpu().numpy()) <= tol, r
        per_row.append(spg)
        if spg and spg[0] is not None:
            sums = [x.double() for x in spg] if sums is None else [a + x.double() for a, x in zip(sums, spg)]
    assert exact >= y0.shape[0] // 2, (exact, y0.shape[0])
    return w, gy, pg, sums, acc, per_row


@pytest.mark.parametrize("method", ["dopri5", "dopri8"])
def test_rows_backprop_kepler(method):
    t = torch.linspace(0, 2.0, 6, dtype=torch.float64)
    _check_rows_against_single(_builtin("kepler"), _kepler_rows(19, torch.float64), t, method, 1e-6, 1e-8,
                               first_step=0.125)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_rows_backprop_frozen_cubic_mlp(dtype):
    tdt = TDT[dtype]
    mod = tfd().rhs.CubicMLP(50, dtype=tdt, generator=torch.Generator().manual_seed(0)).to(DEV)
    for p in mod.parameters():
        p.requires_grad_(False)
    t = torch.linspace(0, 1.0, 5, dtype=torch.float64)
    rtol, atol = (1e-7, 1e-9) if dtype == "float64" else (1e-4, 1e-6)
    _check_rows_against_single(mod, _mlp_rows(41, tdt), t, "dopri5", rtol, atol, first_step=0.25)


def _forward_calls(mod):
    calls = [0]
    mod.register_forward_hook(lambda *a: calls.__setitem__(0, calls[0] + 1))
    return calls


@pytest.mark.parametrize("hidden", [50, 1, 128])
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_rows_backprop_trainable_cubic_mlp(hidden, dtype):
    tdt = TDT[dtype]
    mod = tfd().rhs.CubicMLP(hidden, dtype=tdt, std=0.5, generator=torch.Generator().manual_seed(0)).to(DEV)
    with torch.no_grad():
        mod.b1.normal_(0, 0.1)
        mod.b2.normal_(0, 0.1)
    calls = _forward_calls(mod)
    t = torch.linspace(0, 1.0, 5, dtype=torch.float64)
    rtol, atol = (1e-7, 1e-9) if dtype == "float64" else (1e-4, 1e-6)
    y0 = _mlp_rows(29, tdt)
    w, gy, pg, sums, acc, per_row = _check_rows_against_single(mod, y0, t, "dopri5", rtol, atol, distinct=True,
                                                               first_step=0.25)
    opts = dict(es.OPTIONS, first_step=0.25)
    tol = 1e-10 if dtype == "float64" else 1e-5
    for a, b in zip(pg, sums):
        assert _rel(a.cpu().numpy(), b.cpu().numpy()) <= tol
    # the summed oracle gradients (autograd through np_ref, row by row).  The oracle runs on the CPU with its own matmul
    # and tanh; in fp32 that can move an accept decision and so a row's whole schedule, so fp32 compares the rows whose
    # oracle takes the engine's step count (most of them), summed on both sides, against the fp32 discrete-gradient bar
    osum, esum, same = None, None, 0
    for r in range(y0.shape[0]):
        if dtype == "float32" and _oracle_counts(mod, y0[r:r + 1], t.numpy(), "dopri5", rtol, atol, opts) != int(acc[r]):
            continue
        same += 1
        _, opg = _oracle(mod, y0[r:r + 1], t.numpy(), "dopri5", rtol, atol, w[:, r:r + 1], opts)
        osum = [x.double() for x in opg] if osum is None else [a + x.double() for a, x in zip(osum, opg)]
        esum = [x.double() for x in per_row[r]] if esum is None else [a + x.double() for a, x in zip(esum, per_row[r])]
    assert same >= y0.shape[0] // 2
    if dtype == "float64":
        assert same == y0.shape[0]
        esum = pg
    otol = 1e-10 if dtype == "float64" else 1e-3
    for a, b in zip(esum, osum):
        assert _rel(a.cpu().numpy(), b.numpy()) <= otol, _rel(a.cpu().numpy(), b.numpy())
    # deterministic, and the backward pass calls no forward
    before = calls[0]
    _, gy2, pg2, _, _, _ = _rows_backprop(mod, y0.to(DEV), t, "dopri5", rtol, atol, w.to(DEV), **opts)
    assert calls[0] == before
    assert torch.equal(gy, gy2) and all(torch.equal(a, b) for a, b in zip(pg, pg2))


def test_rows_backprop_capacity_rerun(monkeypatch):
    bp = tfd().backprop
    mod = tfd().rhs.CubicMLP(50, dtype=torch.float64, std=0.5, generator=torch.Generator().manual_seed(0)).to(DEV)
    y0 = _mlp_rows(300, torch.float64).to(DEV)
    t = torch.linspace(0, 1.0, 5, dtype=torch.float64)
    w = torch.randn((5, 300, 2), dtype=torch.float64, generator=torch.Generator().manual_seed(2)).to(DEV)
    monkeypatch.setattr(bp, "ROWS_INITIAL_SLOTS", 1 << 16)
    a = _rows_backprop(mod, y0, t, "adaptive_heun", 1e-6, 1e-8, w)
    assert a[4]["rerun"] is False
    monkeypatch.setattr(bp, "ROWS_INITIAL_SLOTS", 1)
    b = _rows_backprop(mod, y0, t, "adaptive_heun", 1e-6, 1e-8, w)
    assert b[4]["rerun"] is True
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    assert torch.equal(a[3]["row_accepted"], b[3]["row_accepted"])


def test_rows_backprop_launches():
    func = _builtin("lorenz")
    y0 = (torch.randn(500, 3, dtype=torch.float64) + torch.tensor([0.0, 0.0, 20.0], dtype=torch.float64)).to(DEV)
    # T = 1: nothing to reverse, y0.grad = w[0]
    y = y0.clone().requires_grad_(True)
    ys = tfd().odeint(func, y, torch.tensor([0.2], dtype=torch.float64), method="dopri5",
                      options={"independent_rows": True, "backprop": True})
    w = torch.randn_like(ys)
    n0 = _launches()
    (ys * w).sum().backward()
    assert _launches() == n0 and torch.equal(y.grad, w[0])
    # without grad: the plain rows solve, same bits, same launches, no graph
    t = torch.linspace(0, 0.5, 4, dtype=torch.float64)
    n0 = _launches()
    a = tfd().odeint(func, y0, t, method="dopri5", options={"independent_rows": True})
    n1 = _launches()
    b = tfd().odeint(func, y0, t, method="dopri5", options={"independent_rows": True, "backprop": True})
    n2 = _launches()
    assert torch.equal(a, b) and n1 - n0 == n2 - n1 and b.grad_fn is None
    with torch.no_grad():
        c = tfd().odeint(func, y0.clone().requires_grad_(True), t, method="dopri5",
                         options={"independent_rows": True, "backprop": True})
    assert torch.equal(a, c) and c.grad_fn is None


def test_rows_backprop_failure_message_and_memory():
    func = _builtin("lorenz")
    t = torch.linspace(0, 0.5, 4, dtype=torch.float64)
    y0 = (torch.randn(200, 3, dtype=torch.float64) + torch.tensor([0.0, 0.0, 20.0], dtype=torch.float64)).to(DEV)
    bad = y0.clone()
    bad[17, 1] = float("nan")
    msgs = []
    for extra in ({}, {"backprop": True}):
        with pytest.raises(AssertionError) as e:
            tfd().odeint(func, bad.clone().requires_grad_(True), t, method="dopri5",
                         options=dict(extra, independent_rows=True))
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and "row 17" in msgs[0]
    del e

    def run():
        y = y0.clone().requires_grad_(True)
        ys = tfd().odeint(func, y, t, method="dopri5", options={"independent_rows": True, "backprop": True})
        held = torch.cuda.memory_allocated(DEV)
        ys.sum().backward()
        return held

    run()           # the module-level last_stats / last_solver now hold what every later call leaves there
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    held = run()
    assert held - base >= int(tfd().solvers.last_stats["row_accepted"].max()) * 200 * (3 * 8 + 16)
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) <= base          # the record is released with the graph


@pytest.mark.parametrize("method", ["euler", "midpoint", "rk4", "heun"])
def test_fixed_grid_drops_the_flag(method):
    func = _builtin("lorenz")
    y0 = (torch.randn(64, 3, dtype=torch.float64) + torch.tensor([0.0, 0.0, 20.0], dtype=torch.float64)).to(DEV)
    t = torch.linspace(0, 0.2, 4, dtype=torch.float64)
    w = torch.randn((4, 64, 3), dtype=torch.float64).to(DEV)
    res = []
    for extra in ({}, {"independent_rows": True}):
        y = y0.clone().requires_grad_(True)
        ys = tfd().odeint(func, y, t, method=method, options=dict(extra, backprop=True, step_size=0.01))
        (ys * w).sum().backward()
        res.append((ys.detach(), y.grad))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_rows_backprop_at_the_benchmark_size():
    """65 536 Lorenz rows, fp64 dopri5, the ordinary controller: 64 random rows against the single-row path."""
    func = _builtin("lorenz")
    g = torch.Generator().manual_seed(0)
    n = 65536
    y0 = (torch.randn(n, 3, generator=g, dtype=torch.float64) * 5.0 +
          torch.tensor([0.0, 0.0, 25.0], dtype=torch.float64)).to(DEV)
    t = torch.linspace(0, 1.0, 11, dtype=torch.float64)
    w = torch.randn((11, n, 3), generator=g, dtype=torch.float64).to(DEV)
    sol, gy, _, st, bst, launches = _rows_backprop(func, y0, t, "dopri5", 1e-7, 1e-9, w)
    assert launches == 1
    acc = st["row_accepted"].cpu()
    for r in torch.randperm(n, generator=g)[:64].tolist():
        sg, _, sacc = _single_row(func, y0[r:r + 1], t, "dopri5", 1e-7, 1e-9, w[:, r:r + 1])
        assert sacc == int(acc[r])
        assert _rel(gy[r].cpu().numpy(), sg[0].cpu().numpy()) <= 1e-10
