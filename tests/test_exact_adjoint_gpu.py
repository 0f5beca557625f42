"""GPU: ``odeint_adjoint`` bit for bit against the restated reference adjoint (tests/exact_adjoint.py).

Under the exact step schedule, with right-hand sides whose VJPs are elementwise (or exact two-term sums), the forward
solution, ``y0.grad`` and the parameter gradients must equal the oracle's exactly; so must the counts and the final
step size of the forward solve and of every backward interval.  A trainable LinearODE's ``A.grad`` is a reduction over
rows and ``t.grad`` a sum of dot products, so those two are compared within a bound.  The first test checks the
premise the rest stand on: CUDA autograd of each module gives the bits of CPU autograd.
tests/test_exact_adjoint_cpu.py checks the schedule premises and the launch geometry the cases reach."""
import copy
import sys

import numpy as np
import pytest
import torch

import exact_adjoint as xa
import exact_schedule as es
import exact_stream as xs
from test_exact_schedule_gpu import _ratio_bar

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# t.grad against the exactly summed oracle value, relative to sum |f_i g_i| of its dot products (or |t.grad|)
T_GRAD_BOUND = {"float64": 1e-11, "float32": 1e-4}


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _adjoint_module():
    tfd()
    return sys.modules["tfdiffeq_b200.adjoint"]


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


@pytest.fixture(scope="module")
def oracle():
    """One oracle per case, shared by the tests of that case (they run consecutively)."""
    cache = {}

    def get(name):
        if name not in cache:
            cache.clear()
            cache[name] = xa.solve_case(xa.ALL[name])
        return cache[name]
    return get


def _run(case, module, y0, w):
    """The engine's adjoint on a device copy of `module`: (solution, y0 grads, parameter grads, t grad, stats)."""
    m = copy.deepcopy(module).to(DEV)
    y = tuple(torch.tensor(a, device=DEV, requires_grad=True) for a in y0)
    t = torch.tensor(case.t, dtype=torch.float64, device=DEV, requires_grad=True)
    tensor_input = case.kind != "tuple5"
    ys = tfd().odeint_adjoint(m, y[0] if tensor_input else y, t, rtol=case.rtol, atol=case.atol, method=case.method,
                              options=xa.options(case), adjoint_method=case.adjoint_method)
    ys = (ys,) if tensor_input else ys
    loss = sum((s * torch.tensor(w_, device=DEV)).sum() for s, w_ in zip(ys, w) if w_ is not None)
    loss.backward()
    stats = copy.deepcopy(_adjoint_module().last_stats)
    sol = tuple(s.detach().cpu().numpy() for s in ys)
    g_y0 = tuple(v.grad.cpu().numpy() for v in y)
    g_p = [p.grad.cpu().numpy() for p in m.parameters() if p.requires_grad]
    return sol, g_y0, g_p, t.grad.cpu().numpy(), stats


def _equal(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    bad = got != want
    assert not bad.any(), "%s: %d of %d values differ, max |diff| %.3e (first at %s)" % (
        what, int(bad.sum()), bad.size, float(np.abs(got.astype(np.float64) - want).max()), np.argwhere(bad)[0])


def _same_solve(st, s, case, method, what):
    """Counts, final step size and error ratio of an engine solve against the oracle's Solve record."""
    if method in xa.ADAPTIVE:
        assert (st["n_accepted"], st["n_rejected"], st["nfe"]) == (s.stats.n_acc, s.stats.n_rej, s.stats.nfe), (what, st)
        assert st["dt_next"] == s.dt_next, (what, st["dt_next"], s.dt_next)
        m = s.rec.m[-1]
        # a trainable A's gradient is a row reduction: when its component sets the max, m carries that rounding
        bar = 1e-9 if case.kind == "linear_trainable" else _ratio_bar(case.dtype)
        assert abs(st["error_ratio"] - m) <= bar * m, (what, st["error_ratio"], m)
    else:
        assert st["nfe"] == s.stats.nfe, (what, st["nfe"], s.stats.nfe)


# --------------------------------------------------------------------------------------------------
# the premise: CUDA autograd equals CPU autograd
# --------------------------------------------------------------------------------------------------
VJP_CASES = ["lorenz_forced-dopri5-f64-fwd-600001", "lorenz_forced-dopri5-f32-rev-750001",
             "builtin_lorenz-dopri5-f64-fwd-12627", "northstar-frozen", "linear32-trainable-rev", "linear32-external",
             "tuple5-dopri5-f64", "tuple5-dopri5-f32"]


@pytest.mark.parametrize("name", VJP_CASES)
def test_cuda_autograd_equals_cpu_autograd(name):
    """f and the VJPs w.r.t. y and every parameter, at case size, with a random full-mantissa cotangent; the time VJP
    is a reduction and is not compared.  A trainable A's VJP is a reduction over rows: 1e-12 relative."""
    case = xa.ALL[name]
    module = xa.make_module(case)
    y0 = xa.initial_state(case)
    rng = np.random.default_rng(9)
    a = tuple(rng.standard_normal(y.shape).astype(y.dtype) for y in y0)
    call = lambda m, dev: xa.tuple_call(m, case.kind != "tuple5")               # noqa: E731

    def vjp(m, dev):
        m = copy.deepcopy(m).to(dev)
        ps = [p for p in m.parameters() if p.requires_grad]
        y = tuple(torch.tensor(v, device=dev, requires_grad=True) for v in y0)
        tt = torch.tensor(0.1875, dtype=y[0].dtype, device=dev, requires_grad=True)
        f = call(m, dev)(tt, y)
        g = torch.autograd.grad(f, y + tuple(ps), tuple(-torch.tensor(v, device=dev) for v in a), allow_unused=True)
        return [x.detach().cpu().numpy() for x in f] + [None if x is None else x.cpu().numpy() for x in g]
    want, got = vjp(module, "cpu"), vjp(module, DEV)
    for i, (g, w) in enumerate(zip(got, want)):
        if w is None:
            assert g is None
        elif case.kind == "linear_trainable" and i == len(want) - 1:
            assert np.max(np.abs(g - w)) <= 1e-12 * np.max(np.abs(w)), i
        else:
            _equal(g, w, "output %d" % i)


# --------------------------------------------------------------------------------------------------
# the adjoint, bit for bit
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(xa.ALL))
def test_adjoint_is_bit_exact(name, oracle):
    case = xa.ALL[name]
    module, y0, w, res = oracle(name)
    for p in xa.schedule_premises(res, case):
        assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[case.dtype], p
    if case.rows >= 600001:
        lens = xa.augmented_lens(case, module, y0)
        g = xs.build_geom(lens, case.dtype, _sms())
        assert g.cap_exceeded and min(s.passes for s in g.segs if s.n > 1) >= 3 and g.segs[2].blocks >= 1
    sol, g_y0, g_p, g_t, st = _run(case, module, y0, w)
    for i, (g, s_) in enumerate(zip(sol, res.sol)):
        _equal(g, s_, "solution %d" % i)
    _same_solve(st["forward"], res.forward, case, case.method, "forward")
    if case.path is not None:
        # a tensor state reaches the fused paths under odeint_adjoint: the built-in right-hand side in the persistent
        # kernel or in the stage kernels, LinearODE's stage-combine producer
        fwd = st["forward"]
        assert fwd[case.path] and not any(fwd.get(k) for k in {"fused_rhs", "stage_rhs", "stage_func"} - {case.path}), fwd
    bwd = st["backward"]
    assert len(bwd) == len(case.t) - 1 == len(res.backward)
    for j, (b, s) in enumerate(zip(bwd, res.backward)):
        _same_solve(b, s, case, case.adjoint_method or case.method, "backward interval %d" % j)
    for i, (g, want) in enumerate(zip(g_y0, res.g_y0)):
        _equal(g, want, "y0[%d].grad" % i)
    assert len(g_p) == len(res.g_params)
    for i, (g, want) in enumerate(zip(g_p, res.g_params)):
        if case.kind == "linear_trainable":
            assert np.max(np.abs(g - want)) <= 1e-12 * np.max(np.abs(want)), "A.grad"
        else:
            _equal(g, want, "parameter %d grad" % i)
    scale = np.maximum(res.g_t_scale, np.abs(res.g_t))
    err = np.abs(g_t - res.g_t)
    assert np.all(err <= T_GRAD_BOUND[case.dtype] * scale), (g_t, res.g_t, float(np.max(err / scale)))

