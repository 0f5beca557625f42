"""GPU: the linear right-hand side y' = y @ A on the fp64 tensor cores (rhs.LinearODE, b2ode_linear_f64).

The kernel against the fp64 CPU product, its stage combine against the stage kernel's operation order, the row
independence the bit-identity contract rests on, and whole solves: against the oracle, fused against unfused (bit for
bit, both time directions, every adaptive tableau, eager and CUDA graph), against the same system through cuBLAS, the
plain-torch fallbacks, the adjoint's gradients and the weight cache."""
import numpy as np
import pytest
import torch

import np_ref
from problems import PROBLEMS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -53


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _matrix(D, seed=0):
    rng = np.random.default_rng(seed)
    return -0.5 * np.eye(D) + 0.05 * rng.standard_normal((D, D))


def _state_with_dt(dt):
    from tfdiffeq_b200 import _lib
    st = _lib.State()
    st.dt = dt
    return torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(DEV)


def _linear(x, A, stage=None, sign=1.0):
    return tfd().rhs.linear_f64(x, A, sign, stage=stage)


@pytest.mark.parametrize("D", [16, 32, 64, 96, 128])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 1000, 65536])
def test_kernel_accuracy_against_fp64_product(D, M):
    rng = np.random.default_rng(D * 7 + M)
    A = _matrix(D, seed=D)
    Y = rng.standard_normal((M, D))
    got = _linear(torch.tensor(Y, device=DEV), torch.tensor(A, device=DEV)).cpu().numpy()
    ref = Y @ A
    bound = 2 * D * U * (np.abs(Y) @ np.abs(A))
    assert np.all(np.abs(got - ref) <= bound), float(np.max(np.abs(got - ref) / bound))


def _np_combine(y0, ks, coefs, dt):
    """k_rk_stage's order restated in numpy (IEEE multiplies and adds, no contraction)."""
    c = [dt * b for b in coefs]
    acc = c[0] * ks[0]
    for cj, kj in zip(c[1:], ks[1:]):
        acc = acc + cj * kj
    return y0 + acc


@pytest.mark.parametrize("nk", range(14))
def test_fused_stage_combine_is_bit_identical(nk):
    """Every NK instantiation (0 .. 13), at M = 4099 and at an M that gives every warp of the persistent grid at least
    three 16-row blocks (the NK <= 1 path prefetches the next block's first chunk)."""
    from tfdiffeq_b200 import tableaus
    D = 128
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    rng = np.random.default_rng(nk)
    if 1 <= nk <= 5:
        coefs = list(tableaus.DOPRI5.beta[nk - 1])          # dopri5 rows 0, 1, 2, 3, 4 have 1..5 nonzero terms
        assert len(coefs) == nk and all(b != 0.0 for b in coefs)
    else:
        coefs = list(rng.standard_normal(nk))
    dt = 0.0123456789
    A = torch.tensor(_matrix(D), device=DEV)
    state = _state_with_dt(dt)
    for M in (4099, 3 * 16 * 8 * sms + 5):
        y0 = rng.standard_normal((M, D))
        ks = [rng.standard_normal((M, D)) for _ in range(nk)]
        y0_d, ks_d = torch.tensor(y0, device=DEV), [torch.tensor(k, device=DEV) for k in ks]
        ys = torch.empty_like(y0_d)
        out = _linear(y0_d, A, stage=(ks_d, coefs, state.data_ptr(), ys))
        if nk:
            want_y = _np_combine(y0, ks, coefs, dt)
            assert np.array_equal(ys.cpu().numpy(), want_y)
            assert torch.equal(out, _linear(ys, A))
        else:
            assert torch.equal(out, _linear(y0_d, A))
        # without ystage the product is the same
        assert torch.equal(out, _linear(y0_d, A, stage=(ks_d, coefs, state.data_ptr(), None)))
        # the negated image gives the negated product
        assert torch.equal(-out, _linear(y0_d, A, stage=(ks_d, coefs, state.data_ptr(), None), sign=-1.0))


def test_rows_are_independent_of_the_batch():
    D = 128
    rng = np.random.default_rng(11)
    Y = torch.tensor(rng.standard_normal((1000, D)), device=DEV)
    A = torch.tensor(_matrix(D), device=DEV)
    full = _linear(Y, A)
    for r in (0, 1, 15, 16, 17, 500, 999):
        assert torch.equal(full[r:r + 1], _linear(Y[r:r + 1].contiguous(), A)), r
    part = _linear(Y[37:337].contiguous(), A)
    assert torch.equal(full[37:337], part)
    big = torch.cat([Y, Y, Y[:5]])
    assert torch.equal(_linear(big, A)[1000:2000], full)


def _bench_y0(rows, dim=128):
    return np.random.default_rng(100).standard_normal((rows, dim))


def test_solve_matches_oracle():
    rows, dim = 2048, 128
    f_np = PROBLEMS["batched_linear"](backend="numpy", dim=dim, seed=0)
    y0 = _bench_y0(rows, dim)
    t = np.linspace(0., 2., 11)
    st = np_ref.Stats()
    ref = np_ref.odeint(f_np, y0, t, rtol=1e-6, atol=1e-9, method="dopri5", stats=st)
    f = tfd().rhs.LinearODE(f_np.A).to(DEV)
    got = tfd().odeint(f, torch.tensor(y0, device=DEV), torch.tensor(t), rtol=1e-6, atol=1e-9, method="dopri5")
    s = dict(tfd().last_stats)
    assert s["stage_func"]
    assert float(np.max(np.abs(got.cpu().numpy() - ref))) <= 1e-6
    assert (s["n_accepted"], s["n_rejected"], s["nfe"]) == (st.n_acc, st.n_rej, st.nfe)
    assert f.nfe == s["nfe"]


# every adaptive tableau: the ones with stages between the first and the last form those stages inside the kernel
@pytest.mark.parametrize("method,kw", [("dopri5", {}), ("bosh3", {}), ("tsit5", {}), ("dopri8", dict(rtol=1e-9, atol=1e-9)),
                                       ("adaptive_heun", dict(rtol=1e-4, atol=1e-6))])
@pytest.mark.parametrize("reverse", [False, True])
def test_fused_equals_unfused(method, kw, reverse):
    from tfdiffeq_b200 import tableaus
    rows, dim = 4099, 64
    f = tfd().rhs.LinearODE(_matrix(dim, seed=3)).to(DEV)
    y0 = torch.tensor(_bench_y0(rows, dim), device=DEV)
    t = torch.tensor(np.linspace(0., 1., 6)[::-1].copy() if reverse else np.linspace(0., 1., 6))
    kw = dict(dict(rtol=1e-6, atol=1e-9), **kw)
    a = tfd().odeint(f, y0, t, method=method, **kw)
    sa = dict(tfd().last_stats)
    b = tfd().odeint(f, y0, t, method=method, options={"fused_rhs": False}, **kw)
    sb = dict(tfd().last_stats)
    c = tfd().odeint(f, y0, t, method=method, options={"cuda_graph": True}, **kw)
    sc = dict(tfd().last_stats)
    assert sa["stage_func"] == (tableaus.TABLEAUS[method].n_k > 2)
    assert not sb["stage_func"]
    assert sc["cuda_graph"] and sc["stage_func"] == sa["stage_func"]
    assert (sa["n_accepted"], sa["n_rejected"], sa["nfe"]) == (sb["n_accepted"], sb["n_rejected"], sb["nfe"])
    assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())
    assert np.array_equal(a.cpu().numpy(), c.cpu().numpy())


def test_against_cublas_at_northstar_size():
    f_t = PROBLEMS["batched_linear"](backend="torch", device=DEV, dim=128, seed=0)
    f = tfd().rhs.LinearODE(PROBLEMS["batched_linear"](backend="numpy", dim=128, seed=0).A).to(DEV)
    y0 = torch.tensor(_bench_y0(65536), device=DEV)
    t = torch.tensor(np.linspace(0., 2., 11))
    kw = dict(rtol=1e-6, atol=1e-9, method="dopri5")
    a = tfd().odeint(f, y0, t, **kw)
    sa = dict(tfd().last_stats)
    b = tfd().odeint(f_t, y0, t, **kw)
    sb = dict(tfd().last_stats)
    assert sa["stage_func"] and not sb["stage_func"]
    assert (sa["n_accepted"], sa["n_rejected"], sa["nfe"]) == (sb["n_accepted"], sb["n_rejected"], sb["nfe"])
    assert float((a - b).abs().max()) <= 1e-9


@pytest.mark.parametrize("case", ["fp32", "D12", "D256", "autograd"])
def test_plain_torch_fallbacks(case):
    D = {"D12": 12, "D256": 256}.get(case, 128)
    dtype = torch.float32 if case == "fp32" else torch.float64
    f = tfd().rhs.LinearODE(_matrix(D), dtype=dtype).to(DEV)
    y = torch.tensor(np.random.default_rng(5).standard_normal((300, D)), device=DEV, dtype=dtype)
    if case == "autograd":
        assert not f.uses_tensor_cores(y.requires_grad_(True))
        out = f(0.0, y)
        assert out.requires_grad
        assert torch.equal(out.detach(), (y @ f.A).detach())
        return
    with torch.no_grad():
        assert not f.uses_tensor_cores(y)
        assert torch.equal(f(0.0, y), y @ f.A)
    sol = tfd().odeint(f, y, torch.tensor([0., 0.5]), method="dopri5")
    assert not tfd().last_stats["stage_func"] and torch.isfinite(sol).all()


class _PlainLinear(torch.nn.Module):
    def __init__(self, A):
        super(_PlainLinear, self).__init__()
        self.A = torch.nn.Parameter(torch.tensor(A))

    def forward(self, t, y):
        return y @ self.A


def test_adjoint_gradients_match_plain_module():
    D, rows = 32, 64
    A = _matrix(D, seed=9)
    y0_np = np.random.default_rng(9).standard_normal((rows, D))
    t = torch.tensor(np.linspace(0., 1., 5))
    grads = []
    for f in (tfd().rhs.LinearODE(A).to(DEV), _PlainLinear(A).to(DEV)):
        y0 = torch.tensor(y0_np, device=DEV, requires_grad=True)
        sol = tfd().odeint_adjoint(f, y0, t, rtol=1e-9, atol=1e-12, method="dopri5")
        (sol ** 2).sum().backward()
        grads.append((f.A.grad.detach().cpu().numpy(), y0.grad.detach().cpu().numpy()))
    for g_lin, g_plain in zip(*grads):
        np.testing.assert_allclose(g_lin, g_plain, rtol=1e-7, atol=1e-10)


def test_in_place_update_of_A_is_seen_by_the_next_solve():
    D = 64
    f = tfd().rhs.LinearODE(_matrix(D, seed=1)).to(DEV)
    y0 = torch.tensor(_bench_y0(500, D), device=DEV)
    t = torch.tensor(np.linspace(0., 1., 3))
    before = tfd().odeint(f, y0, t, method="dopri5")
    with torch.no_grad():
        f.A.mul_(0.5)                                      # bumps A's version counter
    after = tfd().odeint(f, y0, t, method="dopri5")
    assert tfd().last_stats["stage_func"]
    fresh = tfd().rhs.LinearODE(0.5 * _matrix(D, seed=1)).to(DEV)
    want = tfd().odeint(fresh, y0, t, method="dopri5")
    assert not torch.equal(before, after)
    assert torch.equal(after, want)
