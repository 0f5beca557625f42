"""LatentODEFunc (examples/latent_ode.py's network) per evaluation: a 60-digit reference and a forward error bound.

``reference(mod, y, g)`` evaluates f(y) and the vector-Jacobian product g^T df/dy of the module in mpmath at 60 digits
from the module's weights and the given rows (both read exactly from their binary values).  ``bound(...)`` is a bound on
the error of any evaluation in the state dtype that sums every dot product (bias last) in any order, with elu through
expm1 and its derivative through exp -- the kernels' operation order and torch's cuBLAS / autograd alike:
  * a sum of k rounded terms is off by at most gamma_k * sum |terms|, gamma_k = k u / (1 - k u), u = eps / 2;
  * elu and elu' are Lipschitz with constant 1, so an input error passes through unamplified, and expm1 / exp add at
    most MATH_ULPS ulps of the result (CUDA Programming Guide: expm1f 1, expf 2, expm1 1, exp 1; glibc's are within 1);
  * products of two perturbed values add |x| e_y + |y| e_x + e_x e_y, and one rounding.
Everything is propagated layer by layer in float64 from the reference's magnitudes, and scaled by 1.05 for the
second-order terms the propagation rounds away."""
import mpmath
import numpy as np
import torch

MATH_ULPS = 2          # expm1 / exp, either precision (the largest documented bound, expf's)


def weights(mod):
    """(W1, b1, W2, b2, W3, b3) as float64 numpy arrays (exact images of the module's parameters)."""
    return tuple(p.detach().cpu().double().numpy() for p in
                 (mod.fc1.weight, mod.fc1.bias, mod.fc2.weight, mod.fc2.bias, mod.fc3.weight, mod.fc3.bias))


def _mp(a):
    return [mpmath.mpf(float(v)) for v in np.asarray(a, dtype=np.float64).ravel()]


def reference(mod, y, g):
    """f and g^T df/dy of every row of ``y`` / ``g`` ((n, 4) arrays), plus the intermediates the bound needs, as float64
    arrays rounded from 60 digits: dict(f, gy, a1, z1, a2, z2, t, d2, s, d1)."""
    W1, b1, W2, b2, W3, b3 = weights(mod)
    H = W1.shape[0]
    out = {k: [] for k in ("f", "gy", "a1", "z1", "a2", "z2", "t", "d2", "s", "d1")}
    with mpmath.workdps(60):
        w1 = [_mp(W1[i]) for i in range(H)]
        w2 = [_mp(W2[j]) for j in range(H)]
        w3 = [_mp(W3[d]) for d in range(4)]
        bb1, bb2, bb3 = _mp(b1), _mp(b2), _mp(b3)
        one = mpmath.mpf(1)
        for yr, gr in zip(np.asarray(y, dtype=np.float64), np.asarray(g, dtype=np.float64)):
            yy, gg = _mp(yr), _mp(gr)
            a1 = [mpmath.fsum(yy[d] * w1[i][d] for d in range(4)) + bb1[i] for i in range(H)]
            z1 = [a if a > 0 else mpmath.expm1(a) for a in a1]
            a2 = [mpmath.fsum(z1[i] * w2[j][i] for i in range(H)) + bb2[j] for j in range(H)]
            z2 = [a if a > 0 else mpmath.expm1(a) for a in a2]
            f = [mpmath.fsum(z2[j] * w3[d][j] for j in range(H)) + bb3[d] for d in range(4)]
            t = [mpmath.fsum(w3[d][j] * gg[d] for d in range(4)) for j in range(H)]
            d2 = [t[j] * (one if a2[j] > 0 else mpmath.exp(a2[j])) for j in range(H)]
            s = [mpmath.fsum(w2[j][i] * d2[j] for j in range(H)) for i in range(H)]
            d1 = [s[i] * (one if a1[i] > 0 else mpmath.exp(a1[i])) for i in range(H)]
            gy = [mpmath.fsum(w1[i][d] * d1[i] for i in range(H)) for d in range(4)]
            for k, v in (("f", f), ("gy", gy), ("a1", a1), ("z1", z1), ("a2", a2), ("z2", z2), ("t", t), ("d2", d2),
                         ("s", s), ("d1", d1)):
                out[k].append([float(x) for x in v])
    return {k: np.array(v, dtype=np.float64) for k, v in out.items()}


def _gamma(k, eps):
    u = eps / 2
    return k * u / (1 - k * u)


def bound(mod, y, g, ref, dtype):
    """(bound on |f - f_ref|, bound on |gy - gy_ref|), each (n, 4), for evaluations in ``dtype`` (a numpy dtype name)."""
    eps = float(np.finfo(dtype).eps)
    W1, b1, W2, b2, W3, b3 = (np.abs(w) for w in weights(mod))
    H = W1.shape[0]
    y, g = np.abs(np.asarray(y, dtype=np.float64)), np.abs(np.asarray(g, dtype=np.float64))
    a1, z1, a2, z2 = ref["a1"], np.abs(ref["z1"]), ref["a2"], np.abs(ref["z2"])
    e1, e2 = np.where(a1 > 0, 1.0, np.exp(np.minimum(a1, 0))), np.where(a2 > 0, 1.0, np.exp(np.minimum(a2, 0)))
    t, d2, s, d1 = np.abs(ref["t"]), np.abs(ref["d2"]), np.abs(ref["s"]), np.abs(ref["d1"])
    fn = MATH_ULPS * eps
    E_a1 = _gamma(5, eps) * (y @ W1.T + b1)
    E_z1 = E_a1 + fn * z1
    E_a2 = E_z1 @ W2.T + _gamma(H + 1, eps) * ((z1 + E_z1) @ W2.T + b2)
    E_z2 = E_a2 + fn * z2
    E_f = E_z2 @ W3.T + _gamma(H + 1, eps) * ((z2 + E_z2) @ W3.T + b3)
    E_t = _gamma(4, eps) * (g @ W3)
    E_e2 = E_a2 + fn * e2
    E_d2 = e2 * E_t + (t + E_t) * E_e2 + eps * (d2 + e2 * E_t + (t + E_t) * E_e2)
    E_s = E_d2 @ W2 + _gamma(H, eps) * ((d2 + E_d2) @ W2)
    E_e1 = E_a1 + fn * e1
    E_d1 = e1 * E_s + (s + E_s) * E_e1 + eps * (d1 + e1 * E_s + (s + E_s) * E_e1)
    E_gy = E_d1 @ W1 + _gamma(H, eps) * ((d1 + E_d1) @ W1)
    tiny = float(np.finfo(dtype).tiny)
    return 1.05 * E_f + 4 * tiny, 1.05 * E_gy + 4 * tiny


def torch_eval(mod, y, g, dtype=torch.float64, device="cpu"):
    """The module's forward and autograd VJP on ``device``: (f, gy) as float64 numpy arrays."""
    yt = torch.as_tensor(y, dtype=dtype, device=device).clone().requires_grad_(True)
    gt = torch.as_tensor(g, dtype=dtype, device=device)
    f = mod(torch.zeros((), dtype=dtype, device=device), yt)
    gy, = torch.autograd.grad(f, yt, gt)
    return f.detach().cpu().double().numpy(), gy.detach().cpu().double().numpy()


def rows(n, std, seed, dtype=np.float64):
    """n rows of latent states and cotangents: mixed scales, so that both elu branches occur in both layers."""
    rng = np.random.default_rng(seed)
    y = rng.standard_normal((n, 4)) * np.exp(rng.uniform(-2.0, 1.5, (n, 1)))
    g = rng.standard_normal((n, 4))
    return y.astype(dtype), g.astype(dtype)


def module(hidden, std, dtype, seed):
    """A LatentODEFunc with default-initialised weights rescaled so that their standard deviation is ``std``."""
    import tfdiffeq_b200 as tfd
    gen = torch.Generator().manual_seed(seed)
    mod = tfd.rhs.LatentODEFunc(hidden=hidden, dtype=dtype, generator=gen)
    with torch.no_grad():
        for p in mod.parameters():
            p.copy_(torch.randn(p.shape, dtype=dtype, generator=gen) * std)
    return mod


# --------------------------------------------------------------------------------------------------
# solves under the exact step schedule (tests/exact_schedule.py): the oracle's right-hand side is the device's own
# evaluation on the GPU and the torch module's forward in the CPU check of the premises
# --------------------------------------------------------------------------------------------------
SOLVE_TOL = {("dopri5", "float64"): (1e-8, 1e-10), ("dopri8", "float64"): (1e-8, 1e-10),
             ("dopri5", "float32"): (1e-4, 1e-6), ("dopri8", "float32"): (1e-4, 1e-6)}
SOLVE_FIRST_STEP = 0.5
SOLVE_HORIZON = 2.0          # forward; reverse time goes half as far
FIXED_STEP = 0.013           # not a divisor of the output spacing: interpolated rows


def solve_module(dtype):
    """H = 20 at weight std 0.5 with non-zero biases (CPU, in the state dtype)."""
    return module(20, 0.5, torch.float64 if dtype == "float64" else torch.float32, seed=11)


def solve_setup(method, dtype, reverse):
    """(y0, t, rtol, atol, options) of an adaptive case: 64 rows, the exact schedule's options and output grid."""
    import exact_schedule as es
    y0 = np.random.default_rng(31).standard_normal((64, 4)).astype(dtype)
    h = SOLVE_HORIZON / (2.0 if reverse else 1.0)
    t = es._t_grid(h, (h / 2,), 5)
    rtol, atol = SOLVE_TOL[method, dtype]
    return y0, (-t if reverse else t), rtol, atol, dict(es.OPTIONS, first_step=SOLVE_FIRST_STEP)


def fixed_setup(dtype, reverse):
    y0 = np.random.default_rng(32).standard_normal((64, 4)).astype(dtype)
    t = np.linspace(0.0, 0.1, 6)
    return y0, (-t if reverse else t), dict(step_size=FIXED_STEP)


def torch_rhs(mod):
    """f(t, y) of the module's forward on the CPU, for numpy states (the stand-in of the device's evaluation)."""
    def f(t, y):
        with torch.no_grad():
            return mod(None, torch.from_numpy(np.ascontiguousarray(y))).numpy()
    return f


SOLVE_CASES = [(m, dt, rev) for m in ("dopri5", "dopri8") for dt in ("float64", "float32") for rev in (False, True)]
