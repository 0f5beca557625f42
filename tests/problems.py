"""Right-hand sides used by the parity tests, written once for three backends:

* ``numpy``            -> the oracle (``oracle/np_ref.py``)
* ``torch`` on CPU      -> the unmodified reference over ``oracle/tf_shim.py`` (golden generation only)
* ``torch`` on ``cuda`` -> the product (``tfdiffeq_b200``)

They restate the reference's own fixtures: ``tests/problems.py:13-68`` (ConstantODE / SineODE /
LinearODE, including the degenerate ``A == 0`` of :49), ``examples/ode_demo.py:27-35`` (y**3 spiral),
``examples/lorenz_attractor.py:20-37`` (Lorenz) and ``README.md:67-81`` (Lotka-Volterra).
Every callable is ``f(t, y)`` for a single-tensor state unless it says "tuple".
"""
import math

import numpy as np


def _xp(backend):
    if backend == "numpy":
        return np
    import torch
    return torch


def _const(backend, arr, dtype, device=None):
    arr = np.asarray(arr, dtype=np.float64)
    if backend == "numpy":
        return arr.astype(dtype)
    import torch
    tdt = {"float32": torch.float32, "float64": torch.float64}[np.dtype(dtype).name]
    return torch.tensor(arr, dtype=tdt, device=device)


class Constant(object):
    """tests/problems.py:13-25   y' = a + (y - (a t + b))**5 ,  y = a t + b."""
    a, b = 0.2, 3.0

    def __init__(self, backend="numpy", dtype="float64", device=None):
        pass

    def __call__(self, t, y):
        return self.a + (y - (self.a * t + self.b)) ** 5

    def exact(self, t):
        return self.a * np.asarray(t, dtype=np.float64) + self.b

    def y0(self, t0):
        return np.array(self.a * float(t0) + self.b)


class Sine(object):
    """tests/problems.py:28-40."""

    def __init__(self, backend="numpy", dtype="float64", device=None):
        self.xp = _xp(backend)

    def __call__(self, t, y):
        xp = self.xp
        if xp is not np and not hasattr(t, "dtype"):
            import torch
            t = torch.tensor(t, dtype=y.dtype, device=y.device)
        return 2 * y / t + t ** 4 * xp.sin(2 * t) - t ** 2 + 4 * t ** 3

    def exact(self, t):
        t = np.asarray(t, dtype=np.float64)
        return (-0.5 * t ** 4 * np.cos(2 * t) + 0.5 * t ** 3 * np.sin(2 * t) + 0.25 * t ** 2 * np.cos(2 * t)
                - t ** 3 + 2 * t ** 4 + (math.pi - 0.25) * t ** 2)

    def y0(self, t0):
        return np.array(self.exact(np.float64(t0)))


class Linear(object):
    """tests/problems.py:43-68.  ``degenerate=True`` reproduces the reference's A == 0 (ndarray.transpose(0,1)
    is a no-op, :49); ``degenerate=False`` is the skew-symmetric system that file evidently intended."""

    def __init__(self, backend="numpy", dtype="float64", device=None, dim=10, degenerate=True, seed=0):
        rng = np.random.RandomState(seed)
        U = rng.randn(dim, dim) * 0.1
        A = 2 * U - (U + U.transpose(0, 1)) if degenerate else 2 * U - (U + U.T)
        self.A_np = A
        self.A = _const(backend, A, dtype, device)
        self.dim = dim

    def __call__(self, t, y):
        return (self.A @ y.reshape(self.dim, 1)).reshape(-1)

    def y0(self, t0=None):
        return np.ones(self.dim)

    def exact(self, t):
        import scipy.linalg
        return np.stack([scipy.linalg.expm(self.A_np * float(ti)) @ np.ones(self.dim) for ti in t])


class LotkaVolterra(object):
    """README.md:67-81 / examples/UniversalNeuralODE.ipynb:235-270   a,b,c,d = 1.5,1,3,1."""

    def __init__(self, backend="numpy", dtype="float64", device=None):
        self.xp = _xp(backend)

    def __call__(self, t, y):
        x, z = y[..., 0], y[..., 1]
        return self.xp.stack([1.5 * x - 1.0 * x * z, -3.0 * z + 1.0 * x * z], -1)


class Lorenz(object):
    """examples/lorenz_attractor.py:20-37, vectorised over leading batch axes (state (..., 3))."""
    sigma, beta, rho = 10.0, 8.0 / 3.0, 28.0

    def __init__(self, backend="numpy", dtype="float64", device=None):
        self.xp = _xp(backend)

    def __call__(self, t, y):
        x, yy, z = y[..., 0], y[..., 1], y[..., 2]
        return self.xp.stack([self.sigma * (yy - x), x * (self.rho - z) - yy, x * yy - self.beta * z], -1)


class Spiral(object):
    """examples/ode_demo.py:27-35   y' = (y**3) @ A , A = [[-0.1, 2], [-2, -0.1]]."""

    def __init__(self, backend="numpy", dtype="float64", device=None):
        self.A = _const(backend, [[-0.1, 2.0], [-2.0, -0.1]], dtype, device)

    def __call__(self, t, y):
        return (y ** 3) @ self.A


class SpiralMLP(object):
    """examples/ode_demo.py:115-129   W2 tanh(W1 y**3 + b1) + b2 , 2 -> 50 -> 2 (weights N(0, 0.1), zero bias)."""

    def __init__(self, backend="numpy", dtype="float64", device=None, seed=0, hidden=50):
        rng = np.random.RandomState(seed)
        self.xp = _xp(backend)
        self.W1 = _const(backend, rng.randn(2, hidden) * 0.1, dtype, device)
        self.W2 = _const(backend, rng.randn(hidden, 2) * 0.1, dtype, device)

    def __call__(self, t, y):
        return self.xp.tanh((y ** 3) @ self.W1) @ self.W2


class TupleDecay(object):
    """tuple state of UNEQUAL shapes: (-y, -50 z); api_tests.py:24-57 style (`tuple_f`)."""

    def __init__(self, backend="numpy", dtype="float64", device=None):
        pass

    def __call__(self, t, yz):
        y, z = yz
        return (-y, -50.0 * z)


class TimeDependentTridiag(object):
    """DETEST C-class flavour (tests/DETEST/detest.py:183-202) generalised to dim n, batched over rows:
    y' = y @ T^T with T = tridiag(1, -2, 1), plus a mild explicit time dependence so `t` is exercised."""

    def __init__(self, backend="numpy", dtype="float64", device=None, dim=16):
        T = -2.0 * np.eye(dim) + np.eye(dim, k=1) + np.eye(dim, k=-1)
        self.Tt = _const(backend, T.T, dtype, device)

    def __call__(self, t, y):
        return y @ self.Tt + 0.01 * t


class BatchedLinear(object):
    """SURVEY 8(d) row K, the north-star kernel microbenchmark: y' = y @ A on a (batch, dim) state with
    A = -0.5 I + 0.05 N(0,1) (seeded), i.e. tests/problems.py:43-68's LinearODE batched over rows."""

    def __init__(self, backend="numpy", dtype="float64", device=None, dim=128, seed=0):
        rng = np.random.default_rng(seed)
        self.A = _const(backend, -0.5 * np.eye(dim) + 0.05 * rng.standard_normal((dim, dim)), dtype, device)

    def __call__(self, t, y):
        return y @ self.A


class ExactLinear(object):
    """The north-star system y' = y @ A with every product exact: A = d I + P diag(sgn), P a seeded permutation without
    fixed points and sgn = +-s, i.e. column j holds d on the diagonal and sgn[j] in row src[j] != j.  With d and s powers
    of two every product y_k A_kj is exact and the zero products add nothing, so each output is the single correctly
    rounded sum round(d y_j + sgn_j y_src[j]) whatever the summation order (FMA, split-K, tensor cores); only the sign
    of an exact zero may differ.  The numpy backend computes that two-term gather form, the torch backend ``y @ A``;
    ``A_np`` (float64) is the matrix for ``rhs.LinearODE``."""

    def __init__(self, backend="numpy", dtype="float64", device=None, dim=128, seed=0, d=-0.5, s=1.0 / 16):
        rng = np.random.default_rng(seed)
        perm = rng.permutation(dim)
        while dim > 1 and np.any(perm == np.arange(dim)):
            perm = rng.permutation(dim)
        sgn = np.where(rng.random(dim) < 0.5, -s, s)
        self.src = np.empty(dim, dtype=np.int64)
        self.src[perm] = np.arange(dim)                    # column j takes y[src[j]]
        A = d * np.eye(dim)
        A[self.src, np.arange(dim)] += sgn
        self.A_np, self.dim, self.backend = A, dim, backend
        self.d = np.dtype(dtype).type(d)
        self.sgn = sgn.astype(dtype)
        self.A = _const(backend, A, dtype, device)

    def __call__(self, t, y):
        if self.backend == "numpy":
            return y * self.d + y[..., self.src] * self.sgn
        return y @ self.A


class Kepler(object):
    """DETEST D-class (tests/DETEST/detest.py:263-283) stacked: `orbits` two-body orbits per row, state (..., 4 * orbits)
    laid out [x, y, vx, vy] per orbit; eccentricities spread over 0.1 .. 0.9 (BASELINE config 5's reject-stress system:
    32 orbits = dim 128).  `y0(batch, seed)` perturbs the reference initial data [1-e, 0, 0, sqrt((1+e)/(1-e))]."""

    def __init__(self, backend="numpy", dtype="float64", device=None, orbits=32):
        self.xp, self.orbits = _xp(backend), orbits

    def __call__(self, t, y):
        xp = self.xp
        s = y.reshape(y.shape[:-1] + (self.orbits, 4))
        x, yy, vx, vy = s[..., 0], s[..., 1], s[..., 2], s[..., 3]
        r3 = (x * x + yy * yy) ** 1.5
        return xp.stack([vx, vy, -x / r3, -yy / r3], -1).reshape(y.shape)

    def y0(self, batch, seed=0):
        ecc = 0.1 + 0.8 * np.arange(self.orbits) / max(self.orbits - 1, 1)
        base = np.stack([1 - ecc, np.zeros_like(ecc), np.zeros_like(ecc), np.sqrt((1 + ecc) / (1 - ecc))], -1).reshape(-1)
        rng = np.random.default_rng(seed)
        return base[None, :] * (1.0 + 0.01 * rng.standard_normal((batch, base.size)))


class Detest(object):
    """One problem of the reference's DETEST benchmark (tests/DETEST/detest.py), see tests/detest_problems.py."""

    def __init__(self, backend="numpy", dtype="float64", device=None, name="B1"):
        from detest_problems import make
        self.f, self.y0, self.exact = make(name, _xp(backend), device)

    def __call__(self, t, y):
        return self.f(t, y)


PROBLEMS = {"batched_linear": BatchedLinear, "exact_linear": ExactLinear, "kepler": Kepler, "detest": Detest, "constant": Constant, "sine": Sine, "linear": Linear, "lv": LotkaVolterra, "lorenz": Lorenz,
            "spiral": Spiral, "spiral_mlp": SpiralMLP, "tuple_decay": TupleDecay, "tridiag": TimeDependentTridiag}
