"""The built-in right-hand sides (tfdiffeq_b200/rhs.py, csrc/b2ode_rhs.cuh) one evaluation at a time: high-precision
references, forward error bounds, input tables, and the cases of the solves that use the device's own evaluation as the
oracle's right-hand side.  Importable without a GPU; tests/test_rhs_eval_cpu.py checks the references, the bounds and the
tables, tests/test_rhs_eval_gpu.py and tests/test_exact_rhs_gpu.py use them on the device.

References.  Each system is evaluated in mpmath at DPS digits from the inputs *as stored*: the fp32 / fp64 state converted
exactly, and parameters and weights as the kernel receives them -- ``rhs_params()`` as doubles cast to the state dtype,
the weights as ``rhs_data`` casts them.  They are written from the definitions (Lorenz; Lotka-Volterra;
``-x / (x^2 + y^2)^(3/2)``; ``W2^T tanh(W1^T u + b1) + b2`` with ``u = y^3`` or ``y``), not from the kernels.

Bounds.  With u the unit roundoff of the state dtype (2^-24, 2^-53) and gamma_k = k u / (1 - k u), a value that went
through k correctly rounded operations carries a relative error of at most gamma_k, and a sum of such terms an absolute
error of at most gamma_k sum|terms| (the standard running bound, any summation order).  A library function documented to
p ulp adds a relative 2 p u (one ulp is at most 2 u relative).  The ulp figures are those of the "Mathematical Functions"
appendix of the CUDA C++ Programming Guide (maximum ulp error of the standard functions): powf 4, tanhf 2, pow 2, tanh 2
(newer editions give 1 for tanh; the larger figure is used).  Every assertion is ``|got - ref| <= bound`` with the bound
absolute, so it stays meaningful where terms cancel (Lorenz ``x y - beta z`` near zero).

* Lorenz, Lotka-Volterra: 2 or 3 operations per term, gamma_3 sum|terms|.  Their kernels are +, -, * only, so the tests
  also restate the rounding sequence in numpy (``lorenz_exact``, ``lv_exact``) and require equality; the bound ties that
  restatement to the mathematics.
* Kepler: r2 = x^2 + y^2 carries gamma_2, r2^1.5 turns that into 1.5 gamma_2 <= gamma_3, pow adds 2 p u, the division
  one more rounding: gamma_(4 + 2 p) |ref|, i.e. 6 ulp in fp32 and 4 ulp in fp64.  vx, vy are copied: bound 0.
* CubicMLP: each pre-activation a_h = u0 W1[0,h] + u1 W1[1,h] + b1[h] carries gamma_5 S_h (y^3 two roundings, product
  one, two additions), S_h the sum of the terms' magnitudes; tanh is 1-Lipschitz with slope sech^2, taken at the point of
  [a - da, a + da] nearest zero, plus 2 p u |tanh|; the output sums H products and a bias: the propagated dz_h |W2[h,j]|
  plus gamma_(H + 2) (sum |z_h W2[h,j]| + |b2[j]|).

Bounds hold while every intermediate stays in the normal range.  Rows where one does not (``regular`` False: underflow,
overflow, NaN and inf inputs) are compared by class -- NaN, +inf, -inf, +0, -0, positive, negative -- with the torch
module's ``forward`` on the CPU in the same dtype; for CubicMLP with the definition in numpy's elementwise operations,
because ``forward``'s BLAS products do not overflow where separately rounded products do.
"""
import collections
import copy

import mpmath as mp
import numpy as np

import exact_schedule as es
from problems import PROBLEMS

DPS = 60
MATH_ULPS = {"float32": {"pow": 4, "tanh": 2}, "float64": {"pow": 2, "tanh": 2}}
UNIT = {"float32": mp.mpf(2) ** -24, "float64": mp.mpf(2) ** -53}
DTYPES = ("float64", "float32")


def gamma(k, dtype):
    u = UNIT[dtype]
    return k * u / (1 - k * u)


def _mpf(a):
    """An array of the state dtype as exact mpf values (object array of the same shape)."""
    a = np.asarray(a)
    return np.array([mp.mpf(float(v)) for v in a.ravel()], dtype=object).reshape(a.shape)


def _cast(values, dtype):
    """Parameters as the kernels see them: doubles cast to the state dtype."""
    return [np.dtype(dtype).type(v) for v in values]


def classes(a):
    """Class code per element: 0 NaN, 1 +inf, 2 -inf, 3 +0, 4 -0, 5 positive, 6 negative."""
    a = np.asarray(a)
    neg = np.signbit(a)
    out = np.where(neg, 6, 5)
    out = np.where(a == 0, np.where(neg, 4, 3), out)
    out = np.where(np.isinf(a), np.where(neg, 2, 1), out)
    return np.where(np.isnan(a), 0, out)


# --------------------------------------------------------------------------------------------------
# Lorenz and Lotka-Volterra
# --------------------------------------------------------------------------------------------------
LORENZ_PARAMS = {"default": (10.0, 8.0 / 3.0, 28.0), "a": (7.3, 2.1, 33.7), "b": (12.9, 3.3, 21.4)}
LV_PARAMS = {"a": (1.3, 0.7, 2.9, 0.6), "b": (1.7, 1.9, 3.3, 0.3)}


def lorenz_exact(y, params):
    """The kernel's rounding sequence in numpy, in y's dtype: every operation is one correctly rounded +, - or *."""
    s, b, r = _cast(params, y.dtype)
    x, yy, z = y[..., 0], y[..., 1], y[..., 2]
    return np.stack([s * (yy - x), x * (r - z) - yy, x * yy - b * z], -1)


def lv_exact(y, params):
    a, b, c, d = _cast(params, y.dtype)
    x, z = y[..., 0], y[..., 1]
    return np.stack([a * x - b * x * z, -c * z + d * x * z], -1)


def ref_lorenz(y, params):
    """(reference, bound) of x' = sigma (y - x), y' = x (rho - z) - y, z' = x y - beta z."""
    dtype = y.dtype.name
    with mp.workdps(DPS):
        s, b, r = (mp.mpf(float(p)) for p in _cast(params, dtype))
        g = gamma(3, dtype)
        ref, bnd = [], []
        for x, yy, z in _mpf(y):
            ref.append([s * (yy - x), x * (r - z) - yy, x * yy - b * z])
            bnd.append([g * abs(s * (yy - x)), g * (abs(x * (r - z)) + abs(yy)), g * (abs(x * yy) + abs(b * z))])
    return np.array(ref, dtype=object), np.array(bnd, dtype=object)


def ref_lv(y, params):
    """(reference, bound) of x' = a x - b x z, z' = -c z + d x z."""
    dtype = y.dtype.name
    with mp.workdps(DPS):
        a, b, c, d = (mp.mpf(float(p)) for p in _cast(params, dtype))
        g = gamma(3, dtype)
        ref, bnd = [], []
        for x, z in _mpf(y):
            ref.append([a * x - b * x * z, -c * z + d * x * z])
            bnd.append([g * (abs(a * x) + abs(b * x * z)), g * (abs(c * z) + abs(d * x * z))])
    return np.array(ref, dtype=object), np.array(bnd, dtype=object)


def lorenz_inputs(dtype, seed=21):
    """96 rows: magnitudes from 1e-3 to 1e2 in every sign pattern, rows with z = x y / beta for each parameter set (the
    third output cancels to rounding), and the origin."""
    rng = np.random.default_rng(seed)
    y = rng.standard_normal((96, 3)) * 10.0 ** rng.uniform(-3, 2, (96, 1))
    for k, p in enumerate(LORENZ_PARAMS.values()):
        y[8 * k:8 * k + 8, 2] = y[8 * k:8 * k + 8, 0] * y[8 * k:8 * k + 8, 1] / p[1]
    y[95] = 0.0
    return y.astype(dtype)


def lv_inputs(dtype, seed=22):
    """96 rows: populations from 1e-3 to 1e2, a third of them with a negative component, rows at each parameter set's
    fixed point (c / d, a / b), where both outputs cancel, and the origin."""
    rng = np.random.default_rng(seed)
    y = np.abs(rng.standard_normal((96, 2))) * 10.0 ** rng.uniform(-3, 2, (96, 1))
    y[:32] *= rng.choice([-1.0, 1.0], (32, 2))
    for k, p in enumerate(LV_PARAMS.values()):
        y[40 + 4 * k:44 + 4 * k] = np.array([p[2] / p[3], p[0] / p[1]]) * (1 + 1e-7 * rng.standard_normal((4, 2)))
    y[95] = 0.0
    return y.astype(dtype)


# --------------------------------------------------------------------------------------------------
# Kepler
# --------------------------------------------------------------------------------------------------
def ref_kepler(y):
    """(reference, bound, regular) of [vx, vy, -x / r^3, -y / r^3] on rows of 4.  ``regular``: the row is finite and
    x^2, y^2 (unless the coordinate is zero), r^2, r^3 and the accelerations (unless zero) are all normal numbers."""
    dtype = y.dtype.name
    fi = np.finfo(y.dtype)
    with mp.workdps(DPS):
        lo, hi = mp.mpf(float(fi.tiny)), mp.mpf(float(fi.max)) / 4
        ok = lambda v, zero_ok=False: (zero_ok and v == 0) or lo <= abs(v) <= hi        # noqa: E731
        g = gamma(4 + 2 * MATH_ULPS[dtype]["pow"], dtype)
        n = y.shape[0]
        ref = np.full((n, 4), mp.nan, dtype=object)
        bnd = np.full((n, 4), mp.nan, dtype=object)
        regular = np.zeros(n, dtype=bool)
        for i in range(n):
            if not np.all(np.isfinite(y[i])):
                continue
            x, yy, vx, vy = _mpf(y[i])
            r2 = x * x + yy * yy
            if r2 == 0:
                continue
            r3 = r2 ** mp.mpf(1.5)
            ax, ay = -x / r3, -yy / r3
            ref[i] = [vx, vy, ax, ay]
            bnd[i] = [0, 0, g * abs(ax), g * abs(ay)]
            regular[i] = (ok(x * x, True) and ok(yy * yy, True) and ok(r2) and ok(r3) and ok(ax, True) and ok(ay, True))
    return ref, bnd, regular


def kepler_inputs(dtype, seed=23):
    """Rows of [x, y, vx, vy]:

    * 0..127: the orbit data of ``problems.Kepler.y0`` (y = 0 there: the x axis, both signs of x follow below) with the
      position scaled by 13 radii from 1e-3 to 1e3 and, from row 32 on, rotated by a seeded angle: all four quadrants;
    * 128..135: the axes -- x = 0 with y != 0 and y = 0 with x != 0, both signs;
    * then the edges, per dtype: r^2 normal but r^3 subnormal; r^2 subnormal; x^2 and y^2 flushed to zero; r^2 finite and
      r^3 = inf; r^2 = inf; the origin (NaN from -0 / 0, both zero signs); +-inf and NaN coordinates and velocities.
    """
    rng = np.random.default_rng(seed)
    base = PROBLEMS["kepler"](orbits=8).y0(16, seed=5).reshape(-1, 4)
    scale = 10.0 ** np.linspace(-3, 3, 13)[np.arange(128) % 13]
    th = np.where(np.arange(128) < 32, 0.0, rng.uniform(0, 2 * np.pi, 128))
    x, yy = base[:, 0] * scale, base[:, 1] * scale
    base[:, 0], base[:, 1] = x * np.cos(th) - yy * np.sin(th), x * np.sin(th) + yy * np.cos(th)
    axes = np.array([[0, 0.7], [0, -0.7], [0.7, 0], [-0.7, 0], [0.0, 3e2], [-0.0, 3e-2], [3e2, -0.0], [-3e-2, 0.0]])
    axes = np.concatenate([axes, rng.standard_normal((8, 2))], 1)
    tiny = {"float32": (1e-14, 1e-20, 1e-23), "float64": (1e-105, 1e-160, 1e-170)}[dtype]
    huge = {"float32": (1e19, 2e19), "float64": (1e154, 2e154)}[dtype]
    inf, nan = np.inf, np.nan
    edge = [[s * m, t * m * w, 0.3, -0.2] for m in tiny + huge for s in (1, -1) for t in (1, -1) for w in (0.5, 0.0)]
    edge += [[0.0, 0.0, 1.0, 2.0], [-0.0, 0.0, 1.0, 2.0], [0.0, -0.0, 1.0, 2.0], [-0.0, -0.0, 1.0, 2.0],
             [inf, 1.0, 0.0, 0.0], [-inf, 1.0, 0.0, 0.0], [1.0, inf, 0.0, 0.0], [-1.0, -inf, 0.0, 0.0],
             [inf, -inf, 0.0, 0.0], [nan, 1.0, 0.0, 0.0], [1.0, nan, 0.0, 0.0], [1.0, 1.0, nan, inf],
             [-0.5, 0.5, -inf, nan]]
    return np.concatenate([base, axes, np.array(edge)]).astype(dtype)


# --------------------------------------------------------------------------------------------------
# CubicMLP
# --------------------------------------------------------------------------------------------------
MLP_WIDTHS = (1, 2, 31, 50, 127, 128)


def mlp_module(hidden, cube=True, std=0.1, dtype="float64", seed=0):
    """rhs.CubicMLP with seeded weights at `std` and NON-ZERO biases (b1 at 3 std, b2 at std), on the CPU."""
    import torch
    from tfdiffeq_b200 import rhs
    g = torch.Generator().manual_seed(1000 * hidden + seed)
    tdt = torch.float64 if dtype == "float64" else torch.float32
    m = rhs.CubicMLP(hidden=hidden, cube=cube, std=std, dtype=tdt, generator=g)
    with torch.no_grad():
        m.b1.copy_(torch.randn(hidden, dtype=tdt, generator=g) * (3.0 * std))
        m.b2.copy_(torch.randn(2, dtype=tdt, generator=g) * std)
    return m


def mlp_as(module, dtype):
    """A copy of the module with its weights cast to the state dtype, the cast ``rhs_data`` applies: what ``forward`` must
    be given to accept a state of that dtype, and what the reference uses."""
    import torch
    return copy.deepcopy(module).to(torch.float64 if dtype == "float64" else torch.float32)


def mlp_weights(module, dtype):
    """W1 (2, H), b1 (H), W2 (H, 2), b2 (2) as numpy arrays of the state dtype."""
    m = mlp_as(module, dtype)
    return [p.detach().cpu().numpy() for p in (m.W1, m.b1, m.W2, m.b2)]


def ref_mlp(y, weights, cube):
    """(reference, bound, regular, saturated) of W2^T tanh(W1^T u + b1) + b2, u = y^3 or y.  ``regular``: the row is
    finite and |u| and 2 |u| max|W1| + max|b1| stay a quarter of the dtype's range away from overflow.  ``saturated``: rows with a
    hidden unit whose tanh rounds to +-1 in the state dtype."""
    dtype = y.dtype.name
    fi = np.finfo(y.dtype)
    W1, b1, W2, b2 = weights
    H = W1.shape[1]
    with mp.workdps(DPS):
        u_ = UNIT[dtype]
        p_tanh = 2 * MATH_ULPS[dtype]["tanh"] * u_
        ga, go = gamma(5 if cube else 3, dtype), gamma(H + 2, dtype)
        hi = mp.mpf(float(fi.max)) / 4
        mW1, mb1, mW2, mb2 = _mpf(W1), _mpf(b1), _mpf(W2), _mpf(b2)
        w1max, b1max = max(abs(v) for v in mW1.ravel()), max(abs(v) for v in mb1)
        n = y.shape[0]
        ref = np.full((n, 2), mp.nan, dtype=object)
        bnd = np.full((n, 2), mp.nan, dtype=object)
        regular, saturated = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
        for i in range(n):
            if not np.all(np.isfinite(y[i])):
                continue
            y0, y1 = _mpf(y[i])
            u0, u1 = (y0 ** 3, y1 ** 3) if cube else (y0, y1)
            if max(abs(u0), abs(u1)) > hi or 2 * max(abs(u0), abs(u1)) * w1max + b1max > hi:
                continue
            regular[i] = True
            o, do, so = [mb2[0], mb2[1]], [mp.mpf(0), mp.mpf(0)], [abs(mb2[0]), abs(mb2[1])]
            for h in range(H):
                p0, p1 = u0 * mW1[0, h], u1 * mW1[1, h]
                a = p0 + p1 + mb1[h]
                da = ga * (abs(p0) + abs(p1) + abs(mb1[h]))
                z = mp.tanh(a)
                near = max(abs(a) - da, 0)
                slope = 1 / mp.cosh(near) ** 2 if near < 200 else mp.mpf(0)
                dz = slope * da + p_tanh * (abs(z) + slope * da)
                if 1 - abs(z) < u_ / 2:
                    saturated[i] = True
                for j in range(2):
                    o[j] += z * mW2[h, j]
                    do[j] += dz * abs(mW2[h, j])
                    so[j] += (abs(z) + dz) * abs(mW2[h, j])
            ref[i] = o
            bnd[i] = [do[j] + go * so[j] for j in range(2)]
    return ref, bnd, regular, saturated


def mlp_elementwise(y, weights, cube):
    """The definition in numpy's elementwise IEEE operations of the state dtype, every product rounded on its own: the
    class reference of the rows that overflow.  A BLAS product (``forward``'s) may fuse or widen its accumulation, and so
    keep finite a sum whose first product alone overflows to inf."""
    W1, b1, W2, b2 = weights
    with np.errstate(all="ignore"):
        u = y * y * y if cube else y
        z = np.tanh(u[:, :1] * W1[0] + u[:, 1:] * W1[1] + b1)
        return (z[:, :, None] * W2).sum(1) + b2


def mlp_inputs(dtype, seed=24):
    """40 rows of [y0, y1]: magnitudes from 1e-3 to 1e2 with seeded signs, then 8 rows around the fp32 overflow of y^3
    (|y| = 1e12: y^3 = 1e36 still finite; 5e12: within a factor 3 of the largest fp32; 1e13: y^3 = inf, with equal and
    with opposite signs, where inf W - inf W gives NaN).  In fp64 the same 8 rows are ordinary large inputs."""
    rng = np.random.default_rng(seed)
    y = 10.0 ** rng.uniform(-3, 2, (32, 2)) * rng.choice([-1.0, 1.0], (32, 2))
    y[:4, 1] = y[:4, 0]
    big = np.array([[1e12, -1e12], [1e12, 3.0], [5e12, 5e12], [-5e12, 0.1], [1e13, 1e13], [1e13, -1e13], [-1e13, 1e13],
                    [0.5, -1e13]])
    return np.concatenate([y, big]).astype(dtype)


# --------------------------------------------------------------------------------------------------
# the per-evaluation cases
# --------------------------------------------------------------------------------------------------
EvalCase = collections.namedtuple("EvalCase", "name kind dtype args")

EVAL_CASES = [EvalCase("lorenz-%s-%s" % (k, d[-2:]), "lorenz", d, k) for k in LORENZ_PARAMS for d in DTYPES]
EVAL_CASES += [EvalCase("lv-%s-%s" % (k, d[-2:]), "lv", d, k) for k in LV_PARAMS for d in DTYPES]
EVAL_CASES += [EvalCase("kepler-%s" % d[-2:], "kepler", d, None) for d in DTYPES]
# every width with cube on and off; std alternates so each width meets both, and H = 50, 128 get both with the cube
_MLP = [(h, c, (0.1, 3.0)[(k + c) % 2]) for k, h in enumerate(MLP_WIDTHS) for c in (1, 0)] + [(50, 1, 3.0), (128, 1, 0.1)]
EVAL_CASES += [EvalCase("mlp-h%d-%s-std%g-%s" % (h, "cube" if c else "lin", s, d[-2:]), "mlp", d, (h, bool(c), s, d))
               for h, c, s in _MLP for d in DTYPES]
# a module built in one dtype, evaluated on a state of the other: rhs_data casts the weights
EVAL_CASES += [EvalCase("mlp-h50-built-%s-state-%s" % (b[-2:], d[-2:]), "mlp", d, (50, True, 0.1, b))
               for b, d in (("float32", "float64"), ("float64", "float32"))]
EVAL = {c.name: c for c in EVAL_CASES}

Evaluation = collections.namedtuple("Evaluation", "module y ref bound regular exact forward class_ref saturated")
_CACHE = {}


def evaluation(name):
    """Everything the tests need of one case: the module (CPU; CubicMLP modules in the dtype they were built in), the
    inputs, (reference, bound) as float64 arrays -- the bound rounded up -- the ``regular`` mask, the exact expected
    output where there is one (Lorenz, Lotka-Volterra), the torch module's CPU ``forward`` in the state dtype, and the
    values whose class the rows outside ``regular`` must have (``forward``; for CubicMLP ``mlp_elementwise``)."""
    if name in _CACHE:
        return _CACHE[name]
    import torch
    from tfdiffeq_b200 import rhs
    c = EVAL[name]
    exact, saturated = None, None
    if c.kind == "lorenz":
        module, y = rhs.Lorenz(*LORENZ_PARAMS[c.args]), lorenz_inputs(c.dtype)
        ref, bnd = ref_lorenz(y, LORENZ_PARAMS[c.args])
        regular, exact, fwd_mod = np.ones(len(y), dtype=bool), lorenz_exact(y, LORENZ_PARAMS[c.args]), module
    elif c.kind == "lv":
        module, y = rhs.LotkaVolterra(*LV_PARAMS[c.args]), lv_inputs(c.dtype)
        ref, bnd = ref_lv(y, LV_PARAMS[c.args])
        regular, exact, fwd_mod = np.ones(len(y), dtype=bool), lv_exact(y, LV_PARAMS[c.args]), module
    elif c.kind == "kepler":
        module, y = rhs.Kepler(), kepler_inputs(c.dtype)
        ref, bnd, regular = ref_kepler(y)
        fwd_mod = module
    else:
        h, cube, std, built = c.args
        module, y = mlp_module(h, cube, std, built), mlp_inputs(c.dtype)
        ref, bnd, regular, saturated = ref_mlp(y, mlp_weights(module, c.dtype), cube)
        fwd_mod = mlp_as(module, c.dtype)
    with torch.no_grad(), np.errstate(all="ignore"):
        forward = fwd_mod(0.0, torch.from_numpy(y)).numpy()
    class_ref = mlp_elementwise(y, mlp_weights(module, c.dtype), c.args[1]) if c.kind == "mlp" else forward
    to_f = lambda a, up: np.array([[float(v) * up if mp.isfinite(v) else np.nan for v in r] for r in a])     # noqa: E731
    # float() rounds the 60-digit values to nearest: 1 + 2^-50 keeps the float64 bound an upper bound
    _CACHE[name] = Evaluation(module, y, to_f(ref, 1.0), to_f(bnd, 1.0 + 2.0 ** -50), regular, exact, forward, class_ref,
                             saturated)
    return _CACHE[name]


def within_bound(got, ev):
    """Per-element |got - ref| <= bound on the regular rows, in 60-digit arithmetic's float64 image: the difference of a
    fp32 / fp64 value and the float64-rounded reference is formed in float64, whose own error (2^-53 relative to the
    reference) is far below every bound's gamma_k for fp32 and is covered for fp64 by adding one float64 ulp of ref."""
    r = ev.regular
    diff = np.abs(got[r].astype(np.float64) - ev.ref[r])
    return diff <= ev.bound[r] + np.spacing(np.abs(ev.ref[r])), diff


def device_eval(module, y, time_sign=1.0, offset=0):
    """``b2ode_rhs_eval`` the way the stage path calls it (solvers.py: descriptor from ``rhs_desc``, device scalar t, flat
    y, flat k_out): y a CUDA tensor whose last axis holds rows of the system; `offset` places y and k_out that many
    elements into their allocations.  Returns k with y's shape."""
    import ctypes as C
    import torch
    from tfdiffeq_b200 import _lib
    dev, n = y.device, y.numel()
    rd, weights = module.rhs_desc(y.dtype, dev, time_sign)
    ybuf = torch.empty(n + offset, dtype=y.dtype, device=dev)
    ybuf[offset:].copy_(y.reshape(-1))
    kbuf = torch.full((n + offset,), 12345.0, dtype=y.dtype, device=dev)
    t = torch.zeros((), dtype=y.dtype, device=dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    _lib.check(_lib.lib.b2ode_rhs_eval(_lib.F64 if y.dtype == torch.float64 else _lib.F32, C.byref(rd),
                                       C.c_void_p(t.data_ptr()), C.c_void_p(ybuf[offset:].data_ptr()),
                                       C.c_void_p(kbuf[offset:].data_ptr()), n, sms,
                                       C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    torch.cuda.current_stream(dev).synchronize()
    del weights
    assert offset == 0 or bool((kbuf[:offset] == 12345.0).all())
    return kbuf[offset:].view(y.shape)


# --------------------------------------------------------------------------------------------------
# solves under the exact step schedule (tests/exact_schedule.py) with the device's evaluation as the oracle's func
# --------------------------------------------------------------------------------------------------
# (rtol, atol) per system, tableau and dtype (float64, float32): at least one rejection and a margin on every decision
SOLVE_TOL = {
    ("kepler", "dopri5"): ((1e-6, 1e-8), (1e-4, 1e-5)),
    ("kepler", "tsit5"): ((1e-1, 1e-2), (1e-1, 1e-2)),
    ("kepler", "dopri8"): ((1e-9, 1e-11), (1e-6, 1e-7)),
    # under the reference's bosh3 tableau the oracle halves dt on these orbits until it underflows, at any tolerance
    ("kepler", "bosh3"): (None, None),
    ("kepler", "adaptive_heun"): ((1e-1, 1e-3), (1e-1, 1e-2)),
    ("mlp-h50-cube", "dopri5"): ((1e-4, 1e-6), (1e-5, 1e-6)),
    ("mlp-h50-cube", "tsit5"): ((1e-1, 1e-3), (1e-1, 1e-2)),
    ("mlp-h50-cube", "dopri8"): ((1e-3, 1e-5), (1e-4, 1e-5)),
    ("mlp-h50-cube", "bosh3"): ((1e-2, 1e-4), (1e-3, 1e-4)),
    ("mlp-h50-cube", "adaptive_heun"): ((1e-1, 1e-3), (1e-2, 1e-3)),
    ("mlp-h1-cube", "dopri5"): ((1e-6, 1e-8), (1e-6, 1e-7)),
    ("mlp-h1-lin", "dopri5"): ((1e-8, 1e-10), None),       # fp32: no tolerance gives a rejection within 200 attempts
    ("mlp-h50-lin", "dopri5"): ((1e-6, 1e-8), (1e-6, 1e-7)),
    ("mlp-h128-cube", "dopri5"): ((1e-3, 1e-5), (1e-2, 1e-3)),
    ("mlp-h128-lin", "dopri5"): ((1e-5, 1e-7), (1e-5, 1e-6)),
    ("lorenz", "dopri5"): es.TOLERANCES["lorenz", "dopri5"],
    ("lv", "dopri5"): es.TOLERANCES["lv", "dopri5"],
}


def solve_tol(case):
    key = case.system if case.system.startswith("mlp") else solve_kind(case)
    return SOLVE_TOL[key, case.method][0 if case.dtype == "float64" else 1]


SOLVE_HORIZON = {"kepler": 1.0, "mlp": 2.0, "lorenz": 0.25, "lv": 2.0}      # forward; reverse time goes half as far
SOLVE_FIRST_STEP = {"kepler": 0.5, "mlp": 2.0, "lorenz": 0.25, "lv": 1.0}
SOLVE_ROWS = {"kepler": 12, "mlp": 300, "lorenz": 300, "lv": 300}           # state rows (Kepler: of KEPLER_ORBITS orbits)
FIXED_METHODS = ("euler", "midpoint", "heun", "rk4")
FIXED_STEP = 0.013          # not a divisor of the output spacing: interpolated rows

# system: (kind, args).  CubicMLP args: (hidden, cube, built dtype follows the state's)
SYSTEMS = {"kepler": ("kepler", None), "kepler32": ("kepler", 32)}
SYSTEMS.update({"mlp-h%d-%s" % (h, "cube" if c else "lin"): ("mlp", (h, bool(c))) for h in (1, 50, 128) for c in (1, 0)})
SYSTEMS.update({"lorenz-%s" % k: ("lorenz", k) for k in ("a", "b")})
SYSTEMS.update({"lv-%s" % k: ("lv", k) for k in ("a", "b")})

SolveCase = collections.namedtuple("SolveCase", "name system method dtype reverse path")


def _sc(system, method, dtype, reverse, path):
    return SolveCase("%s-%s-%s-%s-%s" % (system, method, dtype[-2:], "rev" if reverse else "fwd", path), system, method,
                     dtype, reverse, path)


_DIRS = (False, True)
SOLVE_CASES = []
# Kepler: every tableau on the persistent kernel and in the stage kernels (tsit5 only there), both dtypes and directions
SOLVE_CASES += [_sc("kepler", me, dt, rev, "persistent") for me in es.METHODS for dt in DTYPES for rev in _DIRS]
SOLVE_CASES += [_sc("kepler", me, dt, rev, "stages") for me in es.METHODS + ("tsit5",) for dt in DTYPES for rev in _DIRS]
SOLVE_CASES += [_sc("kepler", "dopri5", "float32", True, "stages_graph"),
                _sc("kepler32", "dopri8", "float64", False, "stages_graph")]         # BASELINE config 5 in miniature
SOLVE_CASES += [_sc("kepler", me, dt, rev, "rows") for me in ("dopri5", "dopri8") for dt in DTYPES for rev in _DIRS]
SOLVE_CASES += [_sc("kepler", me, dt, rev, "fixed") for me in FIXED_METHODS for dt in DTYPES for rev in _DIRS]
# CubicMLP with biases: the full path list at H = 50 with the cube (BASELINE config 3's module: rk4, fp32, "fixed"), and
# one case per path family at the other widths and without the cube
_M = "mlp-h50-cube"
SOLVE_CASES += [_sc(_M, me, dt, rev, "persistent") for me in es.METHODS for dt in DTYPES for rev in _DIRS]
SOLVE_CASES += [_sc(_M, me, dt, rev, "stages") for me in es.METHODS + ("tsit5",) for dt in DTYPES for rev in _DIRS]
SOLVE_CASES += [_sc(_M, "dopri5", "float64", False, "stages_graph")]
SOLVE_CASES += [_sc(_M, me, dt, rev, "rows") for me in ("dopri5", "dopri8") for dt in DTYPES for rev in _DIRS]
SOLVE_CASES += [_sc(_M, me, dt, rev, "fixed") for me in FIXED_METHODS for dt in DTYPES for rev in _DIRS]
for _s in [s for s in SYSTEMS if s.startswith("mlp") and s != _M]:
    SOLVE_CASES += [_sc(_s, "dopri5", dt, False, p) for dt in DTYPES for p in ("persistent", "stages", "rows")]
    SOLVE_CASES += [_sc(_s, "rk4", dt, True, "fixed") for dt in DTYPES]
# Lorenz and Lotka-Volterra with non-default parameters, one case per kernel family, against the numpy oracle
for _s in [s for s in SYSTEMS if s.startswith(("lorenz", "lv"))]:
    SOLVE_CASES += [_sc(_s, "dopri5", dt, _s.endswith("b"), p) for dt in DTYPES for p in ("persistent", "stages", "rows")]
    SOLVE_CASES += [_sc(_s, "rk4", dt, _s.endswith("b"), "fixed") for dt in DTYPES]
SOLVE_CASES = [c for c in SOLVE_CASES if c.path == "fixed" or
               SOLVE_TOL[c.system if c.system.startswith("mlp") else SYSTEMS[c.system][0], c.method][c.dtype == "float32"]]
SOLVE = {c.name: c for c in SOLVE_CASES}
assert len(SOLVE) == len(SOLVE_CASES)


def solve_kind(case):
    return SYSTEMS[case.system][0]


def solve_module(case):
    """The rhs module of a case (CPU; CubicMLP in the state dtype, weights at std 0.2, non-zero biases)."""
    from tfdiffeq_b200 import rhs
    kind, args = SYSTEMS[case.system]
    if kind == "kepler":
        return rhs.Kepler()
    if kind == "mlp":
        return mlp_module(args[0], args[1], 0.2, case.dtype, seed=1)
    if kind == "lorenz":
        return rhs.Lorenz(*LORENZ_PARAMS[args])
    return rhs.LotkaVolterra(*LV_PARAMS[args])


def solve_setup(case):
    """(y0, t, rtol, atol, options) of a case.  Adaptive cases: the exact schedule's options with a power-of-two
    first_step and the output grid of exact_schedule._t_grid; fixed-grid cases: six outputs and step_size FIXED_STEP."""
    kind, args = SYSTEMS[case.system]
    rng = np.random.default_rng(31)
    n = SOLVE_ROWS[kind]
    if kind == "kepler":
        y0 = PROBLEMS["kepler"](orbits=args or es.KEPLER_ORBITS).y0(n, seed=7)
    elif kind == "mlp":
        y0 = np.array([2.0, 0.0]) + 0.1 * rng.standard_normal((n, 2))
    elif kind == "lorenz":
        y0 = np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((n, 3))
    else:
        y0 = 1.0 + 0.3 * rng.random((n, 2))
    y0 = y0.astype(case.dtype)
    horizon = SOLVE_HORIZON[kind] / (2.0 if case.reverse else 1.0)
    if case.path == "fixed":
        t = np.linspace(0.0, 0.1, 6)
        return y0, (-t if case.reverse else t), None, None, dict(step_size=FIXED_STEP)
    t = es._t_grid(horizon, (horizon / 2,), 5)
    rtol, atol = solve_tol(case)
    return y0, (-t if case.reverse else t), rtol, atol, dict(es.OPTIONS, first_step=SOLVE_FIRST_STEP[kind])


def numpy_rhs(case, module):
    """The system in numpy.  Exact for Lorenz and Lotka-Volterra (their oracle); for Kepler and CubicMLP a stand-in that
    differs from the device's evaluation in the last bits of pow and tanh -- the CPU test uses it to show that each case
    has rejections and decision margins, which the GPU test then re-checks on the device-evaluated oracle itself."""
    kind, args = SYSTEMS[case.system]
    if kind == "lorenz":
        return lambda t, y: lorenz_exact(y, LORENZ_PARAMS[args])
    if kind == "lv":
        return lambda t, y: lv_exact(y, LV_PARAMS[args])
    if kind == "kepler":
        return PROBLEMS["kepler"](orbits=args or es.KEPLER_ORBITS)
    W1, b1, W2, b2 = mlp_weights(module, case.dtype)
    cube = args[1]
    return lambda t, y: np.tanh((y ** 3 if cube else y) @ W1 + b1) @ W2 + b2


def row_dim(case):
    return {"kepler": 4, "mlp": 2, "lorenz": 3, "lv": 2}[solve_kind(case)]
