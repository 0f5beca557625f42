"""Exact comparisons of ``odeint_adjoint`` (DESIGN.md section 2): the forward solve, ``y0.grad`` and the parameter
gradients bit for bit against an oracle that restates the reference adjoint (tfdiffeq/adjoint.py:35-180) on top of
``oracle/np_ref.py``.

The oracle's vector-Jacobian products come from torch-CPU autograd of the same module class, as the reference's
``GradientTape`` does over the shim (oracle/make_golden_grads.py:51-70).  The comparison is exact when
  1. every VJP is a chain of correctly rounded elementwise operations: right-hand sides built from +, -, * whose
     parameters are shaped like the state, so autograd reduces nothing, or ExactLinear's matrix, whose transpose also
     has two power-of-two entries per column, so ``(-a) @ A^T`` is one rounded two-term sum in any order;
  2. the step schedule is exact (tests/exact_schedule.py).  ``options`` carries it and ``adjoint_options`` inherits it,
     so every backward interval keeps or halves dt as the forward solve does;
  3. the time gradient changes nothing else.  ``dL/dt_i`` and, with a time forcing, ``a^T df/dt`` are reductions whose
     bits differ between devices, but they reach only ``adj_t``, which no derivative reads; its error ratio enters the
     max over components, which the margin premise covers.  ``t.grad`` is compared within a bound.

This module is a plain helper (no fixtures); both test files import it.
"""
import collections
import math

import numpy as np
import torch
import torch.nn as nn

import exact_schedule as es
import np_ref
from problems import PROBLEMS

_TDT = {"float64": torch.float64, "float32": torch.float32}
MAX_NUM_STEPS = 4 * es.MAX_ATTEMPTS
ADAPTIVE = ("dopri5", "bosh3", "adaptive_heun", "dopri8", "tsit5")


# --------------------------------------------------------------------------------------------------
# modules
# --------------------------------------------------------------------------------------------------
def _pow2(rng, shape, lo, hi):
    """+-2**k with k uniform in [lo, hi]."""
    return np.where(rng.random(shape) < 0.5, -1.0, 1.0) * 2.0 ** rng.integers(lo, hi + 1, shape)


class LorenzPerRow(nn.Module):
    """Lorenz with its own sigma, rho, beta per row, each a ``(B,)`` parameter, so that every VJP (w.r.t. y and the
    parameters) is elementwise; ``forcing`` adds ``t * u`` to x' with a ``(B,)`` parameter u, which makes every stage
    time of the forward and of each reverse-time backward solve reach the state, element by element."""

    def __init__(self, rows, dtype, forcing=False, seed=0):
        super(LorenzPerRow, self).__init__()
        rng = np.random.default_rng(seed)
        p = lambda v: nn.Parameter(torch.tensor(v, dtype=_TDT[dtype]))       # noqa: E731
        self.sigma = p(10.0 + rng.uniform(-1.0, 1.0, rows))
        self.rho = p(28.0 + rng.uniform(-2.0, 2.0, rows))
        self.beta = p(8.0 / 3.0 + rng.uniform(-0.25, 0.25, rows))
        self.u = p(rng.uniform(-4.0, 4.0, rows)) if forcing else None

    def forward(self, t, y):
        x, yy, z = y[..., 0], y[..., 1], y[..., 2]
        fx = self.sigma * (yy - x)
        if self.u is not None:
            fx = fx + t.to(y.dtype) * self.u
        return torch.stack([fx, x * (self.rho - z) - yy, x * yy - self.beta * z], -1)


class ExactLinearFunc(nn.Module):
    """problems.ExactLinear as an external ``y @ A`` module: A is a buffer, the module has no parameters."""

    def __init__(self, dim, seed, dtype="float64"):
        super(ExactLinearFunc, self).__init__()
        self.register_buffer("A", torch.tensor(PROBLEMS["exact_linear"](dim=dim, seed=seed).A_np, dtype=_TDT[dtype]))

    def forward(self, t, y):
        return y @ self.A


def linear_module(dim, seed, trainable):
    """rhs.LinearODE on ExactLinear's matrix, A frozen or trainable."""
    import tfdiffeq_b200
    f = tfdiffeq_b200.rhs.LinearODE(PROBLEMS["exact_linear"](dim=dim, seed=seed).A_np)
    f.A.requires_grad_(trainable)
    return f


class Tuple5(nn.Module):
    """A five-tensor state, (n, 3), (n, 3), (m, 2), (m, 2) and (1,): 2 * 5 + 2 = 12 augmented components.  Only
    components of equal shape are coupled; p, q and k are parameters shaped like the state they multiply."""

    def __init__(self, n, m, dtype, seed=0):
        super(Tuple5, self).__init__()
        rng = np.random.default_rng(seed)
        tdt = _TDT[dtype]
        self.p = nn.Parameter(torch.tensor(rng.uniform(-1.0, 1.0, (n, 3)), dtype=tdt))
        self.q = nn.Parameter(torch.tensor(1.5 + rng.uniform(-0.5, 0.5, (m, 2)), dtype=tdt))
        self.k = nn.Parameter(torch.tensor([-0.75], dtype=tdt))

    def forward(self, t, y):
        a, b, c, d, e = y
        x, yy, z = a[..., 0], a[..., 1], a[..., 2]
        fa = torch.stack([10.0 * (yy - x), x * (28.0 - z) - yy, x * yy - 2.5 * z], -1) + 0.5 * b
        fb = self.p * a - 0.25 * b
        fc = c * (self.q - d)
        fd = d * (c - 1.0)
        fe = self.k * e
        return fa, fb, fc, fd, fe


# --------------------------------------------------------------------------------------------------
# the oracle
# --------------------------------------------------------------------------------------------------
def _np(x):
    return x.detach().numpy()


def _tt(t, tdt):
    return torch.tensor(float(t), dtype=tdt)


def tuple_call(module, tensor_input):
    """func on a tuple state: a module of a tensor state is called on the 1-tuple's element (adjoint.py:205-212)."""
    if tensor_input:
        return lambda t, y: (module(t, y[0]),)           # noqa: E731
    return module


def numpy_func(module, dtype, tensor_input):
    """module(t, y) on numpy arrays (tuple in, tuple out): t as a 0-d tensor of the state dtype, as the engine passes
    every stage time."""
    tdt = _TDT[dtype]
    call = tuple_call(module, tensor_input)

    def f(t, y):
        with torch.no_grad():
            out = call(_tt(t, tdt), tuple(torch.from_numpy(np.ascontiguousarray(v)) for v in y))
        return tuple(_np(o) for o in out)
    return f


def solve(func, y0, t, method, rtol, atol, options):
    """np_ref's solver for `method` on a tuple state: es.oracle_solve (attempt record included) for the adaptive
    tableaus, np_ref.odeint for fixed grids and fixed_adams (no record)."""
    if method in ADAPTIVE:
        return es.oracle_solve(func, y0, t, method, rtol, atol, options)
    st = np_ref.Stats()
    t = np.asarray(t, dtype=np.float64)
    sol = np_ref.odeint(func, y0, t, rtol=rtol, atol=atol, method=method, options=dict(options), stats=st)
    return es.Solve(sol, st, None, None, t)


Adjoint = collections.namedtuple("Adjoint", "sol g_y0 g_params g_t g_t_scale forward backward")


def adjoint_oracle(module, y0, t, w, method, rtol, atol, options, adjoint_method=None, tensor_input=True,
                   time_dtype=None):
    """The reference adjoint (tfdiffeq/adjoint.py) for the loss sum_i sum_j <w_i[j], y_i(t_j)> on torch-CPU ``module``.

    y0: tuple of arrays; w: per component an array of shape (T, *y0_i.shape), or None for a component the loss does
    not touch (its output gradient is zero).  Returns the solution, the gradients w.r.t. y0, every trainable parameter
    (in ``module.parameters()`` order) and t, an error scale for each entry of the time gradient, and the Solve record
    of the forward solve and of every backward interval, last interval first.  ``tensor_input``: y0 is the 1-tuple
    of a tensor state and ``module`` takes that tensor.

    The reference stacks func's outputs (adjoint.py:81-83), so its tuple states need equal shapes; here every
    component is a separate array and the VJP is taken per component, which is what the engine does.
    ``time_dtype`` is the dtype of the running time adjoint: None keeps it in the state dtype, as the engine does;
    the reference keeps it in t's dtype (adjoint.py:116)."""
    n = len(y0)
    dtype = y0[0].dtype.name
    sd, tdt = y0[0].dtype.type, _TDT[dtype]
    adjoint_method = method if adjoint_method is None else adjoint_method
    f_params = [p for p in module.parameters() if p.requires_grad]
    t = np.asarray(t, dtype=np.float64)
    fwd = solve(numpy_func(module, dtype, tensor_input), y0, t, method, rtol, atol, options)                 # adjoint.py:54
    ans = fwd.sol
    T = len(t)
    grad_output = tuple(np.zeros_like(a) if g is None else np.asarray(g, dtype=dtype) for g, a in zip(w, ans))
    tdtype = y0[0].dtype if time_dtype is None else np.dtype(time_dtype)
    call = tuple_call(module, tensor_input)

    def augmented_dynamics(tt, y_aug):
        # adjoint.py:71-107: (f, -a^T df/dy, -a^T df/dt, -a^T df/dtheta) by autograd of the same module on the CPU
        y, adj_y = y_aug[:n], y_aug[n:2 * n]
        with torch.enable_grad():
            tt_ = _tt(tt, tdt).requires_grad_(True)
            y_ = tuple(torch.from_numpy(np.array(v)).requires_grad_(True) for v in y)
            f = call(tt_, y_)
            live = [(f_, -torch.from_numpy(np.asarray(a_))) for f_, a_ in zip(f, adj_y) if f_.requires_grad]
            wrt = (tt_,) + y_ + tuple(f_params)
            vjps = torch.autograd.grad([x for x, _ in live], wrt, [g for _, g in live], allow_unused=True) \
                if live else (None,) * len(wrt)
        vjp_t = np.zeros((), dtype=tdtype) if vjps[0] is None else _np(vjps[0]).astype(tdtype)
        vjp_y = tuple(np.zeros_like(v) if g is None else _np(g) for g, v in zip(vjps[1:1 + n], y))
        if f_params:                                                                          # adjoint.py:99-105
            vjp_p = np.concatenate([(np.zeros(p.numel(), dtype=dtype) if g is None else _np(g).reshape(-1))
                                    for g, p in zip(vjps[1 + n:], f_params)])
        else:
            vjp_p = np.zeros((), dtype=dtype)
        return (*(_np(x) for x in f), *vjp_y, vjp_t, vjp_p)

    adj_y = tuple(g[-1] for g in grad_output)                                                # adjoint.py:110-113
    adj_params = np.zeros(sum(p.numel() for p in f_params), dtype=dtype) if f_params else np.zeros((), dtype=dtype)
    adj_time = np.zeros((), dtype=tdtype)                                                    # adjoint.py:116
    time_vjps, scales, backward = [], [], []
    func = numpy_func(module, dtype, tensor_input)
    for i in range(T - 1, 0, -1):                                                            # adjoint.py:118
        ans_i = tuple(a[i] for a in ans)
        func_i = func(sd(t[i]), ans_i)                                                       # adjoint.py:127
        # adjoint.py:133-136, summed exactly and rounded once: the engine's reduction order is its own
        terms = [np.asarray(f_, dtype=np.float64).ravel() * np.asarray(g[i], dtype=np.float64).ravel()
                 for f_, g in zip(func_i, grad_output)]
        dLd_cur_t = tdtype.type(math.fsum(math.fsum(x) for x in terms))
        scales.append(math.fsum(math.fsum(np.abs(x)) for x in terms))
        adj_time = tdtype.type(adj_time - dLd_cur_t)                                        # adjoint.py:138
        time_vjps.append(dLd_cur_t)
        aug_y0 = (*ans_i, *adj_y, np.asarray(adj_time), adj_params)                          # adjoint.py:146
        s = solve(augmented_dynamics, aug_y0, np.array([t[i], t[i - 1]]), adjoint_method, rtol, atol,
                  options)                                                                   # adjoint.py:148-153
        backward.append(s)
        aug = s.sol
        adj_y = tuple(a[1] for a in aug[n:2 * n])                                            # adjoint.py:156-162
        adj_time = np.asarray(aug[2 * n][1])
        adj_params = np.asarray(aug[2 * n + 1][1])
        adj_y = tuple(a + g[i - 1] for a, g in zip(adj_y, grad_output))                      # adjoint.py:164
    time_vjps.append(adj_time)                                                               # adjoint.py:168-169
    g_t = np.array(time_vjps[::-1], dtype=np.float64)
    g_t_scale = np.array([sum(scales)] + scales[::-1])
    g_params, off = [], 0                                                                    # adjoint.py:171-177
    for p in f_params:
        g_params.append(adj_params.reshape(-1)[off:off + p.numel()].reshape(tuple(p.shape)))
        off += p.numel()
    return Adjoint(ans, adj_y, g_params, g_t, g_t_scale, fwd, backward)


# --------------------------------------------------------------------------------------------------
# the case table
# --------------------------------------------------------------------------------------------------
Case = collections.namedtuple("Case", "name kind dtype rows method adjoint_method rtol atol t first_step step_size "
                                      "reverse path seed")

T_GRID = np.array([0.0, 0.0731, 0.1313, 0.1875, 0.25])       # output times over Lorenz's exact-schedule horizon
T_SHORT = np.array([0.0, 0.1313, 0.25])
LORENZ_BATCH = 257                                             # rows of the small per-row Lorenz cases
# dopri8 and tsit5 start lower: from dt = 1/4 their first backward attempts overflow (fp32) or, with tsit5's error
# estimate, shrink dt past max_num_steps
FIRST_STEP = {"dopri8": 1.0 / 16, "tsit5": 1.0 / 16}


def _tol(method, dtype):
    if method in ("dopri5", "bosh3", "adaptive_heun", "dopri8", "tsit5"):
        return es.TOLERANCES["lorenz", method][0 if dtype == "float64" else 1]
    return (1e-6, 1e-8) if dtype == "float64" else (1e-4, 1e-5)


def _lorenz(method, dtype, reverse, forcing, rows=LORENZ_BATCH, adjoint_method=None, t=T_GRID, step_size=None,
            path=None):
    kind = "lorenz_forced" if forcing else "lorenz"
    name = "%s-%s-%s-%s-%d" % (kind, method, "f64" if dtype == "float64" else "f32", "rev" if reverse else "fwd", rows)
    if adjoint_method is not None:
        name += "-adj_" + adjoint_method
    rtol, atol = _tol(method, dtype)
    fs = FIRST_STEP.get(method, es.FIRST_STEP["lorenz"]) if method in ADAPTIVE else None
    return Case(name, kind, dtype, rows, method, adjoint_method, rtol, atol, -t if reverse else t, fs, step_size,
                reverse, path, 3)


SMALL = [_lorenz(me, dt, rev, fo) for me in ("dopri5", "bosh3", "adaptive_heun", "dopri8")
         for dt in es.DTYPES for rev in (False, True) for fo in (False, True)]
# tsit5 forward in time only: in reverse time its backward solves need more than max_num_steps attempts
SMALL += [_lorenz("tsit5", dt, False, fo) for dt in es.DTYPES for fo in (False, True)]
FIXED = [_lorenz(me, "float64", rev, True, step_size=1.0 / 32, t=T_SHORT) for me in ("euler", "midpoint", "rk4")
         for rev in (False, True)]
FIXED += [_lorenz("rk4", "float32", False, True, step_size=1.0 / 32, t=T_SHORT),
          _lorenz("fixed_adams", "float64", False, True, t=np.arange(9) * (1.0 / 32)),
          _lorenz("fixed_adams", "float64", True, False, t=np.arange(9) * (1.0 / 32))]
MIXED = [_lorenz("bosh3", "float64", False, True, adjoint_method="dopri5"),
         _lorenz("dopri8", "float32", True, False, adjoint_method="dopri5")]
# the generic path's grid loops: 600 001 x 3 fp64 and 750 001 x 3 fp32 (tests/exact_stream.py)
LARGE = [_lorenz("dopri5", "float64", False, True, rows=600001, t=T_SHORT),
         _lorenz("dopri5", "float32", True, True, rows=750001, t=T_SHORT)]
# the built-in right-hand side inside the persistent kernel's capacity (ncw3_partial at 132 SMs), and tsit5's stage
# kernels with the right-hand side fused in
BUILTIN = [Case("builtin_lorenz-dopri5-f64-fwd-12627", "builtin_lorenz", "float64", 12627, "dopri5", None, 1e-6, 1e-8,
                T_GRID, 0.25, None, False, "fused_rhs", 3),
           Case("builtin_lorenz-tsit5-f64-fwd-12627", "builtin_lorenz", "float64", 12627, "tsit5", None, 1e-1, 1e-2,
                T_GRID, 1.0 / 16, None, False, "stage_rhs", 3)]
# ExactLinear: the north star (65 536 x 128, A frozen) over a short horizon, a smaller trainable-A LinearODE and the
# external y @ A module
LINEAR = [Case("northstar-frozen", "linear_frozen", "float64", 65536, "dopri5", None, 1e-6, 1e-9,
               np.array([0.0, 0.3, 0.5]), 1.0, None, False, "stage_func", 100),
          Case("linear32-trainable-rev", "linear_trainable", "float64", 4099, "dopri5", None, 1e-8, 1e-10,
               -np.array([0.0, 0.2, 0.45, 0.75]), 0.5, None, True, "stage_func", 101),
          Case("linear32-external", "linear_external", "float64", 4099, "dopri5", None, 1e-8, 1e-10,
               np.array([0.0, 0.2, 0.45, 0.75]), 0.5, None, False, None, 102)]
TUPLE = [Case("tuple5-dopri5-%s" % ("f64" if dt == "float64" else "f32"), "tuple5", dt, 4099, "dopri5", None,
              *_tol("dopri5", dt), T_GRID, 0.25, None, False, None, 5) for dt in es.DTYPES]
TUPLE_M = 1001                  # rows of the (m, 2) components of Tuple5
ALL = {c.name: c for c in SMALL + FIXED + MIXED + LARGE + BUILTIN + LINEAR + TUPLE}
LINEAR_DIM = {"northstar-frozen": 128}


def linear_dim(case):
    return LINEAR_DIM.get(case.name, 32)


def make_module(case):
    """The case's module on the CPU (the GPU test moves a copy to the device)."""
    k = case.kind
    if k in ("lorenz", "lorenz_forced"):
        return LorenzPerRow(case.rows, case.dtype, forcing=k == "lorenz_forced", seed=case.seed)
    if k == "builtin_lorenz":
        import tfdiffeq_b200
        return tfdiffeq_b200.rhs.Lorenz()
    if k == "linear_external":
        return ExactLinearFunc(linear_dim(case), case.seed)
    if k in ("linear_frozen", "linear_trainable"):
        return linear_module(linear_dim(case), case.seed, k == "linear_trainable")
    if k == "tuple5":
        return Tuple5(case.rows, TUPLE_M, case.dtype, seed=case.seed)
    raise KeyError(k)


def initial_state(case):
    """y0 as a tuple of arrays."""
    rng = np.random.default_rng(case.seed)
    if case.kind.startswith("linear"):
        return (rng.standard_normal((case.rows, linear_dim(case))),)
    lor = lambda r: (np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((r, 3))).astype(case.dtype)   # noqa: E731
    if case.kind == "tuple5":
        return (lor(case.rows), (0.1 * rng.standard_normal((case.rows, 3))).astype(case.dtype),
                (1.0 + 0.3 * rng.random((TUPLE_M, 2))).astype(case.dtype),
                (1.0 + 0.3 * rng.random((TUPLE_M, 2))).astype(case.dtype), np.array([0.8125], dtype=case.dtype))
    return (lor(case.rows),)


UNTOUCHED = {"tuple5": 3}        # the output component the loss never reads: its output gradient is None


def loss_weights(case, y0):
    """w per component, shape (T, *y0_i.shape), every entry +-2**k or 0: the second output time carries no weight at
    all and about one entry in eight is zero.  None for the component the loss leaves out."""
    rng = np.random.default_rng(case.seed + 1000)
    T = len(case.t)
    out = []
    for i, y in enumerate(y0):
        if UNTOUCHED.get(case.kind) == i:
            out.append(None)
            continue
        w = _pow2(rng, (T,) + y.shape, -3, 1) * (rng.random((T,) + y.shape) >= 0.125)
        w[1] = 0.0
        out.append(w.astype(y.dtype))
    return tuple(out)


def options(case):
    if case.method in ADAPTIVE:
        return dict(es.OPTIONS, first_step=case.first_step, max_num_steps=MAX_NUM_STEPS)
    return {} if case.step_size is None else dict(step_size=case.step_size)


def solve_case(case):
    """(module, y0, w, Adjoint) of a case."""
    module = make_module(case)
    y0 = initial_state(case)
    w = loss_weights(case, y0)
    res = adjoint_oracle(module, y0, case.t, w, case.method, case.rtol, case.atol, options(case),
                         adjoint_method=case.adjoint_method, tensor_input=case.kind != "tuple5")
    return module, y0, w, res


def schedule_premises(res, case):
    """es.premises of the forward solve and of every backward interval (adaptive methods only)."""
    if case.method not in ADAPTIVE:
        return []
    out = [es.premises(res.forward, case.first_step)]
    if (case.adjoint_method or case.method) in ADAPTIVE:
        out += [es.premises(s, case.first_step) for s in res.backward]
    return out


def augmented_lens(case, module, y0):
    """Element counts of the backward solve's 2n + 2 components (y, adj_y, adj_t, adj_params)."""
    n_params = sum(p.numel() for p in module.parameters() if p.requires_grad)
    lens = [y.size for y in y0]
    return lens + lens + [1, max(1, n_params)]
