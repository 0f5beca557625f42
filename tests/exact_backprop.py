"""Exact comparisons of ``odeint(..., options={'backprop': True})`` (DESIGN.md section 4.2(f)): ``y0.grad`` and every
parameter gradient bit for bit against a restatement of the engine's reverse sweep on top of the oracle's forward solve.

The forward solve is ``oracle/np_ref.py`` under the exact step schedule of tests/exact_schedule.py (fixed grids: its
FixedGrid), recorded per accepted step: y_n, every stage input Y_i, its time tau_i and its k, (t0, t1, dt) and the
outputs [j0, j1) the step emitted.  The reverse sweep (``reverse_sweep``) repeats what backprop.py's ``_Backward.run``
and the kernels compute, operation by operation in the state dtype:
  * a combine (k_bp_combine, and k_bp_rhs's registers) is acc = c_0 x_0, acc += c_j x_j left to right, then base + acc,
    with c_j = fl(dt_n coef_j) (coef_j alone when it has no step); zero coefficients are dropped;
  * the dense-output VJP is bp_dense_quartic / bp_dense_k (b2ode_bp.cuh) with x formed from the output time rounded to
    the state dtype, or k_bp_dense's linear rule on the fixed grid;
  * the stage sweep, adaptive Heun's carry of f0's cotangent into the previous step's last k, the FSAL f0 evaluated at
    the previous step's last stage time, lambda_n as a combine with unscaled coefficients 1, y0.grad = lambda + g[0], and
    the parameter cotangents accumulated as pgrads[i] + g in the engine's call order.
Its vector-Jacobian products are torch-CPU autograd of the same module class (a flat leaf with per-component views, as
the engine calls func), taken at the *forward's* recorded stage inputs and times.  An engine whose recompute does not
reproduce those inputs therefore differs from the restatement, which is what the rk4 cases test.

The comparison is exact for right-hand sides whose VJPs are chains of correctly rounded elementwise operations (per-row
Lorenz, Tuple5, the built-in Lorenz and Lotka-Volterra) or ExactLinear's matrix (tests/exact_adjoint.py).

This module is a plain helper (no fixtures); both test files import it.
"""
import collections
import contextlib

import numpy as np
import torch

import exact_adjoint as ea
import exact_schedule as es
import exact_stream as xs
import np_ref

TDT = ea._TDT
ADAPTIVE = es.METHODS
FIXED = ("euler", "midpoint", "heun", "rk4")
RECORD_SLOTS = 16                # backprop.Record's initial capacity: it doubles while the solve runs


# --------------------------------------------------------------------------------------------------
# the engine's recipes
# --------------------------------------------------------------------------------------------------
Tab = collections.namedtuple("Tab", "beta c_sol c_mid n_k fsal fixed")


def tableau(method):
    from tfdiffeq_b200 import backprop, tableaus
    if method in FIXED:
        beta, c_sol = backprop._FIXED_TAB[method]
        return Tab(beta, c_sol, None, len(c_sol), False, True)
    tb = tableaus.TABLEAUS[method]
    return Tab(tb.beta, tb.c_sol, tb.c_mid, tb.n_k, tb.fsal, False)


def dense_mask(tab):
    """The k's the quartic dense output reaches: f0, f1 and those of y_mid (backprop.py's k_mask)."""
    if tab.fixed:
        return 0
    mask = 1 | (1 << (tab.n_k - 1))
    for j in range(tab.n_k):
        if tab.c_mid[j] != 0.0:
            mask |= 1 << j
    return mask


def combine(base, terms, dt, T):
    """k_bp_combine on tuples of arrays: base + (c_0 x_0 + c_1 x_1 + ...), c_j = fl(T(dt) T(coef_j)) (dt None: T(coef_j)),
    zero coefficients dropped; None when no term is left (the engine then uses base itself)."""
    terms = [(c, x) for c, x in terms if c != 0.0]
    if not terms:
        return None
    cs = [T(c) if dt is None else T(T(dt) * T(c)) for c, _ in terms]
    out = []
    for s in range(len(terms[0][1])):
        acc = cs[0] * terms[0][1][s]
        for c, (_, x) in zip(cs[1:], terms[1:]):
            acc = acc + c * x[s]
        out.append(acc if base is None else base[s] + acc)
    return tuple(out)


def rk4_stage(y, ks, dt, T):
    """fixed_eval's B2ODE_OP_RK4_S2..S4 (b2ode.cu), the fixed-grid rk4 forward's stage inputs after len(ks) k's."""
    d = T(dt)
    out = []
    for s in range(len(y)):
        a = ks[0][s]
        if len(ks) == 1:
            out.append(y[s] + (d * a) / T(3))
        elif len(ks) == 2:
            out.append(y[s] + d * (a / T(-3) + ks[1][s]))
        else:
            out.append(y[s] + d * ((a - ks[1][s]) + ks[2][s]))
    return tuple(out)


def recompute(tab, method, y, ks, i, dt, T, rk4_combine=False):
    """The backward pass's stage input i >= 1 from y_n and k_0 .. k_{i-1}: rk4's forward formula on the fixed grid
    (combine order instead with rk4_combine), the combine of beta_{i-1} otherwise."""
    if method == "rk4" and not rk4_combine:
        return rk4_stage(y, ks[:i], dt, T)
    acc = combine(y, [(tab.beta[i - 1][j], ks[j]) for j in range(i)], dt, T)
    return y if acc is None else acc


# --------------------------------------------------------------------------------------------------
# the oracle's forward solve, recorded per accepted step
# --------------------------------------------------------------------------------------------------
Step = collections.namedtuple("Step", "t0 t1 dt j0 j1 ends y Y tau k")
Forward = collections.namedtuple("Forward", "sol steps t n_acc n_rej solve")


@contextlib.contextmanager
def _capture(attempts):
    orig = np_ref.runge_kutta_step

    def step(func, y0, f0, t0, dt, tableau):
        calls = []

        def f(ti, yi):
            calls.append((ti, yi))
            return func(ti, yi)
        res = orig(f, y0, f0, t0, dt, tableau)
        attempts.append((y0, float(t0), float(dt), calls, res[3]))
        return res
    np_ref.runge_kutta_step = step
    try:
        yield
    finally:
        np_ref.runge_kutta_step = orig


class _RecFixed(np_ref.FixedGrid):
    def __init__(self, *a, **kw):
        np_ref.FixedGrid.__init__(self, *a, **kw)
        self.cells = []

    def _f(self, t, y):
        out = np_ref.FixedGrid._f(self, t, y)
        self._calls.append((t, y, out))
        return out

    def step_func(self, t, dt, y):
        self._calls = []
        dy = np_ref.FixedGrid.step_func(self, t, dt, y)
        self.cells.append((t, dt, y, self._calls))
        return dy


def forward(func, y0, t, method, rtol, atol, options):
    """The oracle's solve of the numpy func (tuple in, tuple out) from the tuple y0 over t, recorded (Forward)."""
    sd = y0[0].dtype.type
    nk = tableau(method).n_k
    if method in ADAPTIVE:
        attempts = []
        with _capture(attempts):
            s = es.oracle_solve(func, y0, t, method, rtol, atol, options)
        tt = s.t
        steps, prev = [], None
        for n, ((y, t0, dt, calls, k), ok) in enumerate(zip(attempts, s.stats.acc_trace)):
            if not ok:
                continue
            t1 = t0 + dt
            js = [j for j in range(1, len(tt)) if t0 < tt[j] <= t1]
            j0, j1 = (js[0], js[-1] + 1) if js else (0, 0)
            if prev is None:
                tau0 = sd(tt[0])
            elif tableau(method).fsal:
                tau0 = prev.tau[-1]
            else:
                tau0 = None                       # adaptive Heun: f0 is the previous step's last k, not an evaluation
            ks = [tuple(k_[i] for k_ in k) for i in range(nk)]
            prev = Step(t0, t1, dt, j0, j1, False, y, [y] + [c[1] for c in calls], [tau0] + [c[0] for c in calls], ks)
            steps.append(prev)
        return Forward(s.sol, steps, tt, s.stats.n_acc, s.stats.n_rej, s)
    t = np.asarray(t, dtype=np.float64)
    if bool(np.all(t[1:] < t[:-1])):                                    # np_ref.odeint's reverse-time wrap
        t = -t
        fwd = func
        func = lambda t_, y_: tuple(-v for v in fwd(-t_, y_))          # noqa: E731
    solver = _RecFixed(func, y0, np_ref.FIXED[method], **options)
    sol = solver.integrate(t)
    ts = t.astype(sd)
    grid = solver.grid_constructor(func, y0, ts)
    steps, j = [], 1
    for i, (t0, dt, y, calls) in enumerate(solver.cells):
        t1 = grid[i + 1]
        j0 = j
        while j < len(ts) and t1 >= ts[j]:
            j += 1
        ends = j > j0 and ts[j - 1] == t1
        steps.append(Step(float(t0), float(t1), float(dt), j0, j, ends, y, [c[1] for c in calls], [c[0] for c in calls],
                          [c[2] for c in calls]))
    return Forward(sol, steps, t, len(steps), 0, None)


# --------------------------------------------------------------------------------------------------
# the reverse sweep
# --------------------------------------------------------------------------------------------------
class _Vjp(object):
    """J^T mu of the engine-frame func (the reverse-time wrapper -f(-t, y) included) by torch-CPU autograd on a flat leaf
    with per-component views; accumulates parameter cotangents as the engine does."""

    def __init__(self, module, y0, tensor_input, reverse):
        self.params = tuple(p for p in module.parameters() if p.requires_grad)
        call = ea.tuple_call(module, tensor_input)
        self.f = (lambda t, y: tuple(-o for o in call(-t, y))) if reverse else call       # noqa: E731
        self.shapes = [y.shape for y in y0]
        self.lens = [y.size for y in y0]
        self.offs = list(np.cumsum([0] + self.lens[:-1]))
        self.tdt = TDT[y0[0].dtype.name]
        self.calls = 0

    def __call__(self, tau, Y, mu, pgrads):
        flat = torch.cat([torch.from_numpy(np.ascontiguousarray(c)).reshape(-1) for c in Y]).requires_grad_(True)
        views = tuple(flat[o:o + n].view(s) for o, n, s in zip(self.offs, self.lens, self.shapes))
        with torch.enable_grad():
            outs = self.f(ea._tt(tau, self.tdt), views)
        self.calls += 1
        live = [(o, torch.from_numpy(np.ascontiguousarray(m)).reshape(o.shape)) for o, m in zip(outs, mu)
                if isinstance(o, torch.Tensor) and o.requires_grad]
        if not live:
            return None
        gs = torch.autograd.grad([o for o, _ in live], (flat,) + self.params, [m for _, m in live], allow_unused=True)
        for i, g in enumerate(gs[1:]):
            if g is not None:
                pgrads[i] = g if pgrads[i] is None else pgrads[i] + g
        if gs[0] is None:
            return None
        g = gs[0].numpy()
        return tuple(g[o:o + n].reshape(s) for o, n, s in zip(self.offs, self.lens, self.shapes))


def _dense_quartic(w, st, t_out, dt, T, tab, mask, drop_f1):
    """bp_dense_quartic + bp_dense_k per component: (a0, a1, {k: mu_k})."""
    t0, den = T(st.t0), T(T(st.t1) - T(st.t0))
    last = tab.n_k - 1
    a0s, a1s, mus = [], [], {k: [] for k in range(tab.n_k) if (mask >> k) & 1}
    for s in range(len(w)):
        z = np.zeros_like(w[s][0])
        GA, GB, GC, GD, G1 = z, z, z, z, z
        for j in range(st.j0, st.j1):
            x = T(T(T(t_out[j]) - t0) / den)
            x2 = T(x * x)
            x3 = T(x2 * x)
            x4 = T(x3 * x)
            gj = w[s][j]
            GA, GB, GC, GD, G1 = GA + gj * x4, GB + gj * x3, GC + gj * x2, GD + gj * x, G1 + gj
        gmid = (T(16) * GA - T(32) * GB) + T(16) * GC
        a0 = (T(18) * GB - T(8) * GA) + T(-11) * GC
        a0s.append((a0 + G1) + gmid)
        a1s.append((T(14) * GB - T(8) * GA) - T(5) * GC)
        f0 = dt * ((T(5) * GB - T(2) * GA) + (GD - T(4) * GC))
        f1 = dt * ((T(2) * GA - T(3) * GB) + GC)
        for k in mus:
            v = T(dt * T(tab.c_mid[k])) * gmid
            if k == 0:
                v = v + f0
            if k == last and not drop_f1:
                v = v + f1
            mus[k].append(v)
    return tuple(a0s), tuple(a1s), {k: tuple(v) for k, v in mus.items()}


def _dense_linear(w, st, t_out, T):
    """k_bp_dense's linear rule: (a0, a1) per component."""
    t0, den = T(st.t0), T(T(st.t1) - T(st.t0))
    a0s, a1s = [], []
    for s in range(len(w)):
        a0 = np.zeros_like(w[s][0])
        a1 = np.zeros_like(w[s][0])
        for j in range(st.j0, st.j1):
            gj = w[s][j]
            if st.ends and j == st.j1 - 1:
                a1 = a1 + gj
                continue
            q = T(T(T(t_out[j]) - t0) / den)
            a1 = a1 + gj * q
            a0 = a0 + gj * T(T(1) - q)
        a0s.append(a0)
        a1s.append(a1)
    return tuple(a0s), tuple(a1s)


Grads = collections.namedtuple("Grads", "y0 params calls")
VARIANTS = (None, "rk4_combine", "tau_t0", "dt_f32", "no_f1")


def reverse_sweep(fwd, method, module, y0, w, tensor_input, reverse, variant=None):
    """The engine's backward pass over the recorded forward `fwd` for output cotangents w (per component (T, *shape), or
    None).  `variant` restates a wrong engine, for the negative controls: rk4's stage inputs in combine order
    ("rk4_combine"), every stage time t_n ("tau_t0"), dt rounded through float32 ("dt_f32"), the quartic's f1 term
    dropped ("no_f1").  Returns Grads(y0 tuple, parameter gradients as tensors, VJP calls)."""
    assert variant in VARIANTS
    T = y0[0].dtype.type
    tab = tableau(method)
    nk, beta, fsal = tab.n_k, tab.beta, tab.fsal
    mask = dense_mask(tab)
    w = tuple(np.zeros((len(fwd.t),) + y.shape, dtype=y.dtype) if g is None else g for g, y in zip(w, y0))
    vjp = _Vjp(module, y0, tensor_input, reverse)
    pgrads = [None] * len(vjp.params)
    lam = tuple(np.zeros_like(y) for y in y0)
    carry = None
    lam_coef = beta[nk - 2] if fsal else tab.c_sol
    for n in range(len(fwd.steps) - 1, -1, -1):
        st = fwd.steps[n]
        dt_raw = float(np.float32(st.dt)) if variant == "dt_f32" else st.dt
        dt = T(dt_raw)
        fresh0 = tab.fixed or fsal or n == 0
        Y, tau = list(st.Y), list(st.tau)
        if variant == "rk4_combine" and method == "rk4":
            Y = [st.y] + [recompute(tab, method, st.y, st.k, i, dt_raw, T, rk4_combine=True) for i in range(1, nk)]
        if variant == "tau_t0":
            tau = [T(st.t0)] * nk
        # dense output
        if tab.fixed:
            g0, a1 = _dense_linear(w, st, fwd.t, T)
            mu_dense = {}
        else:
            g0, a1, mu_dense = _dense_quartic(w, st, fwd.t, dt, T, tab, mask, variant == "no_f1")
        lam = tuple(l_ + a_ for l_, a_ in zip(lam, a1))
        if carry is not None:
            mu_dense[nk - 1] = combine(mu_dense[nk - 1], [(1.0, carry)], None, T)
        # reverse stage sweep
        nus = [None] * (nk - 1)
        for i in range(nk - 2, -1, -1):
            j = i + 1
            terms = [(beta[l][j], nus[l]) for l in range(j, nk - 1) if nus[l] is not None]
            if j < len(lam_coef):
                terms.append((lam_coef[j], lam))
            mu = combine(mu_dense.get(j), terms, dt_raw, T)
            mu = mu_dense.get(j) if mu is None else mu
            nus[i] = None if mu is None else vjp(tau[j], Y[j], mu, pgrads)
        terms = [(beta[l][0], nus[l]) for l in range(nk - 1) if nus[l] is not None] + [(lam_coef[0], lam)]
        xi0 = None
        mu0 = combine(mu_dense.get(0), terms, dt_raw, T)
        mu0 = mu_dense.get(0) if mu0 is None else mu0
        if fresh0:
            xi0 = None if mu0 is None else vjp(tau[0], Y[0], mu0, pgrads)
            carry = None
        else:
            carry = mu0
        lam = combine(g0, [(1.0, v) for v in nus + [xi0] if v is not None] + [(1.0, lam)], None, T)
    gy0 = tuple(l_ + g[0] for l_, g in zip(lam, w))
    params = [torch.zeros_like(p) if g is None else g for g, p in zip(pgrads, vjp.params)]
    return Grads(gy0, params, vjp.calls)


# --------------------------------------------------------------------------------------------------
# cases
# --------------------------------------------------------------------------------------------------
Case = collections.namedtuple("Case", "name kind dtype rows method rtol atol t first_step step_size reverse seed")

T_LORENZ = es._t_grid(0.25, (0.125,), 5)       # outputs inside steps, on a step end, and steps with none
T_LV = es._t_grid(2.0, (1.0,), 5)
T_LINEAR = np.array([0.0, 0.2, 0.45, 1.5])
# the fixed grid: step 0.0125 is not dyadic, so dt has a full mantissa; 0.025, 0.05 and 0.1 are grid points
T_FIXED = np.array([0.0, 0.006, 0.025, 0.031, 0.05, 0.07, 0.1])
FIXED_STEP = 0.0125
ROWS = 4099
BUILTIN_ROWS = 300007          # k_bp_rhs: two passes of 1056 x 256 rows at 132 SMs, the last one partial
LINEAR_ROWS, LINEAR_DIM = 4300, 128


def _short(dtype):
    return "f64" if dtype == "float64" else "f32"


def _lorenz(method, dtype, reverse, rows=ROWS, kind="lorenz_forced", rtol=None, atol=None, t=None):
    if method in FIXED:
        t = T_FIXED if t is None else t
        fs, ss, tol = None, FIXED_STEP, (None, None)
    else:
        t = T_LORENZ if t is None else t
        fs, ss = ea.FIRST_STEP.get(method, es.FIRST_STEP["lorenz"]), None
        tol = es.TOLERANCES["lorenz", method][0 if dtype == "float64" else 1]
    tol = (rtol or tol[0], atol or tol[1])
    name = "%s-%s-%s-%s-%d" % (kind, method, _short(dtype), "rev" if reverse else "fwd", rows)
    return Case(name, kind, dtype, rows, method, tol[0], tol[1], -t if reverse else t, fs, ss, reverse, 3)


def _lv(method, dtype, rows=BUILTIN_ROWS):
    if method in FIXED:
        t, fs, ss, tol = T_FIXED * 10.0, None, FIXED_STEP * 10.0, (None, None)
    else:
        t, fs, ss = T_LV, es.FIRST_STEP["lv"], None
        tol = es.TOLERANCES["lv", method][0 if dtype == "float64" else 1]
    return Case("builtin_lv-%s-%s-fwd-%d" % (method, _short(dtype), rows), "builtin_lv", dtype, rows, method, tol[0],
                tol[1], t, fs, ss, False, 3)


GENERIC = [_lorenz(me, dt, rev) for me in ADAPTIVE for dt in es.DTYPES for rev in (False, True)]
LARGE = [_lorenz(me, dt, False, rows=xs.LORENZ_ROWS[dt]) for me, dt in (("dopri5", "float64"), ("dopri5", "float32"),
                                                                        ("dopri8", "float64"), ("adaptive_heun", "float32"))]
FIXED_CASES = [_lorenz(me, dt, rev) for me in FIXED for dt in es.DTYPES for rev in (False, True)]
TUPLE = [Case("tuple5-%s-%s" % (me, _short(dt)), "tuple5", dt, ROWS, me,
              *(es.TOLERANCES["lorenz", me][0 if dt == "float64" else 1] if me in ADAPTIVE else (None, None)),
              T_LORENZ if me in ADAPTIVE else T_FIXED, 0.25 if me in ADAPTIVE else None,
              None if me in ADAPTIVE else FIXED_STEP, False, 5) for me in ("dopri5", "rk4") for dt in es.DTYPES]
LINEAR = [Case("linear_external-dopri5-f64-%d" % LINEAR_ROWS, "linear_external", "float64", LINEAR_ROWS, "dopri5", 1e-8,
               1e-10, T_LINEAR, 0.5, None, False, 102),
          Case("linear_builtin-dopri5-f64-%d" % LINEAR_ROWS, "linear_builtin", "float64", LINEAR_ROWS, "dopri5", 1e-8,
               1e-10, T_LINEAR, 0.5, None, False, 102)]
# every adaptive tableau on Lorenz in fp64; fp32, Lotka-Volterra and rk4 on a subset (each oracle takes seconds here)
BUILTIN = [_lorenz(me, "float64", False, rows=BUILTIN_ROWS, kind="builtin_lorenz") for me in ADAPTIVE]
BUILTIN += [_lorenz(me, "float32", False, rows=BUILTIN_ROWS, kind="builtin_lorenz") for me in ("dopri5", "rk4")]
BUILTIN += [_lorenz("rk4", "float64", False, rows=BUILTIN_ROWS, kind="builtin_lorenz")]
BUILTIN += [_lv(me, dt) for me, dt in (("dopri5", "float64"), ("dopri5", "float32"), ("adaptive_heun", "float64"),
                                       ("rk4", "float64"))]
# 64 accepted steps after 6 rejections: the record grows 16 -> 32 -> 64 slots while the solve runs (the exact schedule
# never lengthens dt, so its rejections come before the first accepted step)
GROWTH = [_lorenz("dopri5", "float64", False, rtol=1e-9, atol=1e-11)._replace(
    name="lorenz_forced-dopri5-f64-fwd-4099-growth")]
ALL = {c.name: c for c in GENERIC + LARGE + FIXED_CASES + TUPLE + LINEAR + BUILTIN + GROWTH}
# the small versions the CPU test checks against autograd through np_ref
SMALL_ROWS = 5


def make_module(case):
    import tfdiffeq_b200
    k = case.kind
    if k == "lorenz_forced":
        return ea.LorenzPerRow(case.rows, case.dtype, forcing=True, seed=case.seed)
    if k == "builtin_lorenz":
        return tfdiffeq_b200.rhs.Lorenz()
    if k == "builtin_lv":
        return tfdiffeq_b200.rhs.LotkaVolterra()
    if k == "linear_external":
        return ea.ExactLinearFunc(LINEAR_DIM, case.seed)
    if k == "linear_builtin":
        return ea.linear_module(LINEAR_DIM, case.seed, False)
    if k == "tuple5":
        return ea.Tuple5(case.rows, ea.TUPLE_M, case.dtype, seed=case.seed)
    raise KeyError(k)


def initial_state(case):
    if case.kind == "builtin_lv":
        rng = np.random.default_rng(case.seed)
        return ((1.0 + 0.3 * rng.random((case.rows, 2))).astype(case.dtype),)
    if case.kind.startswith("linear"):
        rng = np.random.default_rng(case.seed)
        return (rng.standard_normal((case.rows, LINEAR_DIM)).astype(case.dtype),)
    return ea.initial_state(case)


def options(case):
    if case.method in ADAPTIVE:
        return dict(es.OPTIONS, first_step=case.first_step, max_num_steps=ea.MAX_NUM_STEPS)
    return dict(step_size=case.step_size)


def tensor_input(case):
    return case.kind != "tuple5"


def solve_case(case, variant=None):
    """(module, y0, w, Forward, Grads) of a case."""
    module = make_module(case)
    y0 = initial_state(case)
    w = ea.loss_weights(case, y0)
    f = ea.numpy_func(module, case.dtype, tensor_input(case))
    fwd = forward(f, y0, case.t, case.method, case.rtol, case.atol, options(case))
    g = reverse_sweep(fwd, case.method, module, y0, w, tensor_input(case), case.reverse, variant)
    return module, y0, w, fwd, g


def small(case, rows=SMALL_ROWS):
    """The case at a few rows (Tuple5: n = rows, m = 3), for autograd through np_ref on the CPU."""
    return case._replace(rows=rows, name=case.name + "-small")


