"""Step-size controller probes: solves whose controller decisions can be predicted, a 60-digit restatement of the
reference's controller, and a derived bound on every engine controller's error (DESIGN.md section 2).

The exact-schedule options (tests/exact_schedule.py) clamp every step factor to 1 or 1/2, so no log, exp or pow reaches
dt there.  Here the default options and ``safety=0.8, ifactor=5, dfactor=0.3`` (no value exact in float32) do.

**Probes.**  A probe is one Lorenz trajectory (3 elements) started at ``y0``, solved over ``t = [0, h / 256]`` with
``first_step = h`` (a power of two), ``rtol = 0`` and one ``atol`` per probe set.  Its first attempt runs from a dyadic
h on a +, -, * system, so the engine computes the oracle's error estimate bit for bit (the exact-schedule premise), and
the error ratio m of that attempt is known exactly.  The probes of a set differ only in ``y0``, which places m in the
controller's regimes; they share h and atol, so a whole set is one ``independent_rows`` launch.  A *one-attempt* probe
is accepted at once (the output time lies inside the step).  A *rejecting* probe is rejected, and retried at the step
its rejection produced (at least dfactor h, far beyond h / 256) until an attempt is accepted: twice for dopri5 and
dopri8; bosh3, adaptive_heun and tsit5 need more attempts from a deep rejection, because their error estimates fall
more slowly with dt than their controller exponents assume.  Every decision after the first is checked to be robust,
and the last one is restated at the engine's reported ratio; ``chain_bound`` adds up the errors of the ones between.

**The engine's ratio** of an attempt (b2ode_dev.cuh ``ctrl_decide``, b2ode_fused.cu ``ctrl_fast``), per component,
m = sum(err^2) / (tol^2 n) with tol = atol + rtol max(|y0|, |y1|) in the state dtype, rounded to the state dtype; the max
over components (tsit5: the pooled sum(err^2 / tol^2) / sum(n)).  ``restate`` applies misc.py:267-287 (tsit5.py:53-62)
to it at 60 digits: sqrt correctly rounded in the state dtype (not for tsit5), the exponent rounded through float32 (not
for tsit5), safety / ifactor / dfactor rounded through float32 (``_tf_f64``), the m == 0 branch, and the clamps with
1/ifactor and 1/dfactor formed in float64.

**Bounds** (``dt_bound``) on |dt_next / restated - 1|, u = 2^-53, e the exponent, X = e log2(er) the exponent of the
step factor (er = sqrt(m), tsit5: m), bar the relative error of the family's ratio:

* ``ctrl_decide`` (stage kernels, generic path, rows kernel), grow / shrink branches:
  ratio    e ((bar + u) / 2 + 2u)    (tsit5: e (bar + u)) -- fp64 only: an fp32 m and its sqrt are rounded to fp32, as
           in the restatement, and the probes keep m 2^-45 away from every fp32 rounding boundary
  log2     1 ulp of log2(er), then the multiply by e: |dX| <= 3u |X|, so ln2 3u |X| in 2^X
  exp2     2 ulp: 4u;  1/safety formed on the host and the multiply: 2u;  the final division: u
  The clamps divide dt by the host's fp64 1/ifactor or 1/dfactor, as the reference does: u.  m == 0: dt * ifactor, u.
  The flat band (m < 1, cand >= 1) divides by exactly 1: exact.
* ``ctrl_fast`` (persistent kernel), grow / shrink branches, with L = log2(sum err^2) - log2(tol^2 n):
  logs     1 ulp each, the subtraction and the multiply by -e/2: |dX| <= e u (|log2 sum err^2| + |log2 tol^2 n|) + 2u |X|,
           so ln2 |dX| in 2^X -- the two logarithms cancel, so the error follows their size, not L's
  exp2     4u;  the multiply by safety and by dt: 2u
  ratio    e/2 (bar + 2u): the sum is the family's, tol^2 n is rounded twice (exact for fp32 tol and small n)
  rounding the restatement rounds m and sqrt(m) to the state dtype, ctrl_fast does not: 1.5 e u (fp64), 1.5 e 2^-24 (fp32)
  The clamps multiply dt by ifactor or dfactor where the reference divides by their fp64 reciprocals: 2u.
Every bound carries one more u of slack.

This module is a plain helper (no fixtures); both test files import it.
"""
import collections
import functools
import math

import mpmath
import numpy as np

import np_ref
from problems import PROBLEMS

U = 2.0 ** -53
U32 = 2.0 ** -24
DPS = 60
H100_SMS = 132
METHODS = ("dopri5", "bosh3", "adaptive_heun", "dopri8")
DTYPES = ("float64", "float32")
OPTION_SETS = {"default": dict(safety=0.9, ifactor=10.0, dfactor=0.2),
               "odd": dict(safety=0.8, ifactor=5.0, dfactor=0.3)}
ORDER = {"dopri5": 5, "bosh3": 3, "adaptive_heun": 5, "dopri8": 8, "tsit5": 5}     # ctrl_order of each tableau
# h of each probe set: 1/16, except fp32 dopri8, whose error estimate at 1/16 is swamped by fp32 rounding in the stages
# (m then jitters as y0 moves, instead of following |y0|^2)
FIRST_STEP = {("dopri8", "float32"): 2.0 ** -2}
DIRECTION = np.array([1.0, -0.7, 0.4])                     # y0 = scale * DIRECTION: Lorenz near its fixed point at 0
BASE_SCALE = 1e-7                                          # the scale at which m = 1 (sets atol); the system is linear there
ACCEPT_EDGE = {"float64": 1e-9, "float32": 1e-6}           # m = 1 -+ this at the accept boundary
EDGE = {"float64": 1e-10, "float32": 1e-6}                 # least relative distance of cand from a branch boundary
EDGE_NEAR = 10.0                                           # an edge probe's cand lies within EDGE_NEAR * EDGE of its edge
SECOND_EDGE = {"float64": 1e-6, "float32": 1e-4}           # the second decision's margin from every boundary
ROUNDING_MARGIN = 2.0 ** -45                               # an fp32 m's least relative distance from an fp32 rounding boundary
WINDOW = (1.0 - 2.0 ** -25, 1.0)                           # exact ratios whose fp32 rounding is 1.0f, below 1


def _tf_f64(v):
    return float(np.float64(np.float32(v)))


def _sd(dtype):
    return np.dtype(dtype).type


def mpf(x):
    return mpmath.mpf(float(x))


def round_to(x, dtype):
    """x (mpf) correctly rounded to the dtype, as a python float."""
    if dtype == "float64":
        with mpmath.workprec(53):
            return float(+x)
    with mpmath.workprec(24):
        return float(+x)


# --------------------------------------------------------------------------------------------------
# the controller as the engine is given it
# --------------------------------------------------------------------------------------------------
Params = collections.namedtuple("Params", "safety ifactor dfactor exponent tsit5 q")


def params(method, opts):
    """safety, ifactor, dfactor through float32 (_tf_f64); the exponent of solvers.py _describe; q: the power of m in cand."""
    tsit5 = method == "tsit5"
    e = 1.0 / ORDER[method] if tsit5 else _tf_f64(1.0 / ORDER[method])
    return Params(_tf_f64(opts["safety"]), _tf_f64(opts["ifactor"]), _tf_f64(opts["dfactor"]), e, tsit5,
                  e if tsit5 else e / 2.0)


Decision = collections.namedtuple("Decision", "m_T branch cand dt_next")


def restate(dt, m_exact, P, dtype):
    """misc.py:267-287 / tsit5.py:53-62 at 60 digits on the exact ratio (mpf; already the max or the pooled value)."""
    with mpmath.workdps(DPS):
        m = round_to(m_exact, dtype)
        dt = mpf(dt)
        if m == 0:
            return Decision(0.0, "zero", mpmath.mpf(0), dt * mpf(P.ifactor))
        inv_df = mpmath.mpf(1) if m < 1 else mpf(1.0 / P.dfactor)
        er = mpf(m) if P.tsit5 else mpf(round_to(mpmath.sqrt(mpf(m)), dtype))
        cand = er ** mpf(P.exponent) / mpf(P.safety)
        inv_if = mpf(1.0 / P.ifactor)
        factor = max(inv_if, min(cand, inv_df))
        if factor == inv_if:
            branch = "ifactor"
        elif m < 1:
            branch = "flat" if factor == 1 else "grow"
        else:
            branch = "dfactor" if factor == inv_df else "shrink"
        return Decision(m, branch, cand, dt / factor)


def oracle_dt(dt, m_T, P, dtype):
    """np_ref's controller on the same state-dtype ratio."""
    m = _sd(dtype)(m_T)
    if P.tsit5:
        return float(np_ref.optimal_step_size_tsit5(dt, m, P.safety, P.ifactor, P.dfactor, 5))
    order = round(1.0 / P.exponent)
    return float(np_ref.optimal_step_size(dt, (m,), P.safety, P.ifactor, P.dfactor, order))


# --------------------------------------------------------------------------------------------------
# bounds
# --------------------------------------------------------------------------------------------------
def ratio_bar(family, dtype, n):
    """Relative error of a family's fp64 ratio: the persistent kernel's tagged partials (2^-48 on the sums; the suite's
    bar is 1e-12), or for ctrl_decide n rounded squares, n - 1 additions, tol^2 n and the division: (2n + 4) u.  Its
    fp32 ratio is rounded to fp32 and, on the probes, equals the restatement's."""
    if family == "persistent":
        return 1e-12
    return (2 * n + 4) * U


def dt_bound(impl, d, P, dtype, bar, ssq=None, tol2n=None):
    """Bound on |dt_next / d.dt_next - 1| for ctrl_decide ('decide') or ctrl_fast ('fast') at decision d; ssq and tol2n
    (the sum of squares and tol^2 n) are needed for 'fast'."""
    if d.branch == "flat":
        return 0.0
    if d.branch == "zero":
        return U
    if d.branch in ("ifactor", "dfactor"):
        return (2 if impl == "decide" else 3) * U
    er = d.m_T if P.tsit5 else math.sqrt(d.m_T)
    X = abs(P.exponent * math.log2(er))
    e = P.exponent
    ln2 = math.log(2.0)
    if impl == "decide":
        ratio = 0.0 if dtype == "float32" else (e * (bar + U) if P.tsit5 else e * ((bar + U) / 2 + 2 * U))
        return ratio + ln2 * 3 * U * X + 8 * U
    dX = e * U * (abs(math.log2(ssq)) + abs(math.log2(tol2n))) + 2 * U * X
    rounding = 1.5 * e * (U32 if dtype == "float32" else U)
    return ln2 * dX + 7 * U + e / 2 * (bar + 2 * U) + rounding


# --------------------------------------------------------------------------------------------------
# host emulations of the two controllers (and deliberately wrong variants)
# --------------------------------------------------------------------------------------------------
def emulate_decide(dt, m64, P, dtype, swap_exponent=False, raw_safety=None, f32_log2=False, skip_m_round=False):
    """ctrl_decide on the fp64 ratio m64 (one segment, or the pooled value for tsit5)."""
    T = _sd(dtype)
    m = m64 if skip_m_round else float(T(m64))
    if m == 0.0:
        return dt * P.ifactor
    inv_df = 1.0 if m < 1.0 else 1.0 / P.dfactor
    er = m if P.tsit5 else float(np.sqrt(T(m)))
    e = P.exponent
    if swap_exponent:
        order = round(1.0 / e)
        e = _tf_f64(1.0 / order) if P.tsit5 else 1.0 / order
    lg = float(np.log2(np.float32(er))) if f32_log2 else float(np.log2(er))
    inv_safety = 1.0 / (raw_safety if raw_safety is not None else P.safety)
    cand = float(np.exp2(e * lg)) * inv_safety
    factor = max(1.0 / P.ifactor, min(cand, inv_df))
    return dt / factor


def emulate_fast(dt, ssq, tol2n, P, dtype, old_df=False, f32_log2=False):
    """ctrl_fast on the sum of squares and tol^2 n (fp64 values, as the kernel has them).  old_df: the dfactor switch
    on the unrounded ratio (ssq < tol2n) that fp32 states had."""
    if ssq == 0.0:
        return dt * P.ifactor
    below = tol2n * (1.0 - 2.0 ** -25) if dtype == "float32" and not old_df else tol2n
    if f32_log2:
        L = float(np.log2(np.float32(ssq))) - float(np.log2(np.float32(tol2n)))
    else:
        L = float(np.log2(ssq)) - float(np.log2(tol2n))
    df = 1.0 if ssq < below else P.dfactor
    rf = P.safety * float(np.exp2(-0.5 * P.exponent * L))
    return dt * min(P.ifactor, max(df, rf))


def check_dt(got, d, bound):
    """None if got is within bound of decision d (bit for bit where the bound is 0), else a message."""
    want = float(d.dt_next)
    if bound == 0.0:
        return None if got == want else "%s: %r != %r" % (d.branch, got, want)
    with mpmath.workdps(DPS):
        rel = float(abs(mpf(got) / d.dt_next - 1))
    return None if rel <= bound else "%s: rel. error %.3e > bound %.3e (%.1f u vs %.1f u)" % (
        d.branch, rel, bound, rel / U, bound / U)


def rel_error(got, d):
    with mpmath.workdps(DPS):
        return float(abs(mpf(got) / d.dt_next - 1))


# --------------------------------------------------------------------------------------------------
# one attempt of the oracle, and its exact ratio
# --------------------------------------------------------------------------------------------------
_LORENZ = PROBLEMS["lorenz"](backend="numpy")


def attempt(method, y0, dt):
    """The oracle's attempt from t = 0 (rk_common.py): y0 a tuple of (rows, 3) arrays.  Returns (y1, err)."""
    tab = np_ref.TSIT5 if method == "tsit5" else np_ref.ADAPTIVE[method]
    f = lambda t, y: tuple(_LORENZ(t, c) for c in y)       # noqa: E731
    sd = y0[0].dtype.type
    f0 = f(np.float64(0.0) if method == "tsit5" else sd(0.0), y0)
    y1, _, err, _ = np_ref.runge_kutta_step(f, y0, f0, 0.0, dt, tab)
    return y1, err


Ratio = collections.namedtuple("Ratio", "m ms ssq tol n")


def exact_ratio(y0, y1, err, rtol, atol, pooled):
    """The engine's ratio, exactly: per component fsum(err^2) / (tol^2 n), tol in the state dtype (misc.py:257)."""
    ms, ssqs, tols, ns = [], [], [], []
    with mpmath.workdps(DPS):
        for e, a, b, rt, at in zip(err, y0, y1, rtol, atol):
            sd = a.dtype.type
            mx = max(float(np.max(np.abs(a))), float(np.max(np.abs(b))))
            tol = float(sd(sd(at) + sd(rt) * sd(mx)))
            ssq = mpmath.fsum(mpf(x) ** 2 for x in np.asarray(e).ravel())
            ms.append(ssq / (mpf(tol) ** 2 * e.size))
            ssqs.append(ssq)
            tols.append(tol)
            ns.append(e.size)
        if pooled:
            m = mpmath.fsum(s / mpf(t) ** 2 for s, t in zip(ssqs, tols)) / sum(ns)
        else:
            m = max(ms)
    return Ratio(m, ms, ssqs, tols, ns)


def max_ratio_T(r, dtype):
    """The engine's max over components of the state-dtype ratios (the pooled value, rounded, for tsit5)."""
    return max(round_to(m, dtype) for m in r.ms)


def rounding_margin(m, dtype):
    """Relative distance of an fp32 ratio from the nearest fp32 rounding boundary (inf for fp64 and m = 0)."""
    if dtype == "float64" or m == 0:
        return math.inf
    with mpmath.workdps(DPS):
        f = round_to(m, "float32")
        lo, hi = np.nextafter(np.float32(f), np.float32(0)), np.nextafter(np.float32(f), np.float32(np.inf))
        mids = (mpf(f) + mpf(lo)) / 2, (mpf(f) + mpf(hi)) / 2
        return float(min(abs(m - x) for x in mids) / m)


# --------------------------------------------------------------------------------------------------
# probes
# --------------------------------------------------------------------------------------------------
# regime: the first decision's branch, placed by y0.  REJECTING regimes are rejected and then retried at the step the
# controller chose until an attempt is accepted: twice for dopri5 and dopri8, more often for tableaus whose error
# estimate falls more slowly with dt than their controller exponent assumes (bosh3, adaptive_heun, tsit5).
Probe = collections.namedtuple("Probe", "name regime y0 ratios decisions dts jitters")
ProbeSet = collections.namedtuple("ProbeSet", "name method dtype opts P h atol rtol t probes")

REGIMES = ("zero", "ifactor_clamp", "ifactor_edge", "grow_edge", "grow", "grow_top", "flat_edge", "flat",
           "accept_edge", "window", "reject_edge", "shrink", "dfactor_edge", "dfactor_clamp")
REJECTING = ("reject_edge", "shrink", "dfactor_edge", "dfactor_clamp")
MAX_ATTEMPTS = 12
JITTER_SLACK = 4.0     # the ratio of a later attempt is held to JITTER_SLACK times its measured jitter (see jitter)


def _m_for_cand(c, P):
    """The exact ratio at which cand = c (cand = sqrt(m)^e / safety, tsit5: m^e / safety)."""
    return (P.safety * c) ** (1.0 / P.q)


def _target(regime, P, dtype):
    d, a = EDGE[dtype], ACCEPT_EDGE[dtype]
    inv_if, inv_df = 1.0 / P.ifactor, 1.0 / P.dfactor
    return {
        "ifactor_clamp": _m_for_cand(0.5 * inv_if, P),
        "ifactor_edge": _m_for_cand(inv_if * (1 - 3 * d), P),
        "grow_edge": _m_for_cand(inv_if * (1 + 3 * d), P),
        "grow": _m_for_cand(math.sqrt(inv_if), P),
        "grow_top": _m_for_cand(1 - 3 * d, P),
        "flat_edge": _m_for_cand(1 + 3 * d, P),
        "flat": (_m_for_cand(1.0, P) + 1.0) / 2,
        "accept_edge": 1.0 - a,
        "window": 1.0 - 2.0 ** -26,
        "reject_edge": 1.0 + a,
        "shrink": _m_for_cand(math.sqrt(inv_df), P),
        "dfactor_edge": _m_for_cand(inv_df * (1 - 3 * d), P),
        "dfactor_clamp": _m_for_cand(inv_df * 1.02, P),
    }[regime]


def _near(x, edge, side, dtype):
    """cand x lies on `side` (+1 above, -1 below) of edge, at least EDGE and at most EDGE_NEAR * EDGE away (relative)."""
    r = side * (x / edge - 1)
    return EDGE[dtype] <= r <= EDGE_NEAR * EDGE[dtype]


def _clear(x, P, edge):
    """cand x is at least `edge` (relative) away from every branch boundary."""
    return all(abs(x / b - 1) >= edge for b in (1.0 / P.ifactor, 1.0, 1.0 / P.dfactor))


def regime_holds(regime, d, m_exact, P, dtype):
    """The premise of a probe's first decision: its regime, with the stated margin."""
    cand = float(d.cand)
    inv_if, inv_df = 1.0 / P.ifactor, 1.0 / P.dfactor
    a = ACCEPT_EDGE[dtype]
    e = EDGE[dtype]
    m = float(m_exact)
    if regime == "zero":
        return m == 0 and d.branch == "zero"
    if regime == "window":
        with mpmath.workdps(DPS):
            return (mpf(WINDOW[0]) * (1 + ROUNDING_MARGIN) <= m_exact <= mpf(WINDOW[1]) * (1 - ROUNDING_MARGIN)
                    and d.m_T == 1.0 and d.branch == "shrink" and _clear(cand, P, e))
    if rounding_margin(m_exact, dtype) < ROUNDING_MARGIN:
        return False
    return {
        "ifactor_clamp": d.branch == "ifactor" and cand < inv_if * (1 - e),
        "ifactor_edge": d.branch == "ifactor" and _near(cand, inv_if, -1, dtype),
        "grow_edge": d.branch == "grow" and _near(cand, inv_if, +1, dtype),
        "grow": d.branch == "grow" and _clear(cand, P, e),
        "grow_top": d.branch == "grow" and _near(cand, 1.0, -1, dtype),
        "flat_edge": d.branch == "flat" and _near(cand, 1.0, +1, dtype) and m < 1 - a,
        "flat": d.branch == "flat" and _clear(cand, P, e) and m < 1 - a,
        "accept_edge": d.branch == "flat" and a / 2 <= 1 - m <= 2 * a and _clear(cand, P, e),
        "reject_edge": d.branch == "shrink" and a / 2 <= m - 1 <= 2 * a and _clear(cand, P, e),
        "shrink": d.branch == "shrink" and _clear(cand, P, e),
        "dfactor_edge": d.branch == "shrink" and _near(cand, inv_df, -1, dtype),
        "dfactor_clamp": d.branch == "dfactor" and cand > inv_df * (1 + e),
    }[regime]


def later_holds(d, m_exact, P, dtype, jit):
    """The premise of every decision after the first: robust against its ratio moving by ten times its jitter, with
    SECOND_EDGE to spare -- the accept decision, and cand's distance from every branch boundary (cand moves as m^q)."""
    e = SECOND_EDGE[dtype]
    spread = 1 + 10 * jit
    m = float(m_exact)
    robust = m * spread <= 1 - e if d.m_T <= 1 else m / spread >= 1 + e
    margin = P.q * math.log(spread) + e
    return m > 0 and robust and all(abs(math.log(float(d.cand) * b)) >= margin for b in (P.ifactor, 1.0, P.dfactor))


def jitter(method, y0, dt, atol, P, dtype):
    """Largest relative change of an attempt's exact ratio when its step moves by a few ulps.  A later attempt runs at
    the engine's step, which differs from the restated one by the controller's error; the error estimate cancels
    heavily (for dopri8 by ten digits), so its ratio moves by far more than that error.  fp64: dt (1 + k 2^-52) for
    |k| <= 256; fp32: also the step rounded to fp32 and one and two fp32 ulps away, as the stages see it."""
    def ratio(h):
        y1, err = attempt(method, (y0,), h)
        return exact_ratio((y0,), y1, err, (0.0,), (atol,), P.tsit5).m
    m0 = ratio(dt)
    steps = [dt * (1 + k * 2.0 ** -52) for j in (1, 2, 4, 16, 64, 256) for k in (j, -j)]
    if dtype == "float32":
        f = np.float32(dt)
        steps += [float(f), float(np.nextafter(f, np.float32(0))), float(np.nextafter(f, np.float32(1)))]
        steps += [float(np.nextafter(np.nextafter(f, np.float32(0)), np.float32(0))),
                  float(np.nextafter(np.nextafter(f, np.float32(1)), np.float32(1)))]
    with mpmath.workdps(DPS):
        return max(float(abs(ratio(h) / m0 - 1)) for h in steps) if m0 != 0 else 0.0


def _y0(scale, dtype, ulps=(0, 0, 0)):
    y = (scale * DIRECTION).astype(dtype)
    for i, k in enumerate(ulps):
        for _ in range(abs(k)):
            y[i] = np.nextafter(y[i], y.dtype.type(np.inf) if k > 0 else y.dtype.type(-np.inf))
    return y.reshape(1, 3)


def _evaluate(method, y0, h, atol, P, dtype, first_only=False):
    """(ratios, decisions, dts) of a probe's attempts from y0: attempt i runs at dts[i] (the restated step, rounded to
    fp64), until one is accepted or MAX_ATTEMPTS."""
    ratios, decisions, dts = [], [], [h]
    while True:
        y1, err = attempt(method, (y0,), dts[-1])
        r = exact_ratio((y0,), y1, err, (0.0,), (atol,), P.tsit5)
        d = restate(dts[-1], r.m, P, dtype)
        ratios.append(r)
        decisions.append(d)
        if d.m_T <= 1.0 or first_only or len(decisions) == MAX_ATTEMPTS:
            return ratios, decisions, dts
        dts.append(float(d.dt_next))


def _search(method, dtype, P, h, atol, regime):
    """y0 = scale * DIRECTION whose first ratio meets the regime: secant steps on the scale (m grows as scale^2 near the
    fixed point), then a grid of ulp perturbations of y0.  Returns y0 or None."""
    if regime == "zero":
        return np.zeros((1, 3), dtype=dtype)
    target = _target(regime, P, dtype)
    scale = BASE_SCALE * math.sqrt(target)
    best = (math.inf, scale)
    for _ in range(4):
        y0 = _y0(scale, dtype)
        r, d, _ = _evaluate(method, y0, h, atol, P, dtype, first_only=True)
        if regime_holds(regime, d[0], r[0].m, P, dtype):
            return y0
        m = float(r[0].m)
        best = min(best, (abs(math.log(m / target)), scale))
        scale *= math.sqrt(target / m)
    scale = best[1]      # rounding in the stages makes m jitter around scale^2: continue from the closest scale
    rng = range(-3, 4)
    for k in sorted(((a, b, c) for a in rng for b in rng for c in rng), key=lambda k: sum(map(abs, k))):
        y = _y0(scale, dtype, k)
        r, d, _ = _evaluate(method, y, h, atol, P, dtype, first_only=True)
        if regime_holds(regime, d[0], r[0].m, P, dtype):
            return y
    return None


def set_regimes(dtype):
    return [r for r in REGIMES if dtype == "float32" or r != "window"]


def _base_atol(method, dtype, h):
    """The atol at which y0 = BASE_SCALE * DIRECTION has m = 1 (rtol = 0)."""
    _, err = attempt(method, (_y0(BASE_SCALE, dtype),), h)
    with mpmath.workdps(DPS):
        ssq = mpmath.fsum(mpf(x) ** 2 for x in err[0].ravel())
        return round_to(mpmath.sqrt(ssq / 3), dtype)


def _build_set(method, dtype, opt_name, h):
    P = params(method, OPTION_SETS[opt_name])
    atol = _base_atol(method, dtype, h)
    found = {}
    if dtype == "float32":
        # the fp32 window is narrower than the ratio's steps from one y0 ulp to the next: search atol floats as well
        for k in sorted(range(-8, 9), key=abs):
            a = float(np.float32(atol) + 0)
            for _ in range(abs(k)):
                a = float(np.nextafter(np.float32(a), np.float32(np.inf if k > 0 else -np.inf)))
            y = _search(method, dtype, P, h, a, "window")
            if y is not None:
                atol, found["window"] = a, y
                break
    probes = []
    for regime in set_regimes(dtype):
        y0 = found.get(regime)
        if y0 is None:
            y0 = _search(method, dtype, P, h, atol, regime)
        if y0 is None:
            y0 = _y0(BASE_SCALE * math.sqrt(_target(regime, P, dtype)), dtype)     # fails its premises
        ratios, decisions, dts = _evaluate(method, y0, h, atol, P, dtype)
        jitters = [0.0] + [jitter(method, y0, dt, atol, P, dtype) for dt in dts[1:]]
        probes.append(Probe(regime, regime, y0, ratios, decisions, dts, jitters))
    name = "%s-%s-%s" % (method, "f64" if dtype == "float64" else "f32", opt_name)
    return ProbeSet(name, method, dtype, opt_name, P, h, atol, 0.0, np.array([0.0, h / 256]), probes)


def probe_premises(pr, ps):
    """Failed premises of one probe (an empty list when it meets them all)."""
    bad = []
    d, r = pr.decisions, pr.ratios
    if not regime_holds(pr.regime, d[0], r[0].m, ps.P, ps.dtype):
        bad.append("regime %s: m = %s, cand = %s, branch %s" % (pr.regime, mpmath.nstr(r[0].m, 15),
                                                                mpmath.nstr(d[0].cand, 15), d[0].branch))
    if (pr.regime in REJECTING) != (len(d) > 1):
        bad.append("%d attempts" % len(d))
    if d[-1].m_T > 1.0:
        bad.append("no attempt accepted in %d" % len(d))
    for i in range(1, len(d)):
        if not later_holds(d[i], r[i].m, ps.P, ps.dtype, pr.jitters[i]):
            bad.append("decision %d: m = %s, cand = %s" % (i + 1, mpmath.nstr(r[i].m, 15), mpmath.nstr(d[i].cand, 15)))
    if min(pr.dts) <= ps.t[-1]:
        bad.append("an attempt does not reach the output time")
    return bad


def tol2n(ps):
    return ps.atol * ps.atol * 3.0         # rtol = 0: tol = atol; exact in fp64 for an fp32 atol


def decision_bound(impl, d, r_ssq, ps, bar):
    return dt_bound(impl, d, ps.P, ps.dtype, bar, float(r_ssq), tol2n(ps))


def chain_bound(impl, pr, ps, bar):
    """Bound on the relative error of the step size the engine attempts last (dts[-1]) against the restated chain: each
    rejected attempt adds its decision's bound and the rounding of the restated step to fp64; a decision after the first
    that is not a clamp also moves with its ratio, by q times the ratio's error (the family's bar and JITTER_SLACK times
    the attempt's measured jitter)."""
    delta = 0.0
    for i, (d, r) in enumerate(zip(pr.decisions[:-1], pr.ratios[:-1])):
        sens = 0.0
        if i > 0 and d.branch not in ("ifactor", "dfactor"):
            sens = ps.P.q * (bar + JITTER_SLACK * pr.jitters[i])
        delta = delta + decision_bound(impl, d, r.ssq[0], ps, bar) + sens + U
    return delta


def ratio_tolerance(pr, ps, bar, impl):
    """Relative bound on |reported ratio / exact ratio of the last attempt - 1| (0: equal after rounding to fp32)."""
    if len(pr.decisions) == 1:
        return 0.0 if ps.dtype == "float32" else bar
    return bar + JITTER_SLACK * pr.jitters[-1]


def final_decision(pr, ps, m_reported):
    """The restated last decision at the engine's reported ratio, from the restated step it was attempted at."""
    return restate(pr.dts[-1], mpf(m_reported), ps.P, ps.dtype)


@functools.lru_cache(maxsize=None)
def probe_set(method, dtype, opt_name):
    """The probes of one (tableau, dtype, options) set."""
    return _build_set(method, dtype, opt_name, FIRST_STEP.get((method, dtype), 2.0 ** -4))


SETS = [(me, dt, op) for me in METHODS + ("tsit5",) for dt in DTYPES for op in OPTION_SETS]
SET_NAMES = ["%s-%s-%s" % (me, "f64" if dt == "float64" else "f32", op) for me, dt, op in SETS]


def set_by_name(name):
    return probe_set(*SETS[SET_NAMES.index(name)])


# --------------------------------------------------------------------------------------------------
# multi-segment probes (generic path, dopri5): a tuple of three Lorenz batches with per-component tolerances
# --------------------------------------------------------------------------------------------------
MultiProbe = collections.namedtuple("MultiProbe", "name dtype P h y0 rtol atol t ratio d argmax")


@functools.lru_cache(maxsize=None)
def multi_probe(kind, dtype):
    """kind 'last': the largest ratio is the last component's; 'zero': the second component is at the origin (m = 0) and
    the largest ratio is the first component's.  Both in the growth interval of the default options."""
    P = params("dopri5", OPTION_SETS["default"])
    h = 2.0 ** -5
    rng = np.random.default_rng(3)
    y0 = [np.asarray(1e-3 * (1 + 0.2 * rng.standard_normal((rows, 3))), dtype=dtype) for rows in (2, 1, 3)]
    if kind == "zero":
        y0[1][:] = 0
    y1, err = attempt("dopri5", tuple(y0), h)
    m_top = _m_for_cand(math.sqrt(1.0 / P.ifactor), P)
    share = (0.3, 0.5, 1.0) if kind == "last" else (1.0, 1.0, 0.4)
    rtol = [1e-5, 2e-5, 5e-6]
    atol = []
    for i in range(3):
        ssq = float(np.sum(err[i].astype(np.float64) ** 2)) or 1.0
        mx = max(float(np.max(np.abs(y0[i]))), float(np.max(np.abs(y1[i]))))
        tol = math.sqrt(ssq / (err[i].size * m_top * share[i]))
        atol.append(float(_sd(dtype)(max(tol - rtol[i] * mx, tol / 2))))
    r = exact_ratio(tuple(y0), y1, err, rtol, atol, False)
    d = restate(h, r.m, P, dtype)
    argmax = max(range(3), key=lambda i: r.ms[i])
    return MultiProbe("multi-%s-%s" % (kind, dtype), dtype, P, h, tuple(y0), rtol, atol, np.array([0.0, h / 256]), r, d,
                      argmax)


def multi_premises(mp):
    bad = []
    kind = mp.name.split("-")[1]
    want = 2 if kind == "last" else 0
    if mp.argmax != want:
        bad.append("largest ratio in component %d" % mp.argmax)
    others = sorted(float(m) for i, m in enumerate(mp.ratio.ms) if i != mp.argmax)
    if not others[-1] < 0.9 * float(mp.ratio.ms[mp.argmax]):
        bad.append("largest ratio not clear of the others")
    if kind == "zero" and mp.ratio.ms[1] != 0:
        bad.append("the middle component's ratio is not 0")
    if not (mp.d.branch == "grow" and _clear(float(mp.d.cand), mp.P, SECOND_EDGE[mp.dtype])):
        bad.append("not clear inside the growth interval: cand %s" % mpmath.nstr(mp.d.cand, 15))
    if rounding_margin(mp.ratio.m, mp.dtype) < ROUNDING_MARGIN:
        bad.append("fp32 ratio close to a rounding boundary")
    return bad
