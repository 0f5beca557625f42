"""Exact step schedules: adaptive solves the engine must reproduce bit for bit (DESIGN.md section 2).

With ``safety=0.5, ifactor=1, dfactor=0.5`` and a power-of-two ``first_step`` the reference controller
(``np_ref.optimal_step_size``, ``optimal_step_size_tsit5``) keeps ``dt`` after an accepted attempt
(factor max(1, min(cand, 1)) = 1) and halves it after a rejected one (cand = 2 sqrt(m)^e > 2, so factor = 2).
The engine's controllers (``ctrl_decide``, ``ctrl_fast``) give the same exact values, without a log, exp or pow
reaching dt.  All three option values are exact in float32, which matters because options are rounded through
float32 (``_tf_f64``).  Every step size is then ``first_step * 2**-k`` and every step end a dyadic sum, so each
stage, each ``t1 = t0 + dt`` and each dense output is a chain of correctly rounded IEEE operations.  For
right-hand sides built from +, -, * only, the engine must equal ``oracle/np_ref.py`` exactly, provided no
attempt's error ratio m lies so close to 1 that a rounding difference in the error norm could flip the decision.
``tests/test_exact_schedule_cpu.py`` checks that premise, and the others below, on the oracle for every case
``tests/test_exact_schedule_gpu.py`` runs.

This module is a plain helper (no fixtures); both test files import it.
"""
import collections
import contextlib
import math

import numpy as np

import np_ref
from problems import PROBLEMS

OPTIONS = dict(safety=0.5, ifactor=1.0, dfactor=0.5)
H100_SMS = 132                 # SMs of an H100 SXM: the geometry the CPU test checks
DENSE_ROWS = 3                 # kDenseRows of the persistent kernel for the instantiations below (rows buffered per step)
MAX_ATTEMPTS = 200
MARGIN = {"float64": 1e-9, "float32": 1e-4}      # least |m - 1| that keeps every accept decision robust
N_K = {"adaptive_heun": 2, "bosh3": 4, "dopri5": 7, "tsit5": 7, "dopri8": 14}
DIM = {"lorenz": 3, "lv": 2}


# --------------------------------------------------------------------------------------------------
# the persistent kernel's block geometry (fused_dispatch_s, FusedShape and fused_geometry in b2ode_fused.cu)
# --------------------------------------------------------------------------------------------------
def fused_budget(method, dtype, dim):
    """(MAXT, trajectories per thread) of the k_fused_adaptive instantiation."""
    n_k = N_K[method]
    maxt = {2: 512, 4: 512, 7: 576, 14: 256}[n_k]
    tpt = 2 if n_k == 7 and not (dtype == "float64" and dim > 3) else 1
    return maxt, tpt


Geometry = collections.namedtuple("Geometry", "ncw grid pcw tpt last_traj features")


def fused_geometry(n, sm_count, method, dtype, dim, nsvc=1):
    """Block shape of a batch of n trajectories on a device of `sm_count` SMs, for batches that fit one block per SM
    (the kernel shrinks blocks further when a capped shape cannot stay co-resident; that case is not modelled).

    per_block = ceil(n / SMs), ncw = ceil(per_block / 32) trajectory warps (capped at MAXT / 32 - nsvc), grid =
    ceil(n / (32 ncw)); compute warp w carries trajectory warps w, w + pcw, ... with pcw = ceil(ncw / tpt)."""
    maxt, tpt = fused_budget(method, dtype, dim)
    per_block = -(-n // sm_count)
    ncw = min(max(1, -(-per_block // 32)), maxt // 32 - nsvc)
    grid = -(-n // (32 * ncw))
    if grid > sm_count:
        raise ValueError("batch %d needs %d blocks of %d trajectory warps on %d SMs" % (n, grid, ncw, sm_count))
    pcw = -(-ncw // tpt)
    last = n - (grid - 1) * 32 * ncw                 # trajectories of the last block
    live_warps = -(-last // 32)
    feats = set()
    if ncw > 1:
        feats.add("multi_warp")
    if tpt > 1 and pcw * tpt > ncw:
        feats.add("dead_second_slot")                # a compute warp whose second trajectory warp does not exist
    if tpt > 1 and ncw > pcw:
        feats.add("live_second_slot")                # some compute warp carries two trajectory warps
    if last % 32:
        feats.add("last_block_partial_warp")
    if live_warps < ncw:
        feats.add("last_block_dead_warp")
    if last == 1 and grid > 1:
        feats.add("last_block_one_trajectory")
    if ncw > 1 and last % 32 and 1 < live_warps:
        feats.add("last_block_later_warp_partial")   # the partly live warp is not the block's first
    return Geometry(ncw, grid, pcw, tpt, last, frozenset(feats))


# batches named by the shape they give; each a function of the SM count (the values at 132 SMs in brackets)
BATCHES = {
    "one": lambda sms: 1,
    "ncw2_tail1": lambda sms: 32 * sms + 1,            # [4 225] ncw 2; the last block holds one trajectory
    "ncw3_full": lambda sms: 96 * sms,                 # [12 672] ncw 3, every block full; a dead second slot
    "ncw3_partial": lambda sms: 96 * (sms - 1) + 51,   # [12 627] ncw 3; last block: warp 1 partly live, warp 2 dead
    "full": lambda sms: 65536,                         # ncw 16 (dopri5)
}

# shape features each named batch must produce at 132 SMs, per trajectories-per-thread
BATCH_FEATURES = {
    ("one", 1): {"ncw": 1, "has": {"last_block_partial_warp"}},
    ("ncw2_tail1", 2): {"ncw": 2, "has": {"multi_warp", "live_second_slot", "last_block_one_trajectory",
                                          "last_block_partial_warp", "last_block_dead_warp"}},
    ("ncw2_tail1", 1): {"ncw": 2, "has": {"multi_warp", "last_block_one_trajectory", "last_block_dead_warp"}},
    ("ncw3_full", 2): {"ncw": 3, "has": {"multi_warp", "live_second_slot", "dead_second_slot"},
                       "not": {"last_block_partial_warp", "last_block_dead_warp"}},
    ("ncw3_full", 1): {"ncw": 3, "has": {"multi_warp"}, "not": {"last_block_partial_warp"}},
    ("ncw3_partial", 2): {"ncw": 3, "has": {"multi_warp", "live_second_slot", "dead_second_slot",
                                            "last_block_partial_warp", "last_block_dead_warp",
                                            "last_block_later_warp_partial"}},
    ("ncw3_partial", 1): {"ncw": 3, "has": {"multi_warp", "last_block_partial_warp", "last_block_dead_warp",
                                            "last_block_later_warp_partial"}},
    ("full", 2): {"ncw": 16, "has": {"multi_warp", "live_second_slot"}},
}


# --------------------------------------------------------------------------------------------------
# cases
# --------------------------------------------------------------------------------------------------
def _t_grid(horizon, step_ends, cluster):
    """Output times over [0, horizon] (negated for reverse time by the caller): a coarse non-dyadic grid over the second
    half (the steps before it have no output), a cluster of `cluster` non-dyadic times 1e-6 apart (more rows than the
    kernel buffers, inside one step) and the dyadic times `step_ends`, which an exact schedule reaches exactly (every step
    end is a multiple of the current dt)."""
    grid = list(np.linspace(0.55 * horizon, horizon, 7) * (1.0 - 1.0 / 3001.0))
    c0 = 0.4137 * horizon
    t = sorted(set([0.0] + [c0 + (q + 0.37) * 1e-6 for q in range(cluster)] + grid + list(step_ends)))
    return np.array(t, dtype=np.float64)


Case = collections.namedtuple("Case", "name problem method dtype reverse batch rtol atol first_step t seed outlier")

# (rtol, atol) per system, tableau and dtype (float64, float32): tight enough for rejections and several steps, loose enough
# for at most MAX_ATTEMPTS attempts (tsit5's error estimate as written keeps its steps short)
TOLERANCES = {
    ("lorenz", "dopri5"): ((1e-6, 1e-8), (1e-4, 1e-5)),
    ("lorenz", "tsit5"): ((1e-1, 1e-2), (1e-1, 1e-2)),
    ("lorenz", "dopri8"): ((1e-9, 1e-11), (1e-7, 1e-8)),
    ("lorenz", "bosh3"): ((1e-3, 1e-5), (1e-3, 1e-4)),
    ("lorenz", "adaptive_heun"): ((1e-3, 1e-5), (1e-3, 1e-4)),
    ("lv", "dopri5"): ((1e-8, 1e-10), (1e-5, 1e-6)),
    ("lv", "dopri8"): ((1e-11, 1e-13), (1e-6, 1e-7)),
    ("lv", "bosh3"): ((1e-3, 1e-5), (1e-3, 1e-4)),
    ("lv", "adaptive_heun"): ((1e-3, 1e-5), (1e-3, 1e-4)),
    ("kepler", "dopri5"): ((1e-6, 1e-8), None),
    ("cubic", "dopri5"): ((1e-10, 1e-12), (1e-6, 1e-7)),
}
HORIZON = {"lorenz": 0.25, "lv": 2.0, "kepler": 1.0, "cubic": 2.0}   # forward; reverse time goes half as far
FIRST_STEP = {"lorenz": 0.25, "lv": 1.0, "kepler": 0.5, "cubic": 2.0}


def _case(problem, method, dtype, reverse, batch, outlier=None, seed=7, first_step=True):
    name = "%s-%s-%s-%s-%s" % (problem, method, "f64" if dtype == "float64" else "f32", "rev" if reverse else "fwd", batch)
    if outlier is not None:
        name += "-row%d" % outlier
    if first_step is None:
        name += "-h0"
    horizon = HORIZON[problem] / (2.0 if reverse else 1.0)
    t = _t_grid(horizon, (horizon / 2,), 5)
    rtol, atol = TOLERANCES[problem, method][0 if dtype == "float64" else 1]
    fs = FIRST_STEP[problem] if first_step is True else first_step
    return Case(name, problem, method, dtype, reverse, batch, rtol, atol, fs, -t if reverse else t, seed, outlier)


METHODS = ("dopri5", "bosh3", "adaptive_heun", "dopri8")
DTYPES = ("float64", "float32")

# persistent kernel: every system x tableau x dtype x direction at the partial-block shape, and a sweep of the shapes
PERSISTENT = [_case(pr, me, dt, rev, "ncw3_partial") for pr in ("lorenz", "lv") for me in METHODS for dt in DTYPES
              for rev in (False, True)]
PERSISTENT += [_case("lorenz", "dopri5", dt, rev, b) for dt in DTYPES for rev in (False, True)
               for b in ("one", "ncw2_tail1", "ncw3_full")]
PERSISTENT += [_case("lorenz", "dopri5", "float64", False, "full"), _case("lv", "dopri5", "float32", True, "full")]
PERSISTENT += [_case(pr, me, "float64", False, b) for me in ("bosh3", "adaptive_heun", "dopri8")
               for pr, b in (("lorenz", "ncw2_tail1"), ("lv", "ncw3_full"))]
# at the instantiation's own capacity (b2ode_fused_capacity, known on the device only): premises checked at run time
CAPACITY = [_case("lorenz", me, "float64", False, "capacity") for me in METHODS] + [
    _case("lv", "dopri5", "float32", True, "capacity")]

# rows the outlier (and the NaN) is placed at: trajectory warps 0..2 of block 0, the second slot of compute warp 0 (row 64),
# block 1 (row 96), and the last block's first row, its partly live trajectory warp and the last row
OUTLIER_ROWS = lambda sms: (0, 31, 32, 95, 64, 96, 96 * (sms - 1), 96 * (sms - 1) + 32, 96 * (sms - 1) + 50)   # noqa: E731
OUTLIER = [_case("lorenz", "dopri5", "float64", False, "ncw3_partial", outlier=r) for r in OUTLIER_ROWS(H100_SMS)]

# the generic (per-stage) path, forward and reverse; tsit5 only has it
GENERIC = [_case("lorenz", me, dt, rev, "ncw3_partial") for me in ("dopri5", "tsit5") for dt in DTYPES
           for rev in (False, True)]

# first_step=None: the initial-step heuristic (k_init_* kernels, and the persistent kernel's own two reductions)
INITIAL = [_case("lorenz", me, dt, False, "ncw3_partial", first_step=None) for me in ("dopri5", "dopri8") for dt in DTYPES]

# persistent kernel against the stage kernels on right-hand sides that are not +, -, * only (pow, tanh)
NON_BASIC = [_case("kepler", "dopri5", "float64", False, "r1000")] + [
    _case("cubic", "dopri5", dt, False, "ncw3_partial") for dt in DTYPES]

# bulk finalize: 65 536 x 3 is 384 whole 512-element tiles; 4 099 x 3 leaves a remainder
BULK = [_case("lorenz", "dopri5", "float64", False, "full"), _case("lorenz", "dopri5", "float64", False, "r4099"),
        _case("lorenz", "dopri5", "float32", False, "r4099")]

ALL = {c.name: c for c in PERSISTENT + OUTLIER + GENERIC + INITIAL + NON_BASIC + BULK}


def batch_size(case, sms):
    if case.batch.startswith("r"):
        return int(case.batch[1:])
    return BATCHES[case.batch](sms)


KEPLER_ORBITS = 8     # orbits per row of the Kepler state: (n, 4 * 8), i.e. 8 n trajectories of the kernels


def cubic_weights(dtype):
    """W1, b1, W2, b2 of rhs.CubicMLP(hidden=50) built from generator seed 0 (torch CPU), as numpy arrays."""
    import torch
    g = torch.Generator().manual_seed(0)
    tdt = torch.float64 if dtype == "float64" else torch.float32
    w = [torch.randn(2, 50, dtype=tdt, generator=g) * 0.1, torch.zeros(50, dtype=tdt),
         torch.randn(50, 2, dtype=tdt, generator=g) * 0.1, torch.zeros(2, dtype=tdt)]
    return [x.numpy() for x in w]


def initial_state(case, n):
    """n rows near a common point, the same for a given (problem, seed) and n; the `outlier` row gets a far larger state,
    which dominates both the sum of err^2 and max|y|."""
    rng = np.random.default_rng(case.seed)
    if case.problem == "lorenz":
        y0 = np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((n, 3))
        if case.outlier is not None:
            y0[case.outlier] = 100.0
    elif case.problem == "lv":
        y0 = 1.0 + 0.3 * rng.random((n, 2))
    elif case.problem == "kepler":
        y0 = PROBLEMS["kepler"](orbits=KEPLER_ORBITS).y0(n, seed=case.seed)
    else:
        y0 = np.array([2.0, 0.0]) + 0.1 * rng.standard_normal((n, 2))
    return y0.astype(case.dtype)


def numpy_rhs(case):
    if case.problem == "kepler":
        return PROBLEMS["kepler"](orbits=KEPLER_ORBITS)
    if case.problem == "cubic":
        W1, b1, W2, b2 = cubic_weights(case.dtype)
        return lambda t, y: np.tanh((y ** 3) @ W1 + b1) @ W2 + b2     # noqa: E731
    return PROBLEMS[case.problem](backend="numpy")


def tuple_case(dtype):
    """A tuple state of odd-length components with per-component tolerances (generic path only): two Lorenz batches of
    4 099 and 7 rows (12 297 and 21 elements) and a Lotka-Volterra batch of 1 001 rows (2 002 elements: not a whole
    number of fp32 16-byte packs).  Returns (y0 tuple, numpy func, rtol list, atol list, t, first_step)."""
    rng = np.random.default_rng(11)
    y0 = (np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((4099, 3)), 1.0 + 0.3 * rng.random((1001, 2)),
          np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((7, 3)))
    y0 = tuple(y.astype(dtype) for y in y0)
    lo, lv = PROBLEMS["lorenz"](backend="numpy"), PROBLEMS["lv"](backend="numpy")
    func = lambda t, y: (lo(t, y[0]), lv(t, y[1]), lo(t, y[2]))      # noqa: E731
    if dtype == "float64":
        rtol, atol = [1e-6, 1e-8, 1e-5], [1e-8, 1e-10, 1e-7]
    else:
        rtol, atol = [1e-4, 1e-5, 1e-3], [1e-5, 1e-6, 1e-4]
    return y0, func, rtol, atol, _t_grid(0.25, (0.125,), 5), 0.25


# --------------------------------------------------------------------------------------------------
# the oracle, recording every attempt
# --------------------------------------------------------------------------------------------------
def reference_ratio(err, y0, y1, rtol, atol, pooled=False):
    """The error ratio of one attempt as the engine defines it, exactly summed: per component
    m = fsum(err^2) / (tol^2 n) with tol = atol + rtol * max(|y0|, |y1|) in the state dtype (misc.py:257); the max over
    components, or for tsit5 the pooled sum(err^2 / tol^2) / sum(n) (tsit5.py:126-132)."""
    ms, pooled_sum, pooled_n = [], [], 0
    for e, a, b, rt, at in zip(err, y0, y1, rtol, atol):
        sd = a.dtype.type
        mx = max(float(np.max(np.abs(a))), float(np.max(np.abs(b))))
        tol = float(sd(at) + sd(rt) * sd(mx))
        ssq = math.fsum((np.asarray(e, dtype=np.float64).ravel()) ** 2)
        ms.append(ssq / (tol * tol * float(e.size)))
        pooled_sum.append(ssq / (tol * tol))
        pooled_n += e.size
    return math.fsum(pooled_sum) / pooled_n if pooled else max(ms)


class Record(object):
    def __init__(self):
        self.t0, self.dt, self.m = [], [], []
        self.last = None          # (y0, y1, err) of the last attempt


@contextlib.contextmanager
def _recording(rec, rtol, atol, pooled):
    orig = np_ref.runge_kutta_step

    def step(func, y0, f0, t0, dt, tableau):
        res = orig(func, y0, f0, t0, dt, tableau)
        rec.t0.append(float(t0))
        rec.dt.append(float(dt))
        rec.m.append(reference_ratio(res[2], y0, res[0], rtol, atol, pooled))
        rec.last = (y0, res[0], res[2])
        return res
    np_ref.runge_kutta_step = step
    try:
        yield
    finally:
        np_ref.runge_kutta_step = orig


Solve = collections.namedtuple("Solve", "sol stats rec dt_next t")


def oracle_solve(func, y0, t, method, rtol, atol, options):
    """np_ref.odeint (misc.py:290-329 wrapping included) that also returns the final state's dt and the attempt record.
    y0: an array or a tuple of arrays; rtol / atol: scalars or per-component lists."""
    tensor_input = not isinstance(y0, tuple)
    f = func
    if tensor_input:
        y0 = (y0,)
        f = lambda t_, y_: (func(t_, y_[0]),)                 # noqa: E731
    t = np.asarray(t, dtype=np.float64)
    if len(t) > 1 and bool(np.all(t[1:] < t[:-1])):
        t = -t
        fwd = f
        f = lambda t_, y_: tuple(-v for v in fwd(-t_, y_))   # noqa: E731
    st = np_ref.Stats()
    if method == "tsit5":
        solver = np_ref.Tsit5(f, y0, rtol, atol, stats=st, **options)
    else:
        solver = np_ref.AdaptiveRK(f, y0, rtol, atol, np_ref.ADAPTIVE[method], stats=st, **options)
    rec = Record()
    rl = np_ref._listify(rtol, len(y0))
    al = np_ref._listify(atol, len(y0))
    with _recording(rec, rl, al, pooled=method == "tsit5"):
        sol = solver.integrate(t)
    return Solve(sol[0] if tensor_input else sol, st, rec, float(solver.state[4]), t)


def solve_case(case, sms=H100_SMS, n=None):
    """(y0, oracle Solve) of a case at n rows (default: its batch at `sms` SMs)."""
    n = batch_size(case, sms) if n is None else n
    y0 = initial_state(case, n)
    opts = dict(OPTIONS, first_step=case.first_step)
    return y0, oracle_solve(numpy_rhs(case), y0, case.t, case.method, case.rtol, case.atol, opts)


# --------------------------------------------------------------------------------------------------
# premises of an exact comparison, from the oracle's record
# --------------------------------------------------------------------------------------------------
def steps_with_rows(s):
    """(t0, t1, rows in (t0, t1]) of every accepted attempt, in the oracle's (increasing) time."""
    out = []
    for t0, dt, ok in zip(s.rec.t0, s.rec.dt, s.stats.acc_trace):
        if ok:
            t1 = t0 + dt
            out.append((t0, t1, [j for j in range(1, len(s.t)) if t0 < s.t[j] <= t1]))
    return out


def premises(s, first_step=None):
    """Facts about an oracle solve that decide what a bit-exact comparison with it proves (first_step None: the step
    sizes are checked against the oracle's initial step)."""
    first_step = s.rec.dt[0] if first_step is None else first_step
    dyadic = all(dt == first_step * 2.0 ** round(math.log2(dt / first_step)) and dt <= first_step for dt in s.rec.dt)
    decisions_agree = all((m <= 1.0) == ok for m, ok in zip(s.rec.m, s.stats.acc_trace))
    steps = steps_with_rows(s)
    ends = {t1 for _, t1, _ in steps}
    on_end = [j for j in range(1, len(s.t)) if s.t[j] in ends]
    others = [j for j in range(1, len(s.t)) if j not in on_end]
    return dict(
        dyadic=dyadic,
        decisions_agree=decisions_agree,
        margin=min(abs(m - 1.0) for m in s.rec.m),
        attempts=len(s.rec.m),
        n_rej=s.stats.n_rej,
        max_rows=max(len(r) for _, _, r in steps),
        empty_steps=sum(1 for _, _, r in steps if not r),
        rows_on_step_end=len(on_end),
        # every other output time has a full mantissa, so x = (t - t0) / (t1 - t0) and its powers are rounded
        others_non_dyadic=all(s.t[j] * 2.0 ** 30 != math.floor(s.t[j] * 2.0 ** 30) for j in others),
    )
