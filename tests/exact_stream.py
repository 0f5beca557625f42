"""Exact comparisons of the generic path at the sizes where its kernels stride over their grid (DESIGN.md section 2).

The streaming kernels (k_rk_stage, k_rk_stage0, k_rk_finalize, k_emit_*, k_init_*, k_fixed, k_lincomb, k_reduce) launch
at most 8 x SMs blocks of 256 threads (build_geom, b2ode.cu); seg_for_each (b2ode_dev.cuh) loops over that grid when a
segment is larger, and block 0 finishes the scalar tail of a vector segment.  The row-per-thread kernels k_rk_stage_rhs
(launch_stage_rhs_t) and k_fused_fixed (fused_fixed_dispatch) loop the same way over rows.  The cases below are sized so
that at 132 SMs (H100 SXM) every one of those loops runs several passes, with partial last passes, and the functions
below restate the launch geometry so that the CPU test can check which features each case reaches and the GPU test can
re-check them at the device's own SM count.

The adaptive cases run under tests/exact_schedule.py's exact step schedule and reuse its oracle and premises.  The
north-star system is made exact by its matrix (problems.ExactLinear): at most two non-zero entries per column, each a
power of two, so every output of ``y @ A`` is one correctly rounded sum in any summation order.

This module is a plain helper (no fixtures); both test files import it.
"""
import collections

import numpy as np

import exact_schedule as es
from problems import PROBLEMS

KTHREADS = 256                 # kThreads (b2ode_dev.cuh)
BLOCKS_PER_SM = 8              # the grid cap of every streaming and row kernel: 8 x 256 threads per SM
H100_SMS = es.H100_SMS


def vector_width(dtype):
    """Elements per 16-byte pack (VW in seg_for_each)."""
    return 16 // np.dtype(dtype).itemsize


# --------------------------------------------------------------------------------------------------
# launch geometry
# --------------------------------------------------------------------------------------------------
SegPlan = collections.namedtuple("SegPlan", "n blocks vector passes tail")
SegGeom = collections.namedtuple("SegGeom", "segs grid cap_exceeded")


def build_geom(seg_lens, dtype, sms, vector=None):
    """build_geom (b2ode.cu) and seg_for_each (b2ode_dev.cuh) for segments of `seg_lens` elements.

    Each segment needs ceil(ceil(n / VW) / 256) blocks (at least 1).  If the segments need more than 8 x SMs in all,
    segment s gets floor(cap * need_s / total) blocks, at least 1.  vector[s] says whether the launch takes the 16-byte
    path for segment s (every pointer 16-byte aligned; for k_emit_* also n % VW == 0), default True.  A vector segment
    runs `passes` = ceil((n // VW) / (blocks * 256)) passes over its packs and block 0 then handles the `tail` of
    n % VW elements; a scalar segment runs ceil(n / (blocks * 256)) passes over single elements."""
    w = vector_width(dtype)
    cap = sms * BLOCKS_PER_SM
    need = [max(1, -(-(-(-n // w)) // KTHREADS)) for n in seg_lens]
    tot = sum(need)
    over = tot > cap
    segs = []
    for s, n in enumerate(seg_lens):
        nb = max(1, int(float(cap) * float(need[s]) / float(tot))) if over else need[s]   # the C code's double arithmetic
        vec = True if vector is None else bool(vector[s])
        stride = nb * KTHREADS
        if vec:
            segs.append(SegPlan(n, nb, True, -(-(n // w) // stride), n % w))
        else:
            segs.append(SegPlan(n, nb, False, -(-n // stride), 0))
    return SegGeom(tuple(segs), sum(p.blocks for p in segs), over)


RowGrid = collections.namedtuple("RowGrid", "grid passes partial")


def row_grid(rows, sms):
    """The grid of the one-thread-per-row kernels, k_rk_stage_rhs (launch_stage_rhs_t, b2ode.cu) and k_fused_fixed
    (fused_fixed_dispatch, b2ode_fused.cu): min(max(1, ceil(rows / 256)), 8 x SMs) blocks; thread r handles rows
    r, r + grid * 256, ...  `partial`: the last pass covers only part of the grid."""
    grid = max(1, min(-(-rows // KTHREADS), sms * BLOCKS_PER_SM))
    stride = grid * KTHREADS
    return RowGrid(grid, -(-rows // stride), rows % stride != 0)


# --------------------------------------------------------------------------------------------------
# cases
# --------------------------------------------------------------------------------------------------
# Lorenz on the generic path: an odd element count, so the 16-byte loops leave a scalar tail and the dense output takes
# the scalar path (its rows are not 16-byte aligned); fp64: 4 vector passes and 1 tail element, fp32: 3 passes, 3 elements
LORENZ_ROWS = {"float64": 600001, "float32": 750001}
TSIT5_TOL = (5e-2, 5e-3)       # at these sizes exact_schedule's tsit5 tolerances take the horizon in one step


def _lorenz(method, dtype, reverse, **kw):
    c = es._case("lorenz", method, dtype, reverse, "r%d" % LORENZ_ROWS[dtype], **kw)
    return c._replace(rtol=TSIT5_TOL[0], atol=TSIT5_TOL[1]) if method == "tsit5" else c


LORENZ = [_lorenz(me, dt, rev) for me in ("dopri5", "tsit5") for dt in es.DTYPES for rev in (False, True)]
# first_step=None: k_init_* over the same state
INITIAL = [_lorenz("dopri5", "float64", False, first_step=None)]
ALL = {c.name: c for c in LORENZ + INITIAL}


# the north-star solve: bench.py's northstar workload (65 536 x 128 fp64 dopri5, seed-100 normal y0, rtol 1e-6,
# atol 1e-9) with its matrix replaced by ExactLinear's
LinearCase = collections.namedtuple("LinearCase", "name rows dim seed y0_seed t rtol atol first_step")
NORTH_STAR = LinearCase("northstar", 65536, 128, 0, 100, es._t_grid(2.0, (1.0,), 5), 1e-6, 1e-9, 1.0)
# reverse time on a smaller state, still 4 vector passes in fp64: the -A image of the tensor-core kernel
REVERSE_LINEAR = LinearCase("linear-rev", 65537, 32, 1, 101, -es._t_grid(1.0, (0.5,), 5), 1e-8, 1e-10, 1.0)


def linear_problem(case, backend="numpy", device=None):
    return PROBLEMS["exact_linear"](backend=backend, device=device, dim=case.dim, seed=case.seed)


def linear_y0(case):
    return np.random.default_rng(case.y0_seed).standard_normal((case.rows, case.dim))


def solve_linear(case):
    """(y0, oracle Solve) of a LinearCase."""
    y0 = linear_y0(case)
    opts = dict(es.OPTIONS, first_step=case.first_step)
    return y0, es.oracle_solve(linear_problem(case), y0, case.t, "dopri5", case.rtol, case.atol, opts)


# a tuple state of all B2ODE_MAXSEG = 12 components, large enough in all that build_geom splits the grid in proportion:
# (system, rows) per component.  Component 0 is a single row, component 5 gets one block that loops over several passes,
# and the func returns component MISALIGNED as a view at an odd element offset (the scalar path of every kernel that
# reads func's outputs)
TUPLE12 = (("lorenz", 1), ("lv", 500001), ("lorenz", 333333), ("lorenz", 150001), ("lv", 1001), ("lorenz", 1500),
           ("lv", 7), ("lorenz", 4099), ("lv", 250000), ("lorenz", 17), ("lv", 2), ("lorenz", 33333))
MISALIGNED = 3
ONE_BLOCK = 5
TUPLE12_TOL = {"float64": {"lorenz": (1e-6, 1e-8), "lv": (1e-7, 1e-9)},
               "float32": {"lorenz": (1e-4, 1e-5), "lv": (1e-4, 1e-5)}}


def tuple12_lens():
    return [rows * es.DIM[pr] for pr, rows in TUPLE12]


def tuple12_case(dtype):
    """(y0 tuple, numpy func, rtol list, atol list, t, first_step) of the 12-component state."""
    rng = np.random.default_rng(12)
    y0 = []
    for pr, rows in TUPLE12:
        if pr == "lorenz":
            y0.append(np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((rows, 3)))
        else:
            y0.append(1.0 + 0.3 * rng.random((rows, 2)))
    y0 = tuple(y.astype(dtype) for y in y0)
    fs = {pr: PROBLEMS[pr](backend="numpy") for pr in ("lorenz", "lv")}
    func = lambda t, y: tuple(fs[pr](t, c) for (pr, _), c in zip(TUPLE12, y))      # noqa: E731
    # every component its own tolerances: scale the system's pair by a power of two per component
    rtol = [TUPLE12_TOL[dtype][pr][0] * 2.0 ** (i % 3) for i, (pr, _) in enumerate(TUPLE12)]
    atol = [TUPLE12_TOL[dtype][pr][1] * 2.0 ** (i % 2) for i, (pr, _) in enumerate(TUPLE12)]
    return y0, func, rtol, atol, es._t_grid(0.25, (0.125,), 5), 0.25


# k_fused_fixed (fixed grids with a built-in right-hand side) against np_ref directly: three passes of rows, the last
# one partial.  Forward on the output grid; reverse time on a step_size grid finer than the outputs (interpolated rows)
FIXED_ROWS = 600001
FIXED_METHODS = ("euler", "midpoint", "heun", "rk4")
FIXED_T = np.linspace(0.0, 0.1, 6)
FIXED_T_REV = np.array([0.1, 0.07, 0.03, 0.0])
FIXED_STEP = 0.013


def fixed_y0(problem, dtype, rows=FIXED_ROWS):
    rng = np.random.default_rng(5)
    if problem == "lorenz":
        y0 = np.array([1.0, 1.0, 1.0]) + 0.1 * rng.standard_normal((rows, 3))
    else:
        y0 = 1.0 + 0.3 * rng.random((rows, 2))
    return y0.astype(dtype)


# multistep (fixed_adams / explicit_adams) over k_lincomb / k_reduce at the Lorenz fp64 size
MULTISTEP_T = np.arange(41) * 0.0025


# --------------------------------------------------------------------------------------------------
# what the cases reach
# --------------------------------------------------------------------------------------------------
def features(sms):
    """The geometry features the case table reaches on a device of `sms` SMs, as a set of names."""
    feats = set()
    for dt, rows in LORENZ_ROWS.items():
        n = 3 * rows
        seg = build_geom([n], dt, sms).segs[0]
        if seg.passes >= 3:
            feats.add("vector_3_passes_" + dt)
        if seg.tail and seg.passes >= 2:
            feats.add("vector_tail_after_loop_" + dt)
        emit = build_geom([n], dt, sms, vector=[n % vector_width(dt) == 0]).segs[0]
        if not emit.vector and emit.passes >= 2:
            feats.add("emit_scalar_rows_loop_" + dt)
        g = row_grid(rows, sms)
        if g.passes >= 2 and g.partial:
            feats.add("stage_rhs_loop_partial_" + dt)
    lens = tuple12_lens()
    for dt in es.DTYPES:
        vec = [i != MISALIGNED for i in range(len(lens))]
        g = build_geom(lens, dt, sms, vector=vec)
        if len(lens) == 12:
            feats.add("segments_12")
        if g.cap_exceeded:
            feats.add("proportional_split_" + dt)
        one = g.segs[ONE_BLOCK]
        if one.blocks == 1 and one.passes >= 3:
            feats.add("one_block_loops_" + dt)
        mis = g.segs[MISALIGNED]
        if not mis.vector and mis.passes >= 2:
            feats.add("scalar_segment_loops_" + dt)
    g = row_grid(FIXED_ROWS, sms)
    if g.passes >= 2 and g.partial:
        feats.add("fused_fixed_loop_partial")
    for c in (NORTH_STAR, REVERSE_LINEAR):
        if build_geom([c.rows * c.dim], "float64", sms).segs[0].passes >= 3:
            feats.add("linear_3_passes_" + c.name)
    return feats


FEATURES_132 = {"vector_3_passes_float64", "vector_3_passes_float32", "vector_tail_after_loop_float64",
                "vector_tail_after_loop_float32", "emit_scalar_rows_loop_float64", "emit_scalar_rows_loop_float32",
                "stage_rhs_loop_partial_float64", "stage_rhs_loop_partial_float32", "segments_12",
                "proportional_split_float64", "proportional_split_float32", "one_block_loops_float64",
                "one_block_loops_float32", "scalar_segment_loops_float64", "scalar_segment_loops_float32",
                "fused_fixed_loop_partial", "linear_3_passes_northstar", "linear_3_passes_linear-rev"}
