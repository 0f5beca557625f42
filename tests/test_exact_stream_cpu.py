"""CPU: the premises of tests/test_exact_stream_gpu.py, checked on the oracle at every case's real size, and the launch
geometry the cases are sized for, checked at 132 SMs (H100 SXM).

The adaptive cases must meet tests/exact_schedule.py's exact-schedule premises (dyadic step sizes, decisions robust to a
rounding difference in the error norm, a rejection, a step without output, an output on a step end).  The north-star
cases additionally rest on ExactLinear's matrix: at most two non-zero entries per column, each a signed power of two,
which makes ``y @ A`` exact in any summation order."""
import numpy as np
import pytest

import exact_schedule as es
import exact_stream as xs
from problems import PROBLEMS


def _check_schedule(s, first_step, dtype, rows_per_step=True):
    p = es.premises(s, first_step)
    assert p["dyadic"], "a step size is not first_step * 2**-k"
    assert p["decisions_agree"], "the oracle's decisions disagree with the exactly summed error ratio"
    assert p["margin"] > es.MARGIN[dtype], p["margin"]
    assert p["attempts"] <= es.MAX_ATTEMPTS, p["attempts"]
    assert p["n_rej"] >= 1, "no rejected attempt"
    assert p["empty_steps"] >= 1, "no accepted step without output"
    assert p["rows_on_step_end"] >= 1, "no output time on a step end"
    assert p["others_non_dyadic"], "an output time off the step ends is dyadic"
    if rows_per_step:
        assert p["max_rows"] > es.DENSE_ROWS, "no step with several output rows"
    return p


@pytest.mark.parametrize("name", [c.name for c in xs.LORENZ])
def test_lorenz_case_premises(name):
    case = xs.ALL[name]
    _, s = es.solve_case(case)
    _check_schedule(s, case.first_step, case.dtype)


def test_initial_step_case_premises():
    case = xs.INITIAL[0]
    _, s = es.solve_case(case)
    p = es.premises(s, case.first_step)
    assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[case.dtype], p
    assert s.rec.dt[0] != case.t[-1] and s.stats.n_acc > 1


@pytest.mark.parametrize("case", [xs.NORTH_STAR, xs.REVERSE_LINEAR], ids=lambda c: c.name)
def test_linear_case_premises(case):
    """The north star at its full 65 536 x 128 (about 20 s) and the smaller reverse-time state."""
    _, s = xs.solve_linear(case)
    _check_schedule(s, case.first_step, "float64")
    # the premise of ExactLinear holds for the solution's magnitudes: no product can underflow
    assert np.abs(s.sol).max() < 1e3 and np.min(np.abs(s.sol[s.sol != 0])) > 1e-290


@pytest.mark.parametrize("dtype", es.DTYPES)
def test_tuple12_case_premises(dtype):
    y0, func, rtol, atol, t, first_step = xs.tuple12_case(dtype)
    assert len(y0) == 12 and len(set(rtol)) > 1 and len(set(atol)) > 1
    s = es.oracle_solve(func, y0, t, "dopri5", rtol, atol, dict(es.OPTIONS, first_step=first_step))
    _check_schedule(s, first_step, dtype)


@pytest.mark.parametrize("case", [xs.NORTH_STAR, xs.REVERSE_LINEAR], ids=lambda c: c.name)
def test_exact_linear_matrix_has_two_power_of_two_entries_per_column(case):
    A = xs.linear_problem(case).A_np
    D = case.dim
    assert A.shape == (D, D)
    for j in range(D):
        nz = A[:, j][A[:, j] != 0]
        assert 1 <= nz.size <= 2
        m, e = np.frexp(np.abs(nz))
        assert np.all(m == 0.5), nz                         # every entry +- a power of two
    assert np.all(np.diag(A) == -0.5)
    off = A - np.diag(np.diag(A))
    assert np.all(np.count_nonzero(off, axis=0) == 1)      # a permutation without fixed points: a rotation, not diagonal
    assert np.all(np.count_nonzero(off, axis=1) == 1)
    assert set(np.abs(off[off != 0])) == {1.0 / 16} and (off > 0).any() and (off < 0).any()


@pytest.mark.parametrize("case", [xs.NORTH_STAR, xs.REVERSE_LINEAR], ids=lambda c: c.name)
def test_exact_linear_gather_form_equals_the_matrix_product(case):
    """numpy's ``y @ A`` (BLAS, any order) equals the two-term gather form the oracle uses, bit for bit."""
    f = xs.linear_problem(case)
    y = xs.linear_y0(case)[:257]
    assert np.array_equal(y @ f.A_np, f(0.0, y))
    # also on full-mantissa values after a few exact-schedule-like updates
    z = y + 0.123456789 * f(0.0, y)
    assert np.array_equal(z @ f.A_np, f(0.0, z))
    assert np.array_equal(-(z @ f.A_np), z @ (-f.A_np))     # the reverse-time image: negation is exact


def test_geometry_features_at_132_sms():
    """Which loops of the kernels the case table runs, from a restatement of their launch geometry."""
    feats = xs.features(xs.H100_SMS)
    assert xs.FEATURES_132 <= feats, sorted(xs.FEATURES_132 - feats)


def test_geometry_matches_the_documented_shapes():
    sms = xs.H100_SMS
    # fp64 Lorenz: 1 800 003 elements, 900 001 packs over 1 056 x 256 threads, one element left for block 0
    seg = xs.build_geom([1800003], "float64", sms).segs[0]
    assert (seg.blocks, seg.vector, seg.passes, seg.tail) == (1056, True, 4, 1)
    seg = xs.build_geom([2250003], "float32", sms).segs[0]
    assert (seg.blocks, seg.vector, seg.passes, seg.tail) == (1056, True, 3, 3)
    # the dense output of an odd-length segment is scalar: 7 passes
    assert xs.build_geom([1800003], "float64", sms, vector=[False]).segs[0].passes == 7
    # one pass of the grid: 540 672 fp64 / 1 081 344 fp32 elements, 270 336 rows
    assert xs.build_geom([540672], "float64", sms).segs[0].passes == 1
    assert xs.build_geom([540673], "float64", sms).segs[0][3:] == (1, 1)     # one pass and block 0's tail element
    assert xs.build_geom([540674], "float64", sms).segs[0][3:] == (2, 0)     # one more pack: a second pass
    assert xs.build_geom([1081344], "float32", sms).segs[0].passes == 1
    assert xs.row_grid(270336, sms) == (1056, 1, False)
    assert xs.row_grid(270337, sms) == (1056, 2, True)
    assert xs.row_grid(xs.FIXED_ROWS, sms) == (1056, 3, True)
    assert xs.row_grid(1, sms) == (1, 1, True)
    # below the cap every segment gets what it needs; above it the proportional split, at least one block each
    g = xs.build_geom([1000, 3, 512 * 256], "float64", sms)
    assert not g.cap_exceeded and [p.blocks for p in g.segs] == [2, 1, 256]
    g = xs.build_geom(xs.tuple12_lens(), "float64", sms, vector=[i != xs.MISALIGNED for i in range(12)])
    assert g.cap_exceeded and g.grid <= 8 * sms
    assert g.segs[xs.ONE_BLOCK] == (4500, 1, True, 9, 0)
    assert g.segs[xs.MISALIGNED].vector is False and g.segs[xs.MISALIGNED].passes == 12
    assert g.segs[0] == (3, 1, True, 1, 1)
    g = xs.build_geom(xs.tuple12_lens(), "float32", sms)
    assert g.segs[0] == (3, 1, True, 0, 3)                  # no pack at all: block 0's tail only
    assert g.segs[xs.ONE_BLOCK] == (4500, 1, True, 5, 0)


def test_geometry_scales_with_the_sm_count():
    """The features do not hinge on the exact H100 SXM count: a 114-SM H100 PCIe reaches them too."""
    assert xs.FEATURES_132 <= xs.features(114)
