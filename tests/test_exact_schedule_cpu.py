"""CPU: the premises of tests/test_exact_schedule_gpu.py, checked on the oracle for every case that file runs.

A bit-exact comparison of an adaptive solve with the oracle proves something only if (1) every step size is an exact
power-of-two multiple of the first, (2) no attempt's error ratio is close enough to 1 for a rounding difference in the
error norm to flip its decision, and (3) the solve exercises what can go wrong: a rejection, a step with more output
rows than the persistent kernel buffers, a step without output, an output time on a step end, and otherwise output
times whose x = (t - t0) / (t1 - t0) has a full mantissa.  The block shapes the batch sizes are chosen for are checked
against a restatement of the kernel's geometry at 132 SMs (H100 SXM)."""
import pytest

import exact_schedule as es

EXACT = es.PERSISTENT + es.OUTLIER + es.GENERIC + es.BULK


def _check_exact_premises(p, dtype):
    assert p["dyadic"], "a step size is not first_step * 2**-k"
    assert p["decisions_agree"], "the oracle's decisions disagree with the exactly summed error ratio"
    assert p["margin"] > es.MARGIN[dtype], p["margin"]
    assert p["attempts"] <= es.MAX_ATTEMPTS, p["attempts"]
    assert p["n_rej"] >= 1, "no rejected attempt"
    assert p["max_rows"] > es.DENSE_ROWS, "no step with more output rows than the persistent kernel buffers"
    assert p["empty_steps"] >= 1, "no accepted step without output"
    assert p["rows_on_step_end"] >= 1, "no output time on a step end"
    assert p["others_non_dyadic"], "an output time off the step ends is dyadic"


@pytest.mark.parametrize("name", [c.name for c in EXACT])
def test_exact_case_premises(name):
    case = es.ALL[name]
    _, s = es.solve_case(case)
    _check_exact_premises(es.premises(s, case.first_step), case.dtype)


@pytest.mark.parametrize("dtype", es.DTYPES)
def test_tuple_case_premises(dtype):
    y0, func, rtol, atol, t, first_step = es.tuple_case(dtype)
    s = es.oracle_solve(func, y0, t, "dopri5", rtol, atol, dict(es.OPTIONS, first_step=first_step))
    _check_exact_premises(es.premises(s, first_step), dtype)


@pytest.mark.parametrize("name", [c.name for c in es.INITIAL + es.NON_BASIC])
def test_schedule_premises_of_inexact_cases(name):
    """first_step=None (the schedule is exact relative to the oracle's own initial step) and the right-hand sides with
    pow / tanh (compared between two engine paths): the decisions must be robust, the schedule exact."""
    case = es.ALL[name]
    _, s = es.solve_case(case)
    p = es.premises(s, case.first_step)
    assert p["dyadic"] and p["decisions_agree"]
    assert p["margin"] > es.MARGIN[case.dtype], p["margin"]
    assert p["attempts"] <= es.MAX_ATTEMPTS
    if case in es.NON_BASIC:
        assert p["n_rej"] >= 1 and p["max_rows"] > es.DENSE_ROWS
    else:
        assert s.rec.dt[0] != case.t[-1] and s.stats.n_acc > 1


def test_every_case_is_exercised_on_both_sides():
    """Each tableau of the persistent kernel in both dtypes and directions on both systems; outlier rows in distinct
    trajectory warps, compute-warp slots and blocks."""
    seen = {(c.problem, c.method, c.dtype, c.reverse) for c in es.PERSISTENT if c.batch == "ncw3_partial"}
    assert len(seen) == 2 * len(es.METHODS) * 2 * 2
    g = es.fused_geometry(es.BATCHES["ncw3_partial"](es.H100_SMS), es.H100_SMS, "dopri5", "float64", 3)
    rows = es.OUTLIER_ROWS(es.H100_SMS)
    per_block = 32 * g.ncw
    places = {(r // per_block, (r % per_block) // 32) for r in rows}         # (block, trajectory warp)
    assert {(0, 0), (0, 1), (0, 2), (1, 0), (g.grid - 1, 0), (g.grid - 1, 1)} <= places
    assert rows[-1] == es.BATCHES["ncw3_partial"](es.H100_SMS) - 1
    # row 64 is trajectory warp 2 of block 0: the second slot of compute warp 0 at two trajectories per thread
    assert (64 % per_block) // 32 == g.pcw


@pytest.mark.parametrize("batch,tpt", sorted(es.BATCH_FEATURES))
def test_geometry_at_132_sms(batch, tpt):
    method = "dopri5" if tpt == 2 else "bosh3"
    n = es.BATCHES[batch](es.H100_SMS)
    g = es.fused_geometry(n, es.H100_SMS, method, "float64", 3)
    want = es.BATCH_FEATURES[batch, tpt]
    assert g.tpt == tpt and g.ncw == want["ncw"], g
    assert want["has"] <= g.features, (g.features, want["has"])
    assert not (want.get("not", set()) & g.features), g.features
    assert g.grid <= es.H100_SMS


def test_geometry_matches_the_documented_shapes():
    sms = es.H100_SMS
    assert [es.BATCHES[b](sms) for b in ("one", "ncw2_tail1", "ncw3_full", "ncw3_partial")] == [1, 4225, 12672, 12627]
    g = es.fused_geometry(4225, sms, "dopri5", "float64", 3)
    assert (g.ncw, g.grid, g.pcw, g.last_traj) == (2, 67, 1, 1)
    g = es.fused_geometry(12672, sms, "dopri5", "float32", 3)
    assert (g.ncw, g.grid, g.pcw, g.last_traj) == (3, 132, 2, 96)
    g = es.fused_geometry(12627, sms, "dopri5", "float64", 3)
    assert (g.ncw, g.grid, g.pcw, g.last_traj) == (3, 132, 2, 51)
    g = es.fused_geometry(65536, sms, "dopri5", "float64", 3)
    assert (g.ncw, g.grid, g.pcw) == (16, 128, 8)
    # one trajectory per thread: fp64 Kepler (D = 4) with the 7-k tableau, and the 2-, 4- and 14-k tableaus
    for method, dtype, dim in (("dopri5", "float64", 4), ("bosh3", "float32", 2), ("adaptive_heun", "float64", 3),
                               ("dopri8", "float32", 3)):
        assert es.fused_budget(method, dtype, dim)[1] == 1
    assert es.fused_budget("dopri5", "float32", 4)[1] == 2
    # the trajectory-warp caps: 17 (7 k's), 15 (2 and 4 k's), 7 (14 k's) alone
    for method, cap in (("dopri5", 17), ("bosh3", 15), ("adaptive_heun", 15), ("dopri8", 7)):
        assert es.fused_budget(method, "float64", 3)[0] // 32 - 1 == cap
