"""GPU: the generic path bit for bit against the oracle at sizes where its kernels loop over their grid
(tests/exact_stream.py): several passes of seg_for_each on the vector and the scalar path with block 0's scalar tail,
build_geom's proportional split over 12 components, the row loops of k_rk_stage_rhs and k_fused_fixed, and the
north-star solve at its full 65 536 x 128.

Every adaptive comparison is exact under tests/exact_schedule.py's step schedule: equal solution, equal counts, equal
final step size and an error ratio that matches the oracle's exactly summed one.  Each oracle is computed once and shared
by the arms that follow it.  tests/test_exact_stream_cpu.py checks the premises and the geometry at 132 SMs; the
geometry is re-checked here at the device's SM count."""
import warnings

import numpy as np
import pytest
import torch

import exact_schedule as es
import exact_stream as xs
import np_ref
from golden_util import max_rel_err
from problems import PROBLEMS
from test_exact_schedule_gpu import _assert_exact, _check_premises

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


_ORACLE = {}


def _oracle(key, compute):
    """One oracle solve per case, shared by its arms (the arms of a case run consecutively)."""
    if key not in _ORACLE:
        _ORACLE.clear()            # keep host memory flat: the north-star solution alone is 0.9 GB
        _ORACLE[key] = compute()
    return _ORACLE[key]


def _solve(func, y0, t, method, rtol, atol, first_step, **opts):
    y = tuple(torch.tensor(a, device=DEV) for a in y0) if isinstance(y0, tuple) else torch.tensor(y0, device=DEV)
    # ifactor=1 never grows dt again: a wrong kernel that drives dt down would crawl for hours; every case takes at most
    # es.MAX_ATTEMPTS attempts in all (tests/test_exact_stream_cpu.py), so this bound only stops such a run
    options = dict(es.OPTIONS, max_num_steps=4 * es.MAX_ATTEMPTS, **opts)
    if first_step is not None:
        options["first_step"] = first_step
    sol = tfd().odeint(func, y, torch.tensor(t), rtol=rtol, atol=atol, method=method, options=options)
    st = dict(tfd().last_stats)
    got = tuple(s.cpu().numpy() for s in sol) if isinstance(sol, tuple) else sol.cpu().numpy()
    del sol, y
    return got, st


def test_geometry_at_the_device_sm_count():
    assert xs.FEATURES_132 <= xs.features(_sms()), sorted(xs.FEATURES_132 - xs.features(_sms()))


# --------------------------------------------------------------------------------------------------
# the north star: ExactLinear at 65 536 x 128 fp64, dopri5
# --------------------------------------------------------------------------------------------------
def _linear_arm(case, arm):
    """(func, options, expected stage_func) of an arm."""
    if arm.startswith("func"):
        return xs.linear_problem(case, "torch", DEV), dict(cuda_graph=arm == "func_graph"), False
    f = tfd().rhs.LinearODE(xs.linear_problem(case).A_np).to(DEV)
    if arm == "linear_unfused":
        return f, dict(fused_rhs=False), False
    return f, dict(cuda_graph=arm == "linear_graph"), True


@pytest.mark.parametrize("case,arm", [(c, a) for c in (xs.NORTH_STAR, xs.REVERSE_LINEAR)
                                      for a in ("func", "func_graph", "linear_fused", "linear_unfused", "linear_graph")
                                      if c is xs.NORTH_STAR or a in ("func", "linear_fused", "linear_unfused")],
                         ids=lambda v: v.name if isinstance(v, xs.LinearCase) else v)
def test_linear_system_at_size_is_bit_exact(case, arm):
    """The external ``y @ A`` func (cuBLAS) eagerly and replayed from a CUDA graph, and rhs.LinearODE on the fp64 tensor
    cores with the stage combine fused into its producer, unfused, and replayed; reverse time uses the -A image."""
    seg = xs.build_geom([case.rows * case.dim], "float64", _sms()).segs[0]
    assert seg.passes >= 3
    y0, s = _oracle(case.name, lambda: xs.solve_linear(case))
    p = es.premises(s, case.first_step)
    assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN["float64"], p
    func, opts, stage_func = _linear_arm(case, arm)
    got, st = _solve(func, y0, case.t, "dopri5", case.rtol, case.atol, case.first_step, **opts)
    assert not st["fused_rhs"] and st["stage_func"] == stage_func, st
    assert st["cuda_graph"] == arm.endswith("graph"), st
    _assert_exact(got, st, s, "float64")


# --------------------------------------------------------------------------------------------------
# Lorenz on the generic path: torch func, and the built-in right-hand side above the persistent kernel's capacity
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,arm", [(c.name, a) for c in xs.LORENZ for a in ("func", "builtin")])
def test_lorenz_at_size_is_bit_exact(name, arm):
    """func: the stage, finalize and dense-output kernels over 3-4 vector passes plus block 0's tail (the dense output of
    the odd-length state on the scalar path); builtin: k_rk_stage_rhs over 3 passes of rows, the last one partial, after
    the persistent kernel declined the batch with a RuntimeWarning (tsit5 has no persistent kernel)."""
    case = xs.ALL[name]
    rows = xs.LORENZ_ROWS[case.dtype]
    assert xs.build_geom([3 * rows], case.dtype, _sms()).segs[0].passes >= 3
    y0, s = _oracle(name, lambda: es.solve_case(case))
    _check_premises(s, case)
    run = lambda f: _solve(f, y0, case.t, case.method, case.rtol, case.atol, case.first_step)   # noqa: E731
    if arm == "func":
        got, st = run(PROBLEMS["lorenz"](backend="torch", device=DEV))
        assert not st["stage_rhs"]
    else:
        g = xs.row_grid(rows, _sms())
        assert g.passes >= 3 and g.partial
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            got, st = run(tfd().rhs.Lorenz())
        declined = [x for x in w if issubclass(x.category, RuntimeWarning) and "co-resident" in str(x.message)]
        assert len(declined) == (1 if case.method == "dopri5" else 0), [str(x.message) for x in w]
        assert st["stage_rhs"]
    assert not st["fused_rhs"]
    _assert_exact(got, st, s, case.dtype)


def test_initial_step_at_size_matches_oracle():
    """first_step=None: k_init_*'s reductions loop over the grid; dt_next = h0 * 2**-n_rej pins the initial step."""
    case = xs.INITIAL[0]
    y0, s = _oracle(case.name, lambda: es.solve_case(case))
    p = es.premises(s, case.first_step)
    assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[case.dtype], p
    assert s.dt_next == s.rec.dt[0] * 2.0 ** -s.stats.n_rej
    got, st = _solve(PROBLEMS["lorenz"](backend="torch", device=DEV), y0, case.t, case.method, case.rtol, case.atol, None)
    assert not st["fused_rhs"] and not st["stage_rhs"]
    assert (st["n_accepted"], st["n_rejected"], st["nfe"]) == (s.stats.n_acc, s.stats.n_rej, s.stats.nfe)
    assert abs(st["dt_next"] - s.dt_next) <= 1e-12 * s.dt_next
    assert max_rel_err(got, s.sol) <= 1e-6


# --------------------------------------------------------------------------------------------------
# 12 components over the proportional split
# --------------------------------------------------------------------------------------------------
def _odd_view(x):
    """x's values returned as a view at an odd element offset of a larger buffer: contiguous, not 16-byte aligned."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    buf[1:].copy_(x.reshape(-1))
    return buf[1:].view(x.shape)


@pytest.mark.parametrize("dtype", es.DTYPES)
def test_twelve_component_state_is_bit_exact(dtype):
    """All B2ODE_MAXSEG components with their own tolerances: segments that share the capped grid in proportion, one
    of a single row, one that gets a single block for several passes, and one whose func output is misaligned, so every
    kernel that reads func's outputs takes the scalar path over it, several passes."""
    sms = _sms()
    lens = xs.tuple12_lens()
    g = xs.build_geom(lens, dtype, sms, vector=[i != xs.MISALIGNED for i in range(12)])
    assert g.cap_exceeded and g.segs[xs.ONE_BLOCK].blocks == 1 and g.segs[xs.ONE_BLOCK].passes >= 3
    assert g.segs[xs.MISALIGNED].passes >= 2
    y0, func_np, rtol, atol, t, first_step = xs.tuple12_case(dtype)
    s = es.oracle_solve(func_np, y0, t, "dopri5", rtol, atol, dict(es.OPTIONS, first_step=first_step))
    p = es.premises(s, first_step)
    assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[dtype], p
    fs = {pr: PROBLEMS[pr](backend="torch", device=DEV) for pr in ("lorenz", "lv")}

    def func(tt, y):
        out = [fs[pr](tt, c) for (pr, _), c in zip(xs.TUPLE12, y)]
        out[xs.MISALIGNED] = _odd_view(out[xs.MISALIGNED])
        assert out[xs.MISALIGNED].data_ptr() % 16
        return tuple(out)
    got, st = _solve(func, y0, t, "dopri5", rtol, atol, first_step)
    _assert_exact(got, st, s, dtype)


# --------------------------------------------------------------------------------------------------
# k_fused_fixed: fixed grids with a built-in right-hand side, three passes of trajectories
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", es.DTYPES)
@pytest.mark.parametrize("method", xs.FIXED_METHODS)
@pytest.mark.parametrize("problem", ["lorenz", "lv"])
def test_fused_fixed_grid_at_size_is_bit_exact(problem, method, dtype):
    """Forward on the output grid, and reverse time on a step_size grid whose cells hold interpolated output rows."""
    g = xs.row_grid(xs.FIXED_ROWS, _sms())
    assert g.passes >= 3 and g.partial
    y0 = xs.fixed_y0(problem, dtype)
    f_np = PROBLEMS[problem](backend="numpy")
    f = tfd().rhs.Lorenz() if problem == "lorenz" else tfd().rhs.LotkaVolterra()
    for t, opts in ((xs.FIXED_T, {}), (xs.FIXED_T_REV, dict(step_size=xs.FIXED_STEP))):
        want = np_ref.odeint(f_np, y0, t, method=method, options=dict(opts))
        got = tfd().odeint(f, torch.tensor(y0, device=DEV), torch.tensor(t), method=method, options=dict(opts))
        assert tfd().last_stats["fused_rhs"]
        got = got.cpu().numpy()
        assert got.dtype == want.dtype and got.shape == want.shape
        bad = got != want
        assert not bad.any(), "%d of %d values differ (first at %s)" % (int(bad.sum()), bad.size, np.argwhere(bad)[0])
