"""CPU: the oracle of tests/test_exact_adjoint_gpu.py against the unmodified reference adjoint's golden gradients, and
the premises of the exact comparison, checked on the oracle for every case the GPU file runs.

The exact comparison proves something only if every forward and backward solve keeps the exact schedule with robust
decisions (tests/exact_schedule.py), the products are exact (ExactLinear's A and A^T, power-of-two loss weights) and
the large cases reach the launch geometry they are sized for: several vector passes of every large segment while the
1-element ``adj_t`` segment sits in build_geom's proportional split, and all 12 segments for the 5-tensor state."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import exact_adjoint as xa
import exact_schedule as es
import exact_stream as xs
from grad_cases import GRAD_CASES, build_params, rhs_torch
from problems import PROBLEMS

# agreement of the oracle with the reference adjoint's fixtures, relative to max(1, max |reference|).  The fixtures were
# made with the reference's own arithmetic (TF ops over the torch shim, func's outputs stacked); all but t.grad and the
# two-component case agree exactly.  fp32 also differs in the dtype of adj_t
GOLDEN_BAR = {"float64": 1e-13, "float32": 1e-7}


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(1.0, float(np.max(np.abs(b)))))


class _GradCaseModule(nn.Module):
    def __init__(self, case, params):
        super(_GradCaseModule, self).__init__()
        self.case = case
        self.ps = nn.ParameterDict({n: nn.Parameter(params[n].detach().clone()) for n in sorted(params)})

    def forward(self, t, y):
        return rhs_torch(self.case, self.ps, t, y)


def golden_agreement(name, golden_dir, time_dtype=None):
    """The largest relative difference of the oracle from a golden gradient fixture, per quantity."""
    case = GRAD_CASES[name]
    g = np.load(os.path.join(golden_dir, "grad_" + name + ".npz"))
    tdt = {"float32": torch.float32, "float64": torch.float64}[case["dtype"]]
    m = _GradCaseModule(case, build_params(case, tdt))
    y0 = tuple(np.asarray(v, dtype=case["dtype"]) for v in case["y0"])
    w = tuple(np.asarray(v, dtype=case["dtype"]) for v in case["w"])
    res = xa.adjoint_oracle(m, y0, case["t"], w, case["method"], case["rtol"], case["atol"], case["options"] or {},
                            tensor_input=len(y0) == 1, time_dtype=time_dtype)
    out = {"sol0": _rel(res.sol[0], g["sol0"]), "t": _rel(res.g_t, g["g_t"])}
    for i, v in enumerate(res.g_y0):
        out["y0_%d" % i] = _rel(v, g["g_y0_%d" % i])
    for n, v in zip(m.ps.keys(), res.g_params):
        out["param_" + n] = _rel(v, g["g_param_" + n])
    return out


@pytest.mark.parametrize("name", sorted(GRAD_CASES))
def test_oracle_reproduces_the_reference_adjoint(name, golden_dir):
    """All 7 fixtures of the unmodified reference adjoint: the solution and the gradients w.r.t. y0, t and every
    parameter."""
    agree = golden_agreement(name, golden_dir)
    bar = GOLDEN_BAR[GRAD_CASES[name]["dtype"]]
    assert max(agree.values()) <= bar, agree


def test_time_adjoint_dtype_is_rounding_only(golden_dir):
    """The reference keeps adj_t in t's dtype (float64, adjoint.py:116), the engine in the state dtype.  In the fp32
    fixture both choices give the reference's solution, y0 and parameter gradients bit for bit and its t.grad to fp32
    rounding."""
    engine = golden_agreement("mlp_tanh_f32", golden_dir)
    ref = golden_agreement("mlp_tanh_f32", golden_dir, time_dtype="float64")
    for agree in (engine, ref):
        assert agree["t"] <= GOLDEN_BAR["float32"], agree
        assert all(v == 0.0 for k, v in agree.items() if k != "t"), agree


# --------------------------------------------------------------------------------------------------
# the premises, per case and per backward interval
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(xa.ALL))
def test_case_premises(name):
    case = xa.ALL[name]
    module, y0, w, res = xa.solve_case(case)
    assert len(res.backward) == len(case.t) - 1
    ps = xa.schedule_premises(res, case)
    if case.method in xa.ADAPTIVE:
        assert len(ps) == len(case.t)                      # the forward solve and every backward interval
        for p in ps:
            assert p["dyadic"], "a step size is not first_step * 2**-k"
            assert p["decisions_agree"], "the oracle's decisions disagree with the exactly summed error ratio"
            assert p["margin"] > es.MARGIN[case.dtype], p["margin"]
            assert p["attempts"] <= xa.MAX_NUM_STEPS, p["attempts"]
        assert sum(p["n_rej"] for p in ps) >= 1, "no rejected attempt"
    # every gradient is finite and the loss reaches it
    for g in res.g_y0 + tuple(res.g_params):
        assert np.all(np.isfinite(g)) and np.any(g != 0)
    assert np.all(np.isfinite(res.g_t))


def test_case_table_covers_the_issue():
    """Methods, dtypes and directions the table runs."""
    small = {(c.method, c.dtype, c.reverse, c.kind) for c in xa.SMALL}
    for me in ("dopri5", "bosh3", "adaptive_heun", "dopri8"):
        for dt in es.DTYPES:
            for rev in (False, True):
                assert {(me, dt, rev, "lorenz"), (me, dt, rev, "lorenz_forced")} <= small
    assert {("tsit5", dt, False, k) for dt in es.DTYPES for k in ("lorenz", "lorenz_forced")} <= small
    assert {c.method for c in xa.FIXED} == {"euler", "midpoint", "rk4", "fixed_adams"}
    assert all(c.step_size for c in xa.FIXED if c.method != "fixed_adams")
    assert all(c.adjoint_method not in (None, c.method) for c in xa.MIXED)
    assert {xs.LORENZ_ROWS[c.dtype] for c in xa.LARGE} == {c.rows for c in xa.LARGE} == {600001, 750001}
    paths = {c.path for c in xa.ALL.values()}
    assert {"fused_rhs", "stage_rhs", "stage_func"} <= paths


# --------------------------------------------------------------------------------------------------
# exact products
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c.name for c in xa.LINEAR])
def test_linear_transpose_has_two_power_of_two_entries_per_column(name):
    case = xa.ALL[name]
    A = PROBLEMS["exact_linear"](dim=xa.linear_dim(case), seed=case.seed).A_np
    At = A.T
    for j in range(At.shape[1]):
        nz = At[:, j][At[:, j] != 0]
        assert nz.size == 2
        assert np.all(np.frexp(np.abs(nz))[0] == 0.5), nz


@pytest.mark.parametrize("name", [c.name for c in xa.LINEAR])
def test_linear_products_equal_the_gather_form(name):
    """y @ A and the VJP's a @ A^T in numpy (BLAS, any order) and torch-CPU equal the two-term gather forms bit for bit."""
    case = xa.ALL[name]
    f = PROBLEMS["exact_linear"](dim=xa.linear_dim(case), seed=case.seed)
    y = xa.initial_state(case)[0][:513]
    z = y + 0.123456789 * f(0.0, y)
    for v in (y, z):
        assert np.array_equal(v @ f.A_np, f(0.0, v))
        assert np.array_equal((torch.from_numpy(v) @ torch.from_numpy(f.A_np)).numpy(), f(0.0, v))
        # a @ A^T: column k of A^T is row k of A, i.e. d on the diagonal and sgn[j] at the column j with src[j] == k
        dst = np.empty_like(f.src)
        dst[f.src] = np.arange(f.dim)
        gather = v * f.d + v[:, dst] * f.sgn[dst]
        assert np.array_equal(v @ f.A_np.T, gather)
        assert np.array_equal((torch.from_numpy(v) @ torch.from_numpy(f.A_np).T).numpy(), gather)


@pytest.mark.parametrize("name", list(xa.ALL))
def test_loss_weights_are_powers_of_two(name):
    case = xa.ALL[name]
    y0 = xa.initial_state(case)
    w = xa.loss_weights(case, y0)
    for i, (wi, y) in enumerate(zip(w, y0)):
        if xa.UNTOUCHED.get(case.kind) == i:
            assert wi is None
            continue
        assert wi.dtype == y.dtype and wi.shape == (len(case.t),) + y.shape
        nz = wi[wi != 0]
        assert np.all(np.frexp(np.abs(nz))[0] == 0.5)
        assert not np.any(wi[1]) and np.any(wi[-1]) and 0 < (wi == 0).mean() < 0.5
    assert (xa.UNTOUCHED.get(case.kind) is not None) == (case.kind == "tuple5")


# --------------------------------------------------------------------------------------------------
# launch geometry of the backward solves
# --------------------------------------------------------------------------------------------------
def _aug_geom(case, sms):
    module, y0 = xa.make_module(case), xa.initial_state(case)
    lens = xa.augmented_lens(case, module, y0)
    return lens, xs.build_geom(lens, case.dtype, sms)


@pytest.mark.parametrize("sms", [132, 114])
def test_backward_geometry(sms):
    """The large cases: every large segment of the augmented state loops at least 3 vector passes while adj_t, one
    element, keeps its block in the proportional split.  The 5-tensor state: 12 segments."""
    for case in xa.LARGE:
        lens, g = _aug_geom(case, sms)
        assert len(lens) == 4 and lens[2] == 1 and g.cap_exceeded, lens
        assert all(s.passes >= 3 for s in g.segs if s.n > 1), g
        assert g.segs[2].blocks == 1 and g.segs[2].tail == 1
    for case in xa.TUPLE:
        lens, g = _aug_geom(case, sms)
        assert len(lens) == 12 and min(lens) == 1
        assert len({n for n in lens[:5]}) == 3                   # (n, 3), (m, 2) and a single element
    # the north star's augmented state is two 8.4M-element segments: 15 vector passes each
    lens, g = _aug_geom(xa.ALL["northstar-frozen"], sms)
    assert g.cap_exceeded and all(s.passes >= 3 for s in g.segs if s.n > 1)


def test_adjoint_rejects_more_than_five_tensors():
    """2n + 2 augmented components must fit the engine's 12 segments: a sixth tensor is refused before any solve."""
    import tfdiffeq_b200

    class Six(nn.Module):
        def forward(self, t, y):
            raise AssertionError("the forward solve must not start")
    y0 = tuple(torch.ones(2, dtype=torch.float64) for _ in range(6))
    with pytest.raises(ValueError, match="at most 5"):
        tfdiffeq_b200.odeint_adjoint(Six(), y0, torch.tensor([0.0, 1.0]), method="dopri5")
