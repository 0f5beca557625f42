"""CPU: what the independent-rows adjoint GPU tests (tests/test_rows_adjoint_gpu.py) rely on, checked on the oracle; the
refusals of odeint_adjoint with independent_rows; the ctypes mirror of b2ode_rows_adjoint_desc; and the validation of
b2ode_rows_adjoint_solve, which must reject a bad descriptor before touching the device."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import exact_schedule as es
import rows_adjoint_cases as rac
import tfdiffeq_b200 as tfd
from tfdiffeq_b200 import _lib, tableaus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", [c.name for c in rac.CASES])
def test_pool_premises(name):
    """Every kept pool row's oracle adjoint completes under the exact schedule, with every decision of the forward solve and
    of every backward interval at least the margin away from the threshold; the pool keeps at least one scaled row besides
    the cluster and the rows take different backward schedules."""
    case = rac.ALL[name]
    pool, w, res = rac.pool_adjoints(case)
    assert len(pool) > rac.rc.CLUSTER
    for k, a in enumerate(res):
        for p in rac.premises(a, case):
            assert p["dyadic"] and p["decisions_agree"] and p["margin"] > es.MARGIN[case.dtype], (k, p)
        assert len(a.backward) == len(case.t) - 1
    attempts = {sum(s.stats.n_acc + s.stats.n_rej for s in a.backward) for a in res}
    assert len(attempts) > 1
    assert np.all(w[:, 1] == 0) and np.any(w == 0) and np.all(np.isfinite(w))


def refusal_cases(dev):
    y3 = torch.ones(4, 3, dtype=torch.float64, device=dev)
    t = torch.tensor([0.0, 0.1, 0.2], dtype=torch.float64, device=dev)
    on = {"independent_rows": True, "fused_vjp": True}
    lor = tfd.rhs.Lorenz()
    mlp_train = tfd.rhs.CubicMLP(8, dtype=torch.float64).to(dev)
    mlp_part = tfd.rhs.CubicMLP(8, dtype=torch.float64).to(dev)
    mlp_part.b2.requires_grad_(False)
    lin = tfd.rhs.LinearODE(torch.eye(3, dtype=torch.float64)).to(dev)
    m = dict(method="dopri5")
    return [("flag without fused_vjp", lor, y3, dict(m, options={"independent_rows": True})),
            ("flag in adjoint_options only", lor, y3, dict(m, adjoint_options=on)),
            ("flag in options only", lor, y3, dict(m, options=on, adjoint_options={"fused_vjp": True})),
            ("trainable CubicMLP", mlp_train, y3[:, :2], dict(m, options=on)),
            ("partially frozen CubicMLP", mlp_part, y3[:, :2], dict(m, options=on)),
            ("tuple state", lor, (y3,), dict(m, options=on)),
            ("not a built-in", lin, y3, dict(m, options=on)),
            ("tsit5", lor, y3, dict(method="tsit5", options=on)),
            ("tsit5 backward", lor, y3, dict(m, adjoint_method="tsit5", options=on)),
            ("fixed grid", lor, y3, dict(method="rk4", options=on)),
            ("multistep backward", lor, y3, dict(m, adjoint_method="adams", options=on)),
            ("per-component rtol", lor, y3, dict(m, rtol=[1e-6, 1e-7], options=on)),
            ("fused_rhs False", lor, y3, dict(m, options=dict(on, fused_rhs=False))),
            ("fused_rhs stages", lor, y3, dict(m, options=dict(on, fused_rhs="stages"))),
            ("shared_step_group", lor, y3, dict(m, options=dict(on, shared_step_group=object())))], t


def test_refusals_raise_value_error():
    cases, t = refusal_cases("cpu")
    for name, func, y0, kw in cases:
        with pytest.raises(ValueError):
            tfd.odeint_adjoint(func, y0, t, **kw)
    # a supported call passes the checks and reaches the solver, which has no CPU path
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        tfd.odeint_adjoint(tfd.rhs.Lorenz(), torch.ones(4, 3, dtype=torch.float64), t, method="dopri5",
                           options={"independent_rows": True, "fused_vjp": True})


def test_rows_adjoint_desc_mirror_matches_the_header():
    src = open(os.path.join(ROOT, "include", "b2ode.h")).read()
    body = re.search(r"typedef struct b2ode_rows_adjoint_desc \{(.*?)\} b2ode_rows_adjoint_desc;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names.append(re.findall(r"\*?\s*(\w+)\s*$", decl)[0])
    assert names == [f for f, _ in _lib.RowsAdjointDesc._fields_]
    offs = {f: getattr(_lib.RowsAdjointDesc, f).offset for f, _ in _lib.RowsAdjointDesc._fields_}
    assert offs["ans"] == C.sizeof(_lib.RhsDesc) and C.sizeof(_lib.RowsAdjointDesc) % 8 == 0


BUF = [C.c_void_p(0x10000 * (i + 1)) for i in range(24)]     # never dereferenced: validation runs first


def _desc(lens, tab=tableaus.DOPRI5, dtype=_lib.F64):
    d = _lib.AdaptiveDesc()
    d.dtype, d.nseg, d.n_k, d.fsal, d.sm_count = dtype, len(lens), tab.n_k, 1 if tab.fsal else 0, 132
    for i, n in enumerate(lens):
        d.seg_len[i] = n
    d.dense_kind = 0 if tab.c_mid is not None else 1
    d.controller = _lib.CTRL_TSIT5 if tab.controller == "tsit5" else _lib.CTRL_REFERENCE
    return d


def _rd(kind=_lib.RHS_LORENZ, params=(10.0, 8.0 / 3.0, 28.0), data=None, n_out=3, ws=1 << 20, ws_ptr=None):
    r = _lib.RowsAdjointDesc()
    r.rhs.kind, r.rhs.n_params = kind, len(params)
    for i, v in enumerate(params):
        r.rhs.params[i] = v
    r.rhs.data, r.rhs.time_sign = data, -1.0
    for i, f in enumerate(("ans", "grad_out", "t_out", "grad_y0", "t_grad", "n_acc", "n_rej", "dt_next", "error_ratio",
                           "status")):
        setattr(r, f, BUF[i].value)
    r.n_out, r.first_step = n_out, 0.25
    r.workspace = BUF[12].value if ws_ptr is None else ws_ptr
    r.workspace_bytes = ws
    return r


def test_workspace_bytes():
    lib = _lib.lib
    assert lib.b2ode_rows_adjoint_workspace_bytes(4099, 11, 132) == 16 + 8 * 4099 + 8 * 17 * 11
    assert lib.b2ode_rows_adjoint_workspace_bytes(10 ** 6, 1000, 132) == 16 + 8 * 10 ** 6 + 8 * 264 * 1000
    assert lib.b2ode_rows_adjoint_workspace_bytes(0, 11, 132) == 0 and lib.b2ode_rows_adjoint_workspace_bytes(5, 0, 132) == 0


def test_solve_rejects_bad_descriptors_before_the_device():
    lib = _lib.lib
    ok = (12, 12, 1, 1)
    need = lib.b2ode_rows_adjoint_workspace_bytes(4, 3, 132)
    cases = [
        (_desc(ok), _rd(kind=9), b"unknown built-in right-hand side 9"),
        (_desc((12, 12, 1)), _rd(), b"4 segments"),
        (_desc((10, 10, 1, 1)), _rd(), b"not a multiple of the row size 3"),
        (_desc((8, 8, 1, 252)), _rd(_lib.RHS_CUBIC_MLP, (50.0, 1.0), data=BUF[20].value), b"frozen weights only"),
        (_desc((8, 8, 1, 1)), _rd(_lib.RHS_CUBIC_MLP, (50.0, 1.0), data=None), b"cubic-MLP"),
        (_desc(ok, tab=tableaus.TSIT5), _rd(), b"quartic dense output"),
        (_desc(ok, dtype=7), _rd(), b"dtype"),
        (_desc(ok), _rd(n_out=1), b"n_out must be at least 2"),
        (_desc(ok), _rd(ws=need - 1), b"workspace too small"),
        (_desc(ok), _rd(ws_ptr=BUF[12].value + 8), b"16-byte aligned"),
    ]
    for d, r, text in cases:
        before = lib.b2ode_launch_count()
        rc = lib.b2ode_rows_adjoint_solve(C.byref(d), C.byref(r))
        assert rc in (-1, -3), (text, rc)
        assert text in lib.b2ode_last_error(), (text, lib.b2ode_last_error())
        assert lib.b2ode_launch_count() == before
    r = _rd()
    r.grad_y0 = None
    assert lib.b2ode_rows_adjoint_solve(C.byref(_desc(ok)), C.byref(r)) == -1
    assert b"null buffer" in lib.b2ode_last_error()
    d = _desc(ok)
    d.n_k = 5
    assert lib.b2ode_rows_adjoint_solve(C.byref(d), C.byref(_rd())) == -1
    assert b"2, 4, 7 or 14 k's (got 5)" in lib.b2ode_last_error()
