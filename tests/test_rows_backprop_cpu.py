"""CPU: odeint(..., options={'independent_rows': True, 'backprop': True}) -- its refusals (raised before anything runs),
the ctypes mirrors of b2ode_rows_record_desc / b2ode_rows_bp_desc, the argument checks of b2ode_rows_solve_record and
b2ode_rows_bp (which run before any CUDA call) and b2ode_rows_bp_workspace_bytes."""
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn as nn


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


class Lin(nn.Module):
    def forward(self, t, y):
        return -y


def _go(func, y0, method="dopri5", **opts):
    t = torch.linspace(0, 1, 3, dtype=torch.float64)
    return tfd().odeint(func, y0, t, method=method, options=dict(opts, independent_rows=True, backprop=True))


def test_refusals_raise_before_anything_runs():
    rhs = tfd().rhs
    y = torch.ones(4, 3, dtype=torch.float64, requires_grad=True)     # CPU tensors: any launch would fail differently
    lz = rhs.Lorenz()
    with pytest.raises(ValueError):
        _go(Lin(), y)                                                  # not a built-in
    for method in ("tsit5", "adams", "fixed_adams", "explicit_adams"):
        with pytest.raises(ValueError):
            _go(lz, y, method=method)
    for opts in ({"fused_rhs": False}, {"fused_rhs": "stages"}, {"shared_step_group": object()}, {"cuda_graph": True},
                 {"host_output": object()}):
        with pytest.raises(ValueError):
            _go(lz, y, **opts)
    with pytest.raises(ValueError):
        tfd().odeint(lz, y, torch.linspace(0, 1, 3, dtype=torch.float64), rtol=[1e-6, 1e-6], method="dopri5",
                     options={"independent_rows": True, "backprop": True})
    with pytest.raises(ValueError):
        tfd().odeint(lz, y, torch.linspace(0, 1, 3, dtype=torch.float64, requires_grad=True), method="dopri5",
                     options={"independent_rows": True, "backprop": True})
    m = rhs.CubicMLP(8, dtype=torch.float64)
    m.b2.requires_grad_(False)
    with pytest.raises(ValueError):
        _go(m, torch.ones(4, 2, dtype=torch.float64, requires_grad=True))
    lz2 = rhs.Lorenz()
    lz2.extra = nn.Parameter(torch.ones(2, dtype=torch.float64))
    with pytest.raises(ValueError):
        _go(lz2, y)


def test_fixed_grid_drops_the_flag_before_the_solve():
    bp = tfd().backprop
    opts = {"independent_rows": True, "backprop": True, "step_size": 0.1}
    assert bp.check_options("rk4", opts, torch.zeros(2)) == {"step_size": 0.1}
    assert bp.check_options("dopri5", opts, torch.zeros(2)) == {"independent_rows": True, "step_size": 0.1}


def _header():
    here = os.path.dirname(os.path.abspath(__file__))
    return open(os.path.join(os.path.dirname(here), "include", "b2ode.h")).read()


@pytest.mark.parametrize("name,cls", [("b2ode_rows_record_desc", "RowsRecordDesc"), ("b2ode_rows_bp_desc", "RowsBpDesc")])
def test_ctypes_mirrors_follow_the_header(name, cls):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), _header(), re.S).group(1)
    fields = []
    for decl in re.sub(r"/\*.*?\*/", "", body, flags=re.S).split(";"):
        decl = decl.strip()
        if not decl:
            continue
        names = decl.split(None, 1)[1] if not decl.startswith("const") else decl.split(None, 2)[2]
        for n in re.sub(r"\[[^]]*\]", "", names).split(","):
            fields.append(re.match(r"\**\s*(\w+)", n.strip()).group(1))
    assert [f[0] for f in getattr(tfd()._lib, cls)._fields_] == fields


def _adaptive(lib, n=30, n_k=7, fsal=1):
    d = lib.AdaptiveDesc()
    d.dtype, d.nseg, d.n_k, d.fsal = lib.F64, 1, n_k, fsal
    d.seg_len[0] = n
    return d


def test_bad_descriptors_are_rejected_without_the_device():
    lib = tfd()._lib
    L = lib.lib
    d = _adaptive(lib)
    r = lib.RowsDesc()
    assert L.b2ode_rows_solve_record(C.byref(d), C.byref(r), None) == -1 and b"null record" in L.b2ode_last_error()
    rec = lib.RowsRecordDesc()
    r.y0 = r.out = r.t_out = r.n_acc = r.n_rej = r.dt_next = r.error_ratio = r.status = r.workspace = 256
    r.workspace_bytes, r.n_out = 256, 3
    r.rhs.kind, r.rhs.n_params = lib.RHS_LORENZ, 3
    d.controller = lib.CTRL_REFERENCE
    assert L.b2ode_rows_solve_record(C.byref(d), C.byref(r), C.byref(rec)) == -1 and b"capacity" in L.b2ode_last_error()
    rec.ckpt, rec.sched, rec.capacity = 256, 256, 4
    h = _adaptive(lib, n_k=2, fsal=0)
    h.controller = lib.CTRL_REFERENCE
    assert L.b2ode_rows_solve_record(C.byref(h), C.byref(r), C.byref(rec)) == -1 and b"ckpt_f0" in L.b2ode_last_error()

    b = lib.RowsBpDesc()
    assert L.b2ode_rows_bp(C.byref(d), None) == -1
    b.rhs.kind = 9
    assert L.b2ode_rows_bp(C.byref(d), C.byref(b)) == -1 and b"unknown built-in" in L.b2ode_last_error()
    b.rhs.kind, b.rhs.n_params = lib.RHS_LORENZ, 3
    assert L.b2ode_rows_bp(C.byref(_adaptive(lib, n=31)), C.byref(b)) == -1 and b"multiple" in L.b2ode_last_error()
    b.n_params = 4
    assert L.b2ode_rows_bp(C.byref(d), C.byref(b)) == -1 and b"n_params" in L.b2ode_last_error()
    b.n_params, b.n_out = 0, 1
    assert L.b2ode_rows_bp(C.byref(d), C.byref(b)) == -1 and b"n_out" in L.b2ode_last_error()
    b.n_out = 3
    assert L.b2ode_rows_bp(C.byref(d), C.byref(b)) == -1 and b"null buffer" in L.b2ode_last_error()
    b.ckpt = b.sched = b.n_acc = b.t_out = b.grad_out = b.grad_y0 = b.workspace = 256
    assert L.b2ode_rows_bp(C.byref(_adaptive(lib, n_k=2, fsal=0)), C.byref(b)) == -1 and b"ckpt_f0" in L.b2ode_last_error()
    assert L.b2ode_rows_bp(C.byref(d), C.byref(b)) == -1 and b"capacity" in L.b2ode_last_error()
    b.capacity = 5
    assert L.b2ode_rows_bp(C.byref(d), C.byref(b)) != 0 and b"workspace too small" in L.b2ode_last_error()
    b.workspace_bytes, b.workspace = 16, 8
    assert L.b2ode_rows_bp(C.byref(d), C.byref(b)) == -1 and b"aligned" in L.b2ode_last_error()
    d5 = _adaptive(lib, n_k=5)
    assert L.b2ode_rows_bp(C.byref(d5), C.byref(b)) == -1 and b"2, 4, 7 or 14" in L.b2ode_last_error()


def test_rows_bp_workspace_bytes():
    lib = tfd()._lib
    rd = lib.RhsDesc(kind=lib.RHS_CUBIC_MLP, n_params=2, data=8)
    rd.params[0], rd.params[1] = 50, 1
    P = 5 * 50 + 2
    for rows, sm in ((1, 132), (3000, 132), (10 ** 6, 132), (10 ** 6, 0)):
        grid = min(max((rows + 127) // 128, 1), (sm or 132) * 8)
        assert lib.lib.b2ode_rows_bp_workspace_bytes(C.byref(rd), rows, P, sm) == 16 + grid * P * 8
        assert lib.lib.b2ode_rows_bp_workspace_bytes(C.byref(rd), rows, 0, sm) == 16
    assert lib.lib.b2ode_rows_bp_workspace_bytes(C.byref(rd), 10, 7, 132) == 0          # not 0 or 5 H + 2
    lz = lib.RhsDesc(kind=lib.RHS_LORENZ, n_params=3)
    assert lib.lib.b2ode_rows_bp_workspace_bytes(C.byref(lz), 10, 0, 132) == 16
    assert lib.lib.b2ode_rows_bp_workspace_bytes(C.byref(lz), 0, 0, 132) == 0
    assert lib.lib.b2ode_rows_bp_workspace_bytes(C.byref(lz), 10, 252, 132) == 0


def test_initial_record_size():
    bp = tfd().backprop
    assert bp.ROWS_INITIAL_SLOTS >= 1 and bp.ROWS_INITIAL_BYTES >= 1 << 20
