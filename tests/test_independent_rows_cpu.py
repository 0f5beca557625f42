"""CPU: what the independent-rows GPU tests (tests/test_independent_rows_gpu.py) rely on, checked on the oracle, and the
ctypes mirror of b2ode_rows_desc against the C header.

For every case the GPU file compares bit for bit, each pool row's solve alone must have a dyadic schedule and robust accept
decisions (|m - 1| > MARGIN on every attempt), and the pool must give rows different schedules: at least three distinct
(accepted, rejected) pairs, one row without a rejection and one with at least two, a step with more than one output row and
a step with none."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import exact_schedule as es
import rows_cases as rc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.mark.parametrize("name", list(rc.ALL))
def test_pool_premises(name):
    case = rc.ALL[name]
    pool, solves = rc.pool_solves(case)
    assert len(pool) >= rc.CLUSTER + 2, "too few pool rows complete in the oracle"
    ps = [es.premises(s, case.first_step) for s in solves]
    for i, p in enumerate(ps):
        assert p["dyadic"] and p["decisions_agree"], (i, p)
        assert p["margin"] > es.MARGIN[case.dtype], (i, p)
    pairs = {(s.stats.n_acc, s.stats.n_rej) for s in solves}
    assert len(pairs) >= 3, pairs
    if case.first_step is not None:
        assert min(r for _, r in pairs) == 0 and max(r for _, r in pairs) >= 2, pairs
    assert max(p["max_rows"] for p in ps) > 1
    assert max(p["empty_steps"] for p in ps) >= 1


def test_pool_tiling_uses_every_entry():
    for n_pool in (10, 18):
        idx = rc.tile(n_pool, 4099)
        assert set(idx.tolist()) == set(range(n_pool))
        assert (rc.tile(n_pool, 31) == rc.tile(n_pool, 31)).all()


_OFFSETS_SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "b2ode.h"
#define F(f) printf("%s %zu\n", #f, offsetof(b2ode_rows_desc, f));
int main(void) {
    F(rhs) F(y0) F(out) F(t_out) F(n_out) F(t_start) F(first_step) F(n_acc) F(n_rej) F(dt_next) F(error_ratio) F(status)
    F(workspace) F(workspace_bytes) F(cuda_stream)
    printf("sizeof %zu\n", sizeof(b2ode_rows_desc));
    return 0;
}
"""


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_rows_desc_mirror_matches_the_header(tmp_path):
    from tfdiffeq_b200 import _lib
    src = tmp_path / "rows_offsets.cu"
    src.write_text(_OFFSETS_SRC)
    exe = str(tmp_path / "rows_offsets")
    subprocess.run([NVCC, "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src)], check=True, timeout=300)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60, check=True).stdout
    want = dict((k, int(v)) for k, v in (line.split() for line in out.splitlines()))
    got = {name: getattr(_lib.RowsDesc, name).offset for name, _ in _lib.RowsDesc._fields_}
    got["sizeof"] = C.sizeof(_lib.RowsDesc)
    assert got == want


def test_rows_solve_validates_before_touching_the_device():
    """b2ode_rows_solve rejects bad descriptions with B2ODE_EINVAL before any CUDA call (the buffer addresses below are never
    dereferenced)."""
    from tfdiffeq_b200 import _lib, tableaus
    lib = _lib.lib
    buf = [C.c_void_p(0x1000 * (i + 1)) for i in range(10)]

    def desc(tab=tableaus.DOPRI5, n=12, nseg=1):
        d = _lib.AdaptiveDesc()
        d.dtype, d.nseg, d.n_k, d.fsal = _lib.F64, nseg, tab.n_k, 1
        d.seg_len[0] = n
        d.dense_kind = 0 if tab.c_mid is not None else 1
        d.controller = _lib.CTRL_TSIT5 if tab.controller == "tsit5" else _lib.CTRL_REFERENCE
        return d

    def rows(**kw):
        r = _lib.RowsDesc(rhs=_lib.RhsDesc(kind=_lib.RHS_LORENZ, n_params=3, time_sign=1.0), y0=buf[0], out=buf[1],
                          t_out=buf[2], n_out=2, n_acc=buf[3], n_rej=buf[4], dt_next=buf[5], error_ratio=buf[6],
                          status=buf[7], workspace=buf[8], workspace_bytes=lib.b2ode_rows_workspace_bytes())
        for k, v in kw.items():
            setattr(r, k, v)
        return r

    cases = [(desc(), rows(status=None), b"null buffer"),
             (desc(nseg=2), rows(), b"single-tensor state"),
             (desc(n=10), rows(), b"not a multiple of the row size 3"),
             (desc(tab=tableaus.TSIT5), rows(), b"quartic dense output"),
             (desc(), rows(n_out=0), b"n_out"),
             (desc(), rows(workspace_bytes=8), b"workspace too small")]
    for d, r, text in cases:
        rc_ = lib.b2ode_rows_solve(C.byref(d), C.byref(r))
        msg = lib.b2ode_last_error()
        assert rc_ in (-1, -3) and text in msg, (rc_, msg)
