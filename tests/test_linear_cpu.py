"""CPU (no GPU needed): b2ode_linear_f64 rejects bad arguments before any CUDA call, and the built kernel is what it
claims to be -- fp64 tensor-core instructions (DMMA) and no spills to local memory in any instantiation."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from tfdiffeq_b200 import _lib, rhs

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "tfdiffeq_b200", "libb2ode.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
EINVAL = -1

X, A_IMG, OUT, YS, STATE, K0 = (C.c_void_p(0x10000 * i) for i in range(1, 7))   # never dereferenced


def _call(x=X, k=None, coef=None, nk=0, state=None, ystage=None, img=A_IMG, out=OUT, M=100, D=128):
    return _lib.lib.b2ode_linear_f64(x, k, coef, nk, state, ystage, img, out, M, D, None)


def _stage(nk, ptrs=None):
    ptrs = ptrs if ptrs is not None else [K0.value] * nk
    return (C.c_void_p * max(nk, 1))(*ptrs), (C.c_double * max(nk, 1))(*([0.5] * nk))


def test_image_bytes():
    lib = _lib.lib
    for D in (16, 32, 48, 64, 80, 96, 112, 128):
        assert lib.b2ode_linear_image_bytes(D) == D * D * 8
    for D in (0, 8, 12, 24, 144, 256, -16):
        assert lib.b2ode_linear_image_bytes(D) == -1


@pytest.mark.parametrize("case", ["D12", "D0", "D144", "D256", "M0", "nk_neg", "nk_14", "null_x", "null_img", "null_out",
                                  "misaligned_x", "misaligned_out", "misaligned_img", "misaligned_ystage", "misaligned_k",
                                  "null_k_entry", "nk_without_state", "nk_without_k"])
def test_bad_arguments_are_rejected(case):
    k, coef = _stage(2)
    kw = dict(k=k, coef=coef, nk=2, state=STATE)
    if case.startswith("D"):
        kw["D"] = int(case[1:])
    elif case == "M0":
        kw["M"] = 0
    elif case == "nk_neg":
        kw["nk"] = -1
    elif case == "nk_14":
        k, coef = _stage(14)
        kw.update(k=k, coef=coef, nk=14)
    elif case.startswith("null_") and case != "null_k_entry":
        kw[{"null_x": "x", "null_img": "img", "null_out": "out"}[case]] = None
    elif case.startswith("misaligned_"):
        what = case[len("misaligned_"):]
        if what == "k":
            kw["k"], _ = _stage(2, [K0.value, K0.value + 8])
        else:
            kw[{"x": "x", "out": "out", "img": "img", "ystage": "ystage"}[what]] = C.c_void_p(
                {"x": X, "out": OUT, "img": A_IMG, "ystage": YS}[what].value + 8)
    elif case == "null_k_entry":
        kw["k"], _ = _stage(2, [K0.value, None])
    elif case == "nk_without_state":
        kw["state"] = None
    elif case == "nk_without_k":
        kw["k"] = None
    assert _call(**kw) == EINVAL
    assert b"linear" in _lib.lib.b2ode_last_error()


def test_plain_torch_on_cpu():
    f = rhs.LinearODE(torch.eye(16, dtype=torch.float64) * 2.0)
    y = torch.arange(32, dtype=torch.float64).reshape(2, 16)
    with torch.no_grad():
        assert not f.uses_tensor_cores(y)
        assert torch.equal(f(0.0, y), y @ f.A)
    assert f.nfe == 1 and f.A.dtype == torch.float64 and isinstance(f.A, torch.nn.Parameter)
    with pytest.raises(ValueError):
        rhs.LinearODE(torch.zeros(3, 4))


def test_image_is_the_documented_permutation():
    D = 32
    A = torch.arange(D * D, dtype=torch.float64).reshape(D, D)
    img = rhs._linear_image(A, 1.0).reshape(-1)
    for c in range(D // 16):
        for n in range(D // 8):
            for h in range(2):
                for g in range(8):
                    for t in range(4):
                        for e in range(2):
                            idx = (((c * (D // 8) + n) * 2 + h) * 32 + 4 * g + t) * 2 + e
                            assert img[idx] == A[16 * c + 4 * t + 2 * h + e, 8 * n + g]
    assert torch.equal(rhs._linear_image(A, -1.0).reshape(-1), -img)


KERNELS = ["_Z12k_linear_f64ILi%dEEv12LinearParams" % nk for nk in range(14)]


@pytest.mark.skipif(not (os.path.exists(LIB) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")
@pytest.mark.parametrize("kernel", KERNELS)
def test_linear_kernel_sass_uses_dmma_and_does_not_spill(kernel):
    out = subprocess.run([CUOBJDUMP, "-sass", "-fun", kernel, LIB], capture_output=True, text=True, timeout=300).stdout
    ins = [m.group(1).strip() for m in (re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line) for line in out.splitlines()) if m]
    assert ins, "kernel not found in the library: " + kernel
    ops = [t.split()[0] if not t.startswith("@") else t.split()[1] for t in ins]
    assert any(o.startswith("DMMA") for o in ops)
    assert not any(o.startswith(("LDL", "STL")) for o in ops), "the kernel spills to local memory"
