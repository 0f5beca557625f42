"""GPU: the TF32 tensor-core kernels and the fp64 linear kernel bit for bit on exactly representable operands
(tests/exact_gemm.py), and the element-wise producer path taken by misaligned inputs.

On these operands every partial sum is exact in fp32, so the kernels have exactly one correct output: single-pass TF32
and 3xTF32 dense layers, their stage-combine producer for every nk, the chained three-layer kernel over its ring
configurations and the fp64 linear kernel for every nk are compared with ``torch.equal``; tanh and softplus, which
are not exact, per element in fp32 ulps of the fp64 function of the exact pre-activation.  M is sized from the
device's SM count, and each launch geometry the case was chosen for is asserted before the comparison."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_gemm as eg

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _lib():
    from tfdiffeq_b200 import _lib
    return _lib


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def dev(a, offset=0):
    """`a` on the GPU; `offset` > 0 places it `offset` elements into a fresh buffer (a view that is not 16-byte aligned)."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    buf = torch.empty(t.numel() + offset, dtype=t.dtype, device=DEV)
    v = buf[offset:].view(t.shape)
    v.copy_(t)
    return v


def _state(dt):
    st = _lib().State()
    st.dt = dt
    return torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(DEV)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def run_dense(x, ks, coefs, W, bias, mode, act, ystage=None, out=None):
    """b2ode_dense_layer / _x3 through the C ABI; W as fp32 values, rounded (or split) here as the host does."""
    L = _lib()
    M, K = x.shape
    N = W.shape[0]
    out = torch.empty(M, N, device=DEV) if out is None else out
    nk = len(ks)
    karr = (C.c_void_p * nk)(*[k.data_ptr() for k in ks]) if nk else None
    carr = (C.c_double * nk)(*coefs) if nk else None
    state = _state(eg.DT) if nk else None
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if mode == "tf32":
        w = dev(eg.tf32_rna(W))
        rc = L.lib.b2ode_dense_layer(_ptr(x), karr, carr, nk, _ptr(state), _ptr(ystage), _ptr(w), _ptr(bias), _ptr(out),
                                     M, K, N, act, stream)
    else:
        hi, lo = (dev(h) for h in eg.tf32_split(W))
        rc = L.lib.b2ode_dense_layer_x3(_ptr(x), karr, carr, nk, _ptr(state), _ptr(ystage), _ptr(hi), _ptr(lo), _ptr(bias),
                                        _ptr(out), M, K, N, act, stream)
    torch.cuda.synchronize()
    return rc, out


def _act64(pre, act):
    if act == 1:
        return np.maximum(pre, 0.0)
    if act == 2:
        return np.tanh(pre)
    if act == 3:
        return np.logaddexp(0.0, pre)
    return pre


def check_output(out, pre, act):
    """act 0 / 1: bit for bit.  tanh (tanhf, 2 ulp) and softplus (log1pf(expf), 4 ulp): per element within those ulps of
    the fp64 function of the exact pre-activation, with a floor at the smallest normal."""
    got = out.cpu().numpy().astype(np.float64)
    want = _act64(pre, act)
    if act in (0, 1):
        assert np.array_equal(got, want), int(np.count_nonzero(got != want))
        return
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    bound = (2 if act == 2 else 4) * np.maximum(ulp, 2.0 ** -126)
    err = np.abs(got - want)
    assert np.all(err <= bound), float((err / bound).max())


def _assert_dense_geometry(case, M, sms):
    g = eg.dense_geometry(M, case.K, case.N, sms, case.mode == "x3")
    if "items3" in case.name:
        assert g.items_per_cta >= 3, g
    if "2tiles" in case.name:
        assert g.tiles_n >= 2 and g.last_nt < g.ns * eg.NSUB, g
    return g


@pytest.mark.parametrize("via", ["c_abi", "rhs"])
@pytest.mark.parametrize("case", eg.DENSE_CASES, ids=lambda c: c.name)
def test_dense_layer_exact(case, via):
    sms = _sms()
    ops = eg.dense_operands(case, sms)
    M = ops["x"].shape[0]
    _assert_dense_geometry(case, M, sms)
    _, pre = eg.dense_expected(ops, case)
    x = dev(ops["x"])
    bias = dev(ops["bias"]) if ops["bias"] is not None else None
    if via == "c_abi":
        rc, out = run_dense(x, [], [], ops["W"], bias, case.mode, case.act)
        assert rc == 0
    else:
        from tfdiffeq_b200 import rhs
        out = rhs.dense_layer(x, dev(ops["W"]), bias, ["none", "relu", "tanh", "softplus"][case.act],
                              mode="3xtf32" if case.mode == "x3" else "tf32")
        torch.cuda.synchronize()
    check_output(out, pre, case.act)


@pytest.mark.parametrize("case", eg.STAGE_CASES, ids=lambda c: c.name)
def test_stage_combine_producer_exact(case):
    """A = x + sum_j (dt coef_j) k_j formed by the producer (vector path for K = 100, element-wise for K = 98): ystage
    equals the host combine, the product is exact, and leaving out ystage changes nothing."""
    ops = eg.dense_operands(case, _sms())
    a, pre = eg.dense_expected(ops, case)
    x, ks = dev(ops["x"]), [dev(k) for k in ops["ks"]]
    bias = dev(ops["bias"])
    ys = torch.full_like(x, float("nan"))
    rc, out = run_dense(x, ks, ops["coefs"], ops["W"], bias, case.mode, case.act, ystage=ys)
    assert rc == 0
    assert np.array_equal(ys.cpu().numpy(), a)
    check_output(out, pre, case.act)
    rc, out2 = run_dense(x, ks, ops["coefs"], ops["W"], bias, case.mode, case.act)
    assert rc == 0 and torch.equal(out, out2)


def _mlp3_module(ops):
    D, H = ops["W"][0].shape[1], ops["W"][0].shape[0]
    from tfdiffeq_b200 import rhs
    m = rhs.DenseMLP(D, H, "relu", tensor_cores="tf32").to(DEV)
    with torch.no_grad():
        for fc, w, b in zip((m.fc1, m.fc2, m.fc3), ops["W"], ops["b"]):
            fc.weight.copy_(torch.from_numpy(w))
            fc.bias.copy_(torch.from_numpy(b))
    m.invalidate_tensor_core_cache()
    return m


@pytest.mark.parametrize("case", eg.MLP3_CASES, ids=lambda c: c.name)
def test_mlp3_exact(case):
    """fc1 -> act -> fc2 -> act -> fc3 in one launch: W rounded by k_mlp3_pack (RNA, with ties), hidden activations by
    the Veltkamp split (RNE, with ties), relu or none: bit for bit with the host chain."""
    from tfdiffeq_b200 import rhs
    sms = _sms()
    ops = eg.mlp3_operands(case, sms)
    M = ops["x"].shape[0]
    g = eg.mlp3_geometry(M, case.D, case.H, sms)
    if "tiles3" in case.name:
        assert g.tiles_per_cta >= 3, g
    if case.name.startswith("s2"):
        assert g.stages == 2
    if case.name.startswith("s8"):
        assert g.stages == 8
    if "partial" in case.name:
        layer = 0 if case.D > case.H else 2
        assert g.grp[layer] > 1 and g.subs[layer] % g.grp[layer], g
    a, want, _, _, _ = eg.mlp3_expected(ops, case)
    m = _mlp3_module(ops)
    act = ["none", "relu"][case.act]
    x = dev(ops["x"])
    stage, ys = None, None
    if case.nk:
        state = _state(eg.DT)
        ys = torch.full_like(x, float("nan"))
        stage = ([dev(k) for k in ops["ks"]], ops["coefs"], state.data_ptr(), ys)
    out = rhs.mlp3(x, m.fc1, m.fc2, m.fc3, act, stage=stage)
    torch.cuda.synchronize()
    got = out.cpu().numpy().astype(np.float64)
    assert np.array_equal(got, want), int(np.count_nonzero(got != want))
    if case.nk:
        assert np.array_equal(ys.cpu().numpy(), a)


@pytest.mark.parametrize("nk", range(14))
@pytest.mark.parametrize("D", eg.LINEAR_DIMS)
def test_linear_f64_exact(D, nk):
    """Integer operands (dyadic dt coef_j): every product and partial sum is exact in fp64, so out == Y A bit for bit,
    for +A and -A, with at least three 16-row blocks per warp (the NK <= 1 prefetch of the next block's first chunk)."""
    from tfdiffeq_b200 import rhs
    sms = _sms()
    M = eg.linear_rows(sms)
    assert eg.linear_blocks_per_warp(M, sms)[0] >= 3 and M % 16
    gen = torch.Generator(device=DEV).manual_seed(1000 * D + nk)
    A = torch.randint(-2 ** 10, 2 ** 10 + 1, (D, D), generator=gen, device=DEV).double()
    x = torch.randint(-2 ** 10, 2 ** 10 + 1, (M, D), generator=gen, device=DEV).double()
    ks = [2.0 * torch.randint(-20, 21, (M, D), generator=gen, device=DEV).double() for _ in range(nk)]
    coefs = eg.COEFS[:nk]
    Y = x.clone()
    for c, k in zip(coefs, ks):
        Y += (eg.DT * c) * k                                   # exact: integers well inside 2^53
    want = Y @ A                                              # exact in any summation order (eg.linear_bits <= 50)
    state = _state(eg.DT)
    ys = torch.full_like(x, float("nan")) if nk else None
    out = rhs.linear_f64(x, A, 1.0, stage=(ks, coefs, state.data_ptr(), ys) if nk else None)
    assert torch.equal(out, want)
    if nk:
        assert torch.equal(ys, Y)
    neg = rhs.linear_f64(x, A, -1.0, stage=(ks, coefs, state.data_ptr(), None) if nk else None)
    assert torch.equal(neg, -want)


# ---- misaligned inputs: the element-wise producer path ----------------------------------------------------------

@pytest.mark.parametrize("mode", ["tf32", "x3"])
@pytest.mark.parametrize("which", ["x", "k", "ystage", "W"])
def test_dense_layer_misaligned_operand_matches_aligned(mode, which):
    case = eg.DenseCase("misaligned", 700, 64, 128, 3, mode, 1, True)
    ops = eg.dense_operands(case, _sms())
    a, pre = eg.dense_expected(ops, case)
    bias = dev(ops["bias"])

    def run(off):
        x = dev(ops["x"], off if which == "x" else 0)
        ks = [dev(k, off if which == "k" and j == 2 else 0) for j, k in enumerate(ops["ks"])]
        ys = dev(np.zeros_like(ops["x"]), off if which == "ystage" else 0)
        if which == "W":
            L = _lib()
            out = torch.empty(x.shape[0], case.N, device=DEV)
            karr = (C.c_void_p * 3)(*[k.data_ptr() for k in ks])
            carr = (C.c_double * 3)(*ops["coefs"])
            state = _state(eg.DT)
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            if mode == "tf32":
                w = dev(eg.tf32_rna(ops["W"]), off)
                rc = L.lib.b2ode_dense_layer(_ptr(x), karr, carr, 3, _ptr(state), _ptr(ys), _ptr(w), _ptr(bias), _ptr(out),
                                             x.shape[0], case.K, case.N, case.act, stream)
            else:
                hi, lo = eg.tf32_split(ops["W"])
                hi, lo = dev(hi), dev(lo, off)                    # (held until the kernel has run)
                rc = L.lib.b2ode_dense_layer_x3(_ptr(x), karr, carr, 3, _ptr(state), _ptr(ys), _ptr(hi), _ptr(lo),
                                                _ptr(bias), _ptr(out), x.shape[0], case.K, case.N, case.act, stream)
            torch.cuda.synchronize()
        else:
            rc, out = run_dense(x, ks, ops["coefs"], ops["W"], bias, mode, case.act, ystage=ys)
        assert rc == 0
        return out, ys

    out0, ys0 = run(0)
    out1, ys1 = run(1)
    assert torch.equal(out0, out1) and torch.equal(ys0, ys1)
    assert np.array_equal(ys1.cpu().numpy(), a)
    check_output(out1, pre, case.act)


@pytest.mark.parametrize("which", ["x", "k", "ystage"])
def test_mlp3_misaligned_input_matches_aligned(which):
    from tfdiffeq_b200 import rhs
    case = eg.Mlp3Case("misaligned", 900, 64, 96, 1, 2)
    ops = eg.mlp3_operands(case, _sms())
    _, want, _, _, _ = eg.mlp3_expected(ops, case)
    m = _mlp3_module(ops)
    state = _state(eg.DT)
    outs = []
    for off in (0, 1):
        x = dev(ops["x"], off if which == "x" else 0)
        ks = [dev(k, off if which == "k" and j == 1 else 0) for j, k in enumerate(ops["ks"])]
        ys = dev(np.zeros_like(ops["x"]), off if which == "ystage" else 0)
        outs.append(rhs.mlp3(x, m.fc1, m.fc2, m.fc3, "relu", stage=(ks, ops["coefs"], state.data_ptr(), ys)))
        torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    assert np.array_equal(outs[1].cpu().numpy().astype(np.float64), want)


@pytest.mark.parametrize("mode", [True, "tf32"])
def test_funcs_on_misaligned_views(mode):
    """DenseMLP, Conv2dODEFunc and LinearODE on a contiguous view at an odd element offset (buf[1:].view(...)): the
    same bits as on an aligned copy."""
    from tfdiffeq_b200 import rhs
    torch.manual_seed(8)
    M, D = 300, 32
    buf = torch.randn(M * D + 1, device=DEV)
    xv = buf[1:].view(M, D)
    assert xv.is_contiguous() and xv.data_ptr() % 16
    for chain in (True, False):
        m = rhs.DenseMLP(D, 64, "softplus", tensor_cores=mode, chain=chain).to(DEV)
        with torch.no_grad():
            assert torch.equal(m(0.0, xv), m(0.0, xv.clone()))
    f = rhs.Conv2dODEFunc(16, tensor_cores=mode).to(DEV)
    cbuf = torch.randn(2 * 6 * 6 * 16 + 1, device=DEV)
    cv = cbuf[1:].view(2, 6, 6, 16)
    with torch.no_grad():
        assert torch.equal(f(torch.tensor(0.0), cv), f(torch.tensor(0.0), cv.clone()))
    lin = rhs.LinearODE(torch.randn(D, D, dtype=torch.float64) * 0.1).to(DEV)
    lbuf = torch.randn(M * D + 1, dtype=torch.float64, device=DEV)
    lv = lbuf[1:].view(M, D)
    assert lv.data_ptr() % 16
    with torch.no_grad():
        assert lin.uses_tensor_cores(lv)
        assert torch.equal(lin(0.0, lv), lin(0.0, lv.clone()))


def test_misaligned_out_is_rejected_before_any_launch():
    L = _lib()
    before = L.lib.b2ode_launch_count()
    x = torch.zeros(256, 64, device=DEV)
    W = torch.zeros(64, 64, device=DEV)
    obuf = torch.zeros(256 * 64 + 1, device=DEV)
    out = obuf[1:].view(256, 64)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = L.lib.b2ode_dense_layer(_ptr(x), None, None, 0, None, None, _ptr(W), None, _ptr(out), 256, 64, 64, 0, stream)
    assert rc != 0 and b"aligned" in L.lib.b2ode_last_error()
    rc = L.lib.b2ode_dense_layer_x3(_ptr(x), None, None, 0, None, None, _ptr(W), _ptr(W), None, _ptr(out), 256, 64, 64, 0,
                                    stream)
    assert rc != 0 and b"aligned" in L.lib.b2ode_last_error()
    packed = torch.zeros(L.lib.b2ode_mlp3_packed_bytes(64, 64), dtype=torch.uint8, device=DEV)
    rc = L.lib.b2ode_mlp3(_ptr(x), None, None, 0, None, None, _ptr(packed), None, None, None, _ptr(out), 256, 64, 64, 0,
                          stream)
    assert rc != 0 and b"aligned" in L.lib.b2ode_last_error()
    assert L.lib.b2ode_launch_count() == before
