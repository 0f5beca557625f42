"""GPU: the tensor-core (wgmma) dense layer (b2ode_dense_layer, SURVEY 8f-3) against an fp64 product of the
TF32-rounded operands (what the tensor core is specified to compute), with and without the fused
Runge-Kutta stage combine as the A-operand producer."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def lib():
    from tfdiffeq_b200 import _lib
    return _lib


def tf32_round(x):
    """cvt.rna.tf32.f32: round the fp32 mantissa to 10 bits, nearest, ties away from zero."""
    i = x.contiguous().view(torch.int32)
    r = ((i.to(torch.int64) + 0x1000) & 0xFFFFE000).to(torch.int32)
    return r.view(torch.float32)


def run_layer(x, W, bias, act, ks=None, coefs=None, dt=None, want_ystage=False):
    L = lib()
    M, K = x.shape
    N = W.shape[0]
    out = torch.empty(M, N, dtype=torch.float32, device=DEV)
    ystage = torch.empty_like(x) if want_ystage else None
    state = None
    karr, carr, nk = None, None, 0
    if ks:
        nk = len(ks)
        karr = (C.c_void_p * nk)(*[k.data_ptr() for k in ks])
        carr = (C.c_double * nk)(*coefs)
        st = L.State()
        st.dt = dt
        state = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(DEV)
    L.check(L.lib.b2ode_dense_layer(C.c_void_p(x.data_ptr()), karr, carr, nk,
                                    C.c_void_p(state.data_ptr()) if state is not None else None,
                                    C.c_void_p(ystage.data_ptr()) if ystage is not None else None,
                                    C.c_void_p(tf32_round(W).data_ptr()), C.c_void_p(bias.data_ptr()) if bias is not None else None,
                                    C.c_void_p(out.data_ptr()), M, K, N, act,
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return out, ystage


def reference(a, W, bias, act):
    r = tf32_round(a).double() @ tf32_round(W).double().t()
    if bias is not None:
        r = r + bias.double()
    if act == 1:
        r = torch.relu(r)
    elif act == 2:
        r = torch.tanh(r)
    elif act == 3:
        r = torch.nn.functional.softplus(r)
    return r


@pytest.mark.parametrize("M,K,N", [(128, 64, 64), (128, 32, 16), (1000, 64, 256), (300, 100, 48), (257, 36, 16),
                                   (512, 256, 512), (4096, 784, 256), (65, 7, 32)])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_dense_layer_matches_tf32_reference(M, K, N, act):
    g = torch.Generator(device="cpu").manual_seed(M * 7 + K * 3 + N)
    x = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    out, _ = run_layer(x, W, b, act)
    ref = reference(x, W, b, act)
    err = float((out.double() - ref).abs().max())
    scale = max(1.0, float(ref.abs().max()))
    assert err <= 2e-5 * scale, (M, K, N, act, err)


# stage-row coefficients for up to 8 k's (the producer's NK = 1 .. 8 instantiations)
STAGE_COEFS = [19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729, 9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176]


def host_stage_input(y0, ks, coefs, dt):
    """k_rk_stage's fp32 order: (dt*beta_j) rounded to fp32, times k_j, summed left to right, then y0 + sum."""
    dt32 = torch.tensor(dt, dtype=torch.float32)
    acc = None
    for c, k in zip(coefs, ks):
        term = (dt32 * torch.tensor(c, dtype=torch.float32)).item() * k
        acc = term if acc is None else acc + term
    return y0 + acc


def test_dense_layer_with_fused_stage_combine():
    """A = y0 + sum_j (dt*beta_j) k_j built in the kernel (same fp32 operation order as k_rk_stage), then the GEMM;
    every stage-combine width the producer is instantiated for (nk = 1 .. 8)."""
    g = torch.Generator(device="cpu").manual_seed(5)
    M, K, N = 777, 64, 128
    y0 = torch.randn(M, K, generator=g).to(DEV)
    ks = [torch.randn(M, K, generator=g).to(DEV) for _ in range(8)]
    dt = 0.0371
    W = (torch.randn(N, K, generator=g) / 8).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    for nk in range(1, 9):
        out, ystage = run_layer(y0, W, b, 1, ks=ks[:nk], coefs=STAGE_COEFS[:nk], dt=dt, want_ystage=True)
        a = host_stage_input(y0, ks[:nk], STAGE_COEFS[:nk], dt)
        assert torch.equal(ystage, a), nk                                        # bit-identical stage input
        ref = reference(a, W, b, 1)
        assert float((out.double() - ref).abs().max()) <= 2e-5 * max(1.0, float(ref.abs().max())), nk


def run_layer_x3(x, W, bias, act, ks=None, coefs=None, dt=None, want_ystage=False):
    """b2ode_dense_layer_x3 through the C ABI: W split on the host as W_hi = tf32(W), W_lo = tf32(W - W_hi)."""
    L = lib()
    M, K = x.shape
    N = W.shape[0]
    out = torch.empty(M, N, dtype=torch.float32, device=DEV)
    ystage = torch.empty_like(x) if want_ystage else None
    state = None
    karr, carr, nk = None, None, 0
    if ks:
        nk = len(ks)
        karr = (C.c_void_p * nk)(*[k.data_ptr() for k in ks])
        carr = (C.c_double * nk)(*coefs)
        st = L.State()
        st.dt = dt
        state = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(DEV)
    hi = tf32_round(W)
    lo = tf32_round(W - hi)
    L.check(L.lib.b2ode_dense_layer_x3(C.c_void_p(x.data_ptr()), karr, carr, nk,
                                       C.c_void_p(state.data_ptr()) if state is not None else None,
                                       C.c_void_p(ystage.data_ptr()) if ystage is not None else None,
                                       C.c_void_p(hi.data_ptr()), C.c_void_p(lo.data_ptr()),
                                       C.c_void_p(bias.data_ptr()) if bias is not None else None,
                                       C.c_void_p(out.data_ptr()), M, K, N, act,
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return out, ystage


def exact_reference(a, W, bias, act):
    """fp64 product of the UNROUNDED fp32 operands: what an fp32 matmul approximates."""
    r = a.double() @ W.double().t()
    if bias is not None:
        r = r + bias.double()
    return {0: lambda v: v, 1: torch.relu, 2: torch.tanh, 3: torch.nn.functional.softplus}[act](r)


@pytest.mark.parametrize("M,K,N", [(128, 64, 64), (128, 32, 16), (1000, 64, 256), (300, 100, 48), (257, 36, 16),
                                   (512, 256, 512), (4096, 784, 256), (65, 7, 32)])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_dense_layer_3xtf32_is_fp32_accurate(M, K, N, act):
    """The default numeric mode: split operands, fp32 accumulation.  Error vs the exact product must be at the level of
    an fp32 matmul (a few 1e-7 relative per term), i.e. ~500x below single-pass TF32's 2^-11 per operand, and not worse
    than cuBLAS's fp32 SGEMM on the same operands by more than a small factor."""
    g = torch.Generator(device="cpu").manual_seed(M * 7 + K * 3 + N)
    x = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    out, _ = run_layer_x3(x, W, b, act)
    ref = exact_reference(x, W, b, act)
    scale = max(1.0, float(ref.abs().max()))
    err = float((out.double() - ref).abs().max())
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        sg = torch.addmm(b, x, W.t())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    sg = {0: lambda v: v, 1: torch.relu, 2: torch.tanh, 3: torch.nn.functional.softplus}[act](sg)
    err_sgemm = float((sg.double() - ref).abs().max())
    # fp32 accumulation of K terms: ~sqrt(K) * 2^-24 typical, a few times that at the maximum over M*N outputs (the
    # tensor core's accumulator rounding is not specified to be round-to-nearest)
    assert err <= 1e-6 * max(4.0, K ** 0.5) * scale, (M, K, N, act, err)
    assert err <= 16 * err_sgemm + 1e-6 * scale, (err, err_sgemm)
    # and ~3 orders of magnitude tighter than single-pass TF32 on the same inputs
    tf, _ = run_layer(x, W, b, act)
    err_tf32 = float((tf.double() - ref).abs().max())
    assert err < err_tf32 / 20 or err_tf32 < 1e-6


def test_dense_layer_3xtf32_with_fused_stage_combine():
    g = torch.Generator(device="cpu").manual_seed(6)
    M, K, N = 777, 64, 128
    y0 = torch.randn(M, K, generator=g).to(DEV)
    ks = [torch.randn(M, K, generator=g).to(DEV) for _ in range(8)]
    dt = 0.0371
    W = (torch.randn(N, K, generator=g) / 8).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    for nk in range(1, 9):
        out, ystage = run_layer_x3(y0, W, b, 1, ks=ks[:nk], coefs=STAGE_COEFS[:nk], dt=dt, want_ystage=True)
        a = host_stage_input(y0, ks[:nk], STAGE_COEFS[:nk], dt)
        assert torch.equal(ystage, a), nk                                        # bit-identical stage input
        ref = exact_reference(a, W, b, 1)
        assert float((out.double() - ref).abs().max()) <= 4e-6 * max(1.0, float(ref.abs().max())), nk


def test_dense_layer_argument_checks():
    L = lib()
    x = torch.zeros(4, 8, device=DEV)
    W = torch.zeros(10, 8, device=DEV)
    out = torch.zeros(4, 10, device=DEV)
    rc = L.lib.b2ode_dense_layer(C.c_void_p(x.data_ptr()), None, None, 0, None, None, C.c_void_p(W.data_ptr()), None,
                                 C.c_void_p(out.data_ptr()), 4, 8, 10, 0, None)
    assert rc == -1 and b"multiple of 16" in L.lib.b2ode_last_error()


@pytest.mark.parametrize("mode", [True, "tf32"])
def test_dense_mlp_func_through_odeint(mode):
    """rhs.DenseMLP (the reference's ODEFunc) as func: tensor-core layers + stage combine fused into layer 1
    == tensor-core layers behind the ordinary stage kernel (bit for bit: the stage input is identical).  The default
    mode (3xTF32) must agree with the plain-torch fp32 module well inside north_star's 1e-3 fp32 bar; single-pass TF32
    (opt-in) does not have to.  bosh3 (stage rows of 1 .. 3 k's) and tsit5 (up to 6) fuse as well; a reverse-time solve
    does not fuse and gives the same bits either way."""
    import tfdiffeq_b200 as tfd
    torch.manual_seed(0)
    m = tfd.rhs.DenseMLP(32, 64, "relu", tensor_cores=mode).to(DEV)
    y0 = torch.randn(1000, 32, device=DEV)
    t = torch.tensor([0., 0.5, 1.0])
    kw = dict(rtol=1e-3, atol=1e-3, method="dopri5")
    for method, tt in (("bosh3", t), ("tsit5", t), ("dopri5", t.flip(0).contiguous()), ("dopri5", t)):
        a = tfd.odeint(m, y0, tt, **dict(kw, method=method))
        sa = dict(tfd.last_stats)
        b = tfd.odeint(m, y0, tt, options=dict(fused_rhs=False), **dict(kw, method=method))   # separate stage kernel
        sb = dict(tfd.last_stats)
        assert sa["stage_func"] == bool(tt[-1] > tt[0]) and not sb["stage_func"], (method, sa["stage_func"])
        assert (sa["n_accepted"], sa["n_rejected"], sa["nfe"]) == (sb["n_accepted"], sb["n_rejected"], sb["nfe"])
        assert torch.equal(a, b), method
    m.tensor_cores = False
    c = tfd.odeint(m, y0, t, **kw)                                          # plain torch fp32 func
    sc = dict(tfd.last_stats)
    assert abs(sa["n_accepted"] - sc["n_accepted"]) <= 1
    tol = 2e-3 if mode == "tf32" else 1e-4          # the fp32 parity bar is 1e-3; the default mode sits 10x inside it
    assert float((a - c).abs().max()) <= tol * max(1.0, float(c.abs().max()))
    assert m.nfe > 0
    # CUDA-graph replay of the tensor-core attempt
    m.tensor_cores = mode
    d = tfd.odeint(m, y0, t, options=dict(cuda_graph=True), **kw)
    assert torch.equal(a, d)


def test_dense_mlp_trains_through_the_adjoint():
    import tfdiffeq_b200 as tfd
    torch.manual_seed(1)
    m = tfd.rhs.DenseMLP(16, 32, "tanh").to(DEV)
    y0 = torch.randn(64, 16, device=DEV, requires_grad=True)
    out = tfd.odeint_adjoint(m, y0, torch.tensor([0., 1.]), rtol=1e-4, atol=1e-5, method="dopri5")
    out[-1].pow(2).mean().backward()
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())
    assert y0.grad is not None


# ---- the chained three-layer kernel (b2ode_mlp3) ------------------------------------------------------------------

@torch.no_grad()
def chain_reference(a, m, act):
    h = reference(a, m.fc1.weight, m.fc1.bias, act).float()
    h = reference(h, m.fc2.weight, m.fc2.bias, act).float()
    return reference(h, m.fc3.weight, m.fc3.bias, 0)


# 37 965 rows = 297 tiles: more than two per SM on the persistent grid (132 SMs), plus a partial last tile
@pytest.mark.parametrize("M,D,H", [(128, 64, 256), (1000, 32, 64), (300, 16, 16), (257, 48, 80), (4096, 256, 256),
                                   (37965, 64, 128), (65, 112, 208)])
@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_mlp3_matches_chained_tf32_reference(M, D, H, act):
    import tfdiffeq_b200 as tfd
    torch.manual_seed(M + D + H)
    m = tfd.rhs.DenseMLP(D, H, act).to(DEV)
    x = torch.randn(M, D, device=DEV)
    out = tfd.rhs.mlp3(x, m.fc1, m.fc2, m.fc3, act)
    torch.cuda.synchronize()
    ref = chain_reference(x, m, {"relu": 1, "tanh": 2}[act])
    err = float((out.double() - ref).abs().max())
    # TF32 rounding of a hidden activation can flip on a 1-ulp fp32 difference in the accumulator: 2^-11 relative
    # on one element of a K-term dot product
    assert err <= 2e-3 * max(1.0, float(ref.abs().max())), err
    # and it is the same function as the three separate tensor-core layers
    h1 = tfd.rhs.dense_layer(x, m.fc1.weight, m.fc1.bias, act, mode="tf32")
    h2 = tfd.rhs.dense_layer(h1, m.fc2.weight, m.fc2.bias, act, mode="tf32")
    sep = tfd.rhs.dense_layer(h2, m.fc3.weight, m.fc3.bias, "none", mode="tf32")
    # (hidden activations are rounded ties-to-even here, ties-away there: an exact tie moves one activation by 2^-11)
    assert float((out - sep).abs().max()) <= 2e-4 * max(1.0, float(sep.abs().max()))


def test_mlp3_with_fused_stage_combine_and_repeat_launches():
    import tfdiffeq_b200 as tfd
    L = lib()
    torch.manual_seed(11)
    M, D, H = 5000, 64, 256
    m = tfd.rhs.DenseMLP(D, H, "relu").to(DEV)
    y0 = torch.randn(M, D, device=DEV)
    ks = [torch.randn(M, D, device=DEV) for _ in range(5)]
    coefs = [9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656]
    st = L.State()
    st.dt = 0.0123
    state = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(DEV)
    ystage = torch.empty_like(y0)
    outs = [tfd.rhs.mlp3(y0, m.fc1, m.fc2, m.fc3, "relu", stage=(ks, coefs, state.data_ptr(), ystage)) for _ in range(3)]
    torch.cuda.synchronize()
    dt32 = torch.tensor(st.dt, dtype=torch.float32)
    acc = None
    for c, k in zip(coefs, ks):
        term = (dt32 * torch.tensor(c, dtype=torch.float32)).item() * k
        acc = term if acc is None else acc + term
    a = y0 + acc
    assert torch.equal(ystage, a)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    ref = chain_reference(a, m, 1)
    assert float((outs[0].double() - ref).abs().max()) <= 2e-3 * max(1.0, float(ref.abs().max()))


def test_mlp3_argument_checks_and_per_layer_fallback():
    import tfdiffeq_b200 as tfd
    L = lib()
    x = torch.zeros(4, 24, device=DEV)
    rc = L.lib.b2ode_mlp3(C.c_void_p(x.data_ptr()), None, None, 0, None, None, C.c_void_p(x.data_ptr()), None, None, None,
                          C.c_void_p(x.data_ptr()), 4, 24, 32, 0, None)
    assert rc == -1 and b"multiples of 16" in L.lib.b2ode_last_error()
    assert L.lib.b2ode_mlp3_packed_bytes(24, 32) == -1
    assert L.lib.b2ode_mlp3_packed_bytes(64, 256) == (2 * 256 + 8 * 256 + 8 * 64) * 128
    # widths beyond the activation tile fall back to the per-layer kernels
    m = tfd.rhs.DenseMLP(32, 512, "relu", tensor_cores="tf32").to(DEV)
    assert not m.chained()
    y = torch.randn(100, 32, device=DEV)
    with torch.no_grad():
        a = m(0.0, y)
        m.tensor_cores = False
        b = m(0.0, y)
    assert float((a - b).abs().max()) <= 5e-3 * max(1.0, float(b.abs().max()))


def test_dense_mlp_chained_equals_per_layer_through_odeint():
    import tfdiffeq_b200 as tfd
    torch.manual_seed(3)
    m = tfd.rhs.DenseMLP(64, 128, "tanh", tensor_cores="tf32").to(DEV)
    assert m.chained()
    y0 = torch.randn(2000, 64, device=DEV)
    t = torch.tensor([0., 1.0])
    kw = dict(rtol=1e-4, atol=1e-4, method="dopri5")
    a = tfd.odeint(m, y0, t, **kw)
    sa = dict(tfd.last_stats)
    m.chain = False
    b = tfd.odeint(m, y0, t, **kw)
    sb = dict(tfd.last_stats)
    assert abs(sa["n_accepted"] - sb["n_accepted"]) <= 1
    assert float((a - b).abs().max()) <= 1e-3 * max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("mode", [True, "tf32"])
def test_mlp3_repacks_when_a_weight_changes(mode):
    import tfdiffeq_b200 as tfd
    torch.manual_seed(4)
    m = tfd.rhs.DenseMLP(32, 64, "relu", tensor_cores=mode).to(DEV)
    x = torch.randn(300, 32, device=DEV)
    with torch.no_grad():
        a = m(0.0, x).clone()
        m.fc2.weight.mul_(0.5)
        b = m(0.0, x)
        m.tensor_cores = False
        ref = m(0.0, x)
    assert not torch.equal(a, b)
    assert float((b - ref).abs().max()) <= 5e-3 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("mode", [True, "tf32"])
def test_weight_cache_never_serves_a_dead_models_weights(mode):
    """ADVICE r1: caches keyed by id() could alias a freed model whose addresses the allocator hands out again.  Build a
    model, evaluate it, free it, build a new one of the same shape (same `_version`, very likely the same storage) --
    the tensor-core path must use the NEW weights."""
    import gc
    import tfdiffeq_b200 as tfd
    x = torch.randn(200, 32, device=DEV)
    for seed in range(4):
        torch.manual_seed(100 + seed)
        m = tfd.rhs.DenseMLP(32, 64, "relu", tensor_cores=mode).to(DEV)
        with torch.no_grad():
            got = m(0.0, x)
            m.tensor_cores = False
            want = m(0.0, x)
        tol = 5e-3 if mode == "tf32" else 1e-5
        assert float((got - want).abs().max()) <= tol * max(1.0, float(want.abs().max())), seed
        del m, got, want
        gc.collect()
    # .data mutation does not bump _version: explicit invalidation is the documented way
    torch.manual_seed(7)
    m = tfd.rhs.DenseMLP(32, 64, "relu", tensor_cores=mode).to(DEV)
    with torch.no_grad():
        m(0.0, x)
        m.fc1.weight.data.mul_(2.0)
        m.invalidate_tensor_core_cache()
        got = m(0.0, x)
        m.tensor_cores = False
        want = m(0.0, x)
    assert float((got - want).abs().max()) <= (5e-3 if mode == "tf32" else 1e-5) * max(1.0, float(want.abs().max()))


@pytest.mark.parametrize("mode", [True, "tf32"])
def test_conv2d_odefunc_tensor_core_path(mode):
    """rhs.Conv2dODEFunc (tfdiffeq/models/conv_odenet.py:45-143) on an NHWC state: 1x1 convs on the tensor-core dense-layer
    kernel (+ cuDNN channels-last 3x3) against the same module in plain fp32 torch; through odeint with the stage
    combine fused into conv1, bit-identical to the unfused stage kernel."""
    import tfdiffeq_b200 as tfd
    torch.manual_seed(2)
    f = tfd.rhs.Conv2dODEFunc(64, tensor_cores=mode).to(DEV)
    x = torch.randn(6, 28, 28, 64, device=DEV)
    with torch.no_grad():
        got = f(torch.tensor(0.0, device=DEV), x)
        f.tensor_cores = False
        old = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            want = f(torch.tensor(0.0, device=DEV), x)
        finally:
            torch.backends.cudnn.allow_tf32 = old
        f.tensor_cores = mode
    assert got.shape == x.shape and got.is_contiguous()
    tol = 5e-3 if mode == "tf32" else 2e-5
    assert float((got - want).abs().max()) <= tol * max(1.0, float(want.abs().max()))
    t = torch.tensor([0., 1.])
    kw = dict(rtol=1e-3, atol=1e-3, method="dopri5")
    a = tfd.odeint(f, x, t, options=dict(max_num_steps=1000), **kw)
    sa = dict(tfd.last_stats)
    b = tfd.odeint(f, x, t, options=dict(max_num_steps=1000, fused_rhs=False), **kw)
    sb = dict(tfd.last_stats)
    assert (sa["n_accepted"], sa["n_rejected"], sa["nfe"]) == (sb["n_accepted"], sb["n_rejected"], sb["nfe"])
    assert torch.equal(a, b)
    f.tensor_cores = False
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        c = tfd.odeint(f, x, t, options=dict(max_num_steps=1000), **kw)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    tol = 3e-3 if mode == "tf32" else 1e-4
    assert float((a - c).abs().max()) <= tol * max(1.0, float(c.abs().max()))
