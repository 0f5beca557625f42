"""Built-in right-hand sides (SURVEY.md 8(f)-2).

Each class is an ordinary ``nn.Module`` -- ``forward(t, y)`` is written in plain torch ops and works anywhere
(on the generic path, on CPU, under autograd).  When an instance is handed to ``odeint`` with an adaptive
Runge-Kutta method and a single ``(..., k * dim)`` CUDA state, the solver recognises it and runs the WHOLE solve in
one persistent kernel (``b2ode_fused_solve``): every trajectory lives in one thread's registers, HBM traffic is
the solution slab only.  Batches that cannot stay co-resident (and tsit5, whose dense output needs all k's) take the
per-stage kernels with the right-hand side evaluated inside the stage kernel (``b2ode_rk_stage_rhs``): one launch per
stage, no ``forward`` call at all.  For ``Lorenz``, ``LotkaVolterra`` and ``Kepler`` the kernel evaluates exactly the
same IEEE operations in the same order as ``forward`` does (``pow(x, 1.5)`` is the same routine in torch and in the
library), so both agree to the last bit per evaluation; ``CubicMLP.forward`` and ``LatentODEFunc.forward`` multiply
through cuBLAS and agree to rounding.  ``forward`` takes the same ``(..., k * dim)`` states the kernels do.  ``options={'fused_rhs': False}`` forces
the generic path.  ``odeint_adjoint(..., adjoint_options={'fused_vjp': True})`` also runs the backward pass's augmented
dynamics (``f`` and its vector-Jacobian products) in the stage kernels; see ``odeint_adjoint``.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib


class BuiltinRHS(nn.Module):
    kind = None      # B2ODE_RHS_* code
    dim = None       # size of the last state axis
    # a built-in whose kernels differentiate its weights: (count in words, names) of the parameters, in the order the
    # kernels flatten them; they train all together or not at all
    trainable_weights = None

    def rhs_params(self):
        raise NotImplementedError

    def rows(self, y):
        """A ``(..., k * dim)`` state as ``(..., k, dim)``: the rows the kernels solve (a view for k = 1)."""
        if y.shape[-1] == self.dim:
            return y
        return y.reshape(y.shape[:-1] + (y.shape[-1] // self.dim, self.dim))

    def rhs_data(self, dtype, device):
        """Device buffer of staged weights for the kernel (None for parameter-free systems)."""
        return None

    def rhs_desc(self, dtype, device, time_sign):
        """``(_lib.RhsDesc, weights)`` for the kernels; the caller keeps ``weights`` referenced until the launches that
        read the descriptor are enqueued.  ``time_sign`` -1 describes the reversed system (misc.py:318-321)."""
        prm = self.rhs_params()
        weights = self.rhs_data(dtype, device)
        rd = _lib.RhsDesc(kind=self.kind, n_params=len(prm), time_sign=float(time_sign),
                          data=weights.data_ptr() if weights is not None else None)
        rd.params[:len(prm)] = prm
        return rd, weights


def weights_all_or_none(func):
    """True when ``func``'s parameters are exactly its ``trainable_weights``, in order, all trainable or all frozen."""
    params = list(func.parameters())
    names = func.trainable_weights[1]
    try:
        named = [func.get_parameter(n) for n in names]
    except AttributeError:           # a weight replaced by a buffer or a plain tensor
        return False
    return (len(params) == len(named) and all(p is q for p, q in zip(params, named))
            and len({p.requires_grad for p in params}) == 1)


class Lorenz(BuiltinRHS):
    """examples/lorenz_attractor.py:20-37, vectorised over leading batch axes: state (..., 3)."""
    kind, dim = _lib.RHS_LORENZ, 3

    def __init__(self, sigma=10.0, beta=8.0 / 3.0, rho=28.0):
        super(Lorenz, self).__init__()
        self.sigma, self.beta, self.rho = float(sigma), float(beta), float(rho)

    def rhs_params(self):
        return [self.sigma, self.beta, self.rho]

    def forward(self, t, y):
        s = self.rows(y)
        x, yy, z = s[..., 0], s[..., 1], s[..., 2]
        return torch.stack([self.sigma * (yy - x), x * (self.rho - z) - yy, x * yy - self.beta * z], -1).reshape(y.shape)


class LotkaVolterra(BuiltinRHS):
    """README.md:67-81: x' = a x - b x z, z' = -c z + d x z; state (..., 2)."""
    kind, dim = _lib.RHS_LOTKA_VOLTERRA, 2

    def __init__(self, a=1.5, b=1.0, c=3.0, d=1.0):
        super(LotkaVolterra, self).__init__()
        self.a, self.b, self.c, self.d = float(a), float(b), float(c), float(d)

    def rhs_params(self):
        return [self.a, self.b, self.c, self.d]

    def forward(self, t, y):
        s = self.rows(y)
        x, z = s[..., 0], s[..., 1]
        return torch.stack([self.a * x - self.b * x * z, -self.c * z + self.d * x * z], -1).reshape(y.shape)


class Kepler(BuiltinRHS):
    """DETEST class D (tests/DETEST/detest.py:263-283): two-body orbits, ``[x, y, vx, vy]`` per orbit, any number of orbits
    stacked along the last state axis (BASELINE config 5: 32 orbits = dim 128).  The kernels see the state as rows of 4."""
    kind, dim = _lib.RHS_KEPLER, 4

    def rhs_params(self):
        return []

    def forward(self, t, y):
        s = self.rows(y)
        x, yy, vx, vy = s[..., 0], s[..., 1], s[..., 2], s[..., 3]
        r3 = (x * x + yy * yy) ** 1.5
        return torch.stack([vx, vy, -x / r3, -yy / r3], -1).reshape(y.shape)


class CubicMLP(BuiltinRHS):
    """examples/ode_demo.py:115-129 (BASELINE config 3): ``W2 . tanh(W1 . y**3 + b1) + b2`` with a 2 -> H -> 2
    network (H <= 128); ``cube=False`` drops the ``y**3``.  Weights are ordinary ``nn.Parameter`` s, so the module
    trains like any other through ``odeint_adjoint``.  By default its backward solves take the vector-Jacobian products
    from torch autograd of ``forward``; with ``adjoint_options={'fused_vjp': True}`` the stage kernels evaluate them on the
    device, the parameter cotangents summed over all rows in a fixed order (all four weights trainable, or none).
    """
    kind, dim = _lib.RHS_CUBIC_MLP, 2
    trainable_weights = ("four", ("W1", "b1", "W2", "b2"))

    def __init__(self, hidden=50, cube=True, std=0.1, dtype=torch.float32, generator=None):
        super(CubicMLP, self).__init__()
        if not 1 <= hidden <= 128:
            raise ValueError("hidden width must be in [1, 128]")
        self.hidden, self.cube = int(hidden), bool(cube)
        self.W1 = nn.Parameter(torch.randn(2, hidden, dtype=dtype, generator=generator) * std)
        self.b1 = nn.Parameter(torch.zeros(hidden, dtype=dtype))
        self.W2 = nn.Parameter(torch.randn(hidden, 2, dtype=dtype, generator=generator) * std)
        self.b2 = nn.Parameter(torch.zeros(2, dtype=dtype))

    def rhs_params(self):
        return [float(self.hidden), 1.0 if self.cube else 0.0]

    def rhs_data(self, dtype, device):
        with torch.no_grad():
            return torch.cat([self.W1.reshape(-1), self.b1.reshape(-1), self.W2.reshape(-1), self.b2.reshape(-1)]).to(
                device=device, dtype=dtype).contiguous()

    def forward(self, t, y):
        s = self.rows(y)
        u = s ** 3 if self.cube else s
        return (torch.tanh(u @ self.W1 + self.b1) @ self.W2 + self.b2).reshape(y.shape)


class LatentODEFunc(BuiltinRHS):
    """examples/latent_ode.py:105-120 (``LatentODEfunc``): ``fc3(elu(fc2(elu(fc1(z)))))``, a 4 -> H -> H -> 4 network on
    ``(..., k * 4)`` latent states, H <= 32.  ``fc1``, ``fc2`` and ``fc3`` are ``nn.Linear`` layers initialised like
    ``nn.Linear``'s default (uniform in +-1/sqrt(fan_in)), drawn from ``generator``.  The kernels evaluate it with explicit
    mul/add in index order, ``expm1`` for elu and ``exp`` for its derivative; ``forward`` multiplies through cuBLAS, so the
    two agree to rounding.  It trains through ``odeint(..., options={'backprop': True})`` and ``odeint_adjoint`` (with
    ``fused_vjp`` the stage kernels take the vector-Jacobian products), the parameter cotangents summed over all rows in
    a fixed order (all six parameters trainable, or none)."""
    kind, dim = _lib.RHS_LATENT_MLP, 4
    trainable_weights = ("six", ("fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias"))

    def __init__(self, latent_dim=4, hidden=20, dtype=torch.float32, generator=None):
        super(LatentODEFunc, self).__init__()
        if latent_dim != 4:
            raise ValueError("latent_dim must be 4 (the kernels hold a row of 4 in registers), got %r" % (latent_dim,))
        if not 1 <= hidden <= 32:
            raise ValueError("hidden width must be in [1, 32], got %r" % (hidden,))
        self.latent_dim, self.hidden = 4, int(hidden)
        self.fc1 = nn.Linear(4, self.hidden, dtype=dtype)
        self.fc2 = nn.Linear(self.hidden, self.hidden, dtype=dtype)
        self.fc3 = nn.Linear(self.hidden, 4, dtype=dtype)
        with torch.no_grad():
            for fc in (self.fc1, self.fc2, self.fc3):
                bound = 1.0 / math.sqrt(fc.in_features)
                for p in (fc.weight, fc.bias):
                    p.copy_(torch.rand(p.shape, dtype=dtype, generator=generator) * (2 * bound) - bound)

    def rhs_params(self):
        return [float(self.hidden)]

    def rhs_data(self, dtype, device):
        with torch.no_grad():
            return torch.cat([p.reshape(-1) for p in (self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias,
                                                      self.fc3.weight, self.fc3.bias)]).to(device=device, dtype=dtype).contiguous()

    def forward(self, t, y):
        s = self.rows(y)
        return self.fc3(F.elu(self.fc2(F.elu(self.fc1(s))))).reshape(y.shape)


_ACT = {None: 0, "none": 0, "relu": 1, "tanh": 2, "softplus": 3}

# numeric modes of the tensor-core func
#   "3xtf32" (default, also `True`): every product is split hi/lo and accumulated in fp32 -- as accurate as fp32 FMAs,
#            so solutions stay within north_star's 1e-3 fp32 bar of the reference's fp32 matmuls
#   "tf32"   (opt-in): single-pass TF32 (10-bit mantissa operands), the chained one-launch kernel; ~1e-3 relative error
#            per evaluation -- faster, but it does NOT meet the fp32 parity bar over a whole solve
#   False    : plain torch everywhere
_MODES = {True: "3xtf32", "3xtf32": "3xtf32", "tf32": "tf32", False: None, None: None}

# set by odeint_adjoint for the duration of its forward and backward solves: "tf32" is promoted to "3xtf32" so that the
# forward pass, the backward reconstruction of y (both under no_grad on the tensor cores) and the VJPs (autograd, fp32)
# integrate the same dynamics to fp32 rounding
_FORCE_ACCURATE = [0]


def _round_tf32(w):
    """Round-to-nearest (ties away from zero, what cvt.rna.tf32.f32 does) to TF32's 10 explicit mantissa bits."""
    i = w.contiguous().view(torch.int32)
    return ((i + 0x1000) & -0x2000).view(torch.float32)


class _WeightCache(object):
    """Derived images of a weight tensor (TF32-rounded copy, hi/lo split, packed shared-memory image), rebuilt when the
    weight changes.  Entries hold a weak reference to the weight they were built from and are only hit when that very
    object is still alive (`ref() is weight`) -- an `id()` recycled by a new tensor can never alias an old entry -- and
    are dropped when the weight is collected.  Validity is (data_ptr, _version, shape): in-place updates through
    autograd-visible ops (optimizer steps, `copy_`, `add_`) bump `_version`; writes through `.data` do NOT --
    call `invalidate(weight)` (or `DenseMLP.invalidate_tensor_core_cache()`) after those."""

    def __init__(self):
        self._d = {}

    @staticmethod
    def _key(ws):
        return tuple((w.data_ptr(), w._version, tuple(w.shape)) for w in ws)

    def get(self, tag, ws, build):
        ws = tuple(ws)
        slot = (tag,) + tuple(id(w) for w in ws)
        hit = self._d.get(slot)
        key = self._key(ws)
        if hit is not None and hit[0] == key and all(r() is w for r, w in zip(hit[1], ws)):
            return hit[2]
        import weakref
        d = self._d

        def _drop(_ref, slot=slot, d=d):
            d.pop(slot, None)
        with torch.no_grad():
            val = build(*[w.detach() for w in ws])
        d[slot] = (key, tuple(weakref.ref(w, _drop) for w in ws), val)
        return val

    def invalidate(self, weight=None):
        if weight is None:
            self._d.clear()
            return
        for slot in [s for s in self._d if id(weight) in s[1:]]:
            self._d.pop(slot, None)


_CACHE = _WeightCache()


def invalidate(weight=None):
    """Forget the cached tensor-core images of `weight` (all weights when None): needed after `.data` mutation."""
    _CACHE.invalidate(weight)


def _tf32_weight(weight):
    return _CACHE.get("tf32", (weight,), _round_tf32)


def _split_weight(weight):
    """(W_hi, W_lo) of the 3xTF32 split: W_hi = tf32(W), W_lo = tf32(W - W_hi) (the subtraction is exact in fp32)."""
    def build(w):
        hi = _round_tf32(w.reshape(w.shape[0], -1))
        lo = _round_tf32(w.reshape(w.shape[0], -1).contiguous() - hi)
        return hi, lo
    return _CACHE.get("x3", (weight,), build)


def _stage_args(stage):
    import ctypes as C
    if stage is None:
        return None, None, 0, None, None
    ks, coefs, state, ys = stage
    nk = len(ks)
    return (C.c_void_p * nk)(*[k.data_ptr() for k in ks]), (C.c_double * nk)(*coefs), nk, state, ys


def dense_layer(x, weight, bias, act="none", stage=None, mode="3xtf32"):
    """``act(x @ weight.T + bias)`` on the tensor cores (wgmma), fp32 storage: ``b2ode_dense_layer_x3`` (mode "3xtf32",
    fp32-accurate products) or ``b2ode_dense_layer`` (mode "tf32").  ``weight`` is ``[N, K]`` (``nn.Linear.weight``; a 1x1
    convolution's ``[F, C, 1, 1]`` kernel is the same matrix) and ``x`` any contiguous tensor whose last axis is K.

    ``stage = (k_tensors, coefs, state_ptr, ystage_or_None)`` makes the Runge-Kutta stage combine the A-operand
    producer: A = x + sum_j (dt * coefs[j]) * k_tensors[j], dt read from the device state."""
    import ctypes as C
    K = x.shape[-1]
    M = x.numel() // K
    N = weight.shape[0]
    out = torch.empty(x.shape[:-1] + (N,), dtype=torch.float32, device=x.device)
    karr, carr, nk, state, ys = _stage_args(stage)

    def ptr(t):
        return C.c_void_p(t.data_ptr()) if t is not None else None
    stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
    if mode == "3xtf32":
        hi, lo = _split_weight(weight)
        _lib.check(_lib.lib.b2ode_dense_layer_x3(ptr(x), karr, carr, nk, C.c_void_p(state) if state else None, ptr(ys),
                                                 ptr(hi), ptr(lo), ptr(bias), ptr(out), M, K, N, _ACT[act], stream))
    else:
        _lib.check(_lib.lib.b2ode_dense_layer(ptr(x), karr, carr, nk, C.c_void_p(state) if state else None, ptr(ys),
                                              ptr(_tf32_weight(weight)), ptr(bias), ptr(out), M, K, N, _ACT[act], stream))
    return out


def _mlp3_packed(fc1, fc2, fc3):
    """The three weights as ``b2ode_mlp3``'s shared-memory image, rebuilt only when a weight changes."""
    import ctypes as C

    def build(w1, w2, w3):
        H, D = w1.shape
        nbytes = _lib.lib.b2ode_mlp3_packed_bytes(D, H)
        if nbytes < 0:
            raise ValueError("mlp3 needs dim and hidden to be multiples of 16 in [16, 256]")
        packed = torch.empty(nbytes, dtype=torch.uint8, device=w1.device)
        cw = [w.contiguous() for w in (w1, w2, w3)]
        _lib.check(_lib.lib.b2ode_mlp3_pack(
            C.c_void_p(cw[0].data_ptr()), C.c_void_p(cw[1].data_ptr()), C.c_void_p(cw[2].data_ptr()), D, H,
            C.c_void_p(packed.data_ptr()), C.c_void_p(torch.cuda.current_stream(packed.device).cuda_stream)))
        return packed
    return _CACHE.get("mlp3", (fc1.weight, fc2.weight, fc3.weight), build)


def mlp3(x, fc1, fc2, fc3, act="relu", stage=None):
    """``fc3(act(fc2(act(fc1(x)))))`` in one launch (``b2ode_mlp3``, single-pass TF32): hidden activations never reach
    HBM.  ``stage`` as in :func:`dense_layer`."""
    import ctypes as C
    M, D = x.shape
    H = fc1.weight.shape[0]
    out = torch.empty((M, D), dtype=torch.float32, device=x.device)
    karr, carr, nk, state, ys = _stage_args(stage)

    def ptr(t):
        return C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(_lib.lib.b2ode_mlp3(
        ptr(x), karr, carr, nk, C.c_void_p(state) if state else None, ptr(ys),
        ptr(_mlp3_packed(fc1, fc2, fc3)), ptr(fc1.bias), ptr(fc2.bias), ptr(fc3.bias), ptr(out), M, D, H, _ACT[act],
        C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
    return out


class _TensorCoreFunc(nn.Module):
    """Shared mode handling of the GEMM-backed funcs."""

    def _mode(self):
        m = _MODES[self.tensor_cores]
        if m == "tf32" and _FORCE_ACCURATE[0]:
            m = "3xtf32"
        return m

    def invalidate_tensor_core_cache(self):
        for p in self.parameters():
            _CACHE.invalidate(p)


class DenseMLP(_TensorCoreFunc):
    """The reference's ``ODEFunc`` (tfdiffeq/models/dense_odenet.py:11-92, time-independent form): fc1 -> act ->
    fc2 -> act -> fc3 on a ``(batch, dim)`` state, counting ``nfe`` like the reference does (:78).

    Under ``torch.no_grad()`` on a CUDA fp32 state -- which is how ``odeint`` evaluates ``func`` -- the three layers
    run on the tensor cores (wgmma), and the adaptive solvers feed the first layer straight from the stage combine (the
    stage input never round-trips HBM for the GEMM).  ``tensor_cores``: ``True`` / ``"3xtf32"`` (default) keeps fp32
    accuracy by splitting every operand into two TF32 halves (three tensor-core passes, fp32 accumulation), so the
    solution stays within the fp32 parity bar of the reference's fp32 matmuls; ``"tf32"`` opts into single-pass TF32
    and the chained one-launch kernel (faster, ~1e-3 relative error per evaluation); ``False`` is plain torch.  With
    autograd enabled (training, ``odeint_adjoint``'s VJPs) it is plain torch."""

    def __init__(self, dim, hidden, non_linearity="relu", tensor_cores=True, dtype=torch.float32, chain=True):
        super(DenseMLP, self).__init__()
        if non_linearity not in ("relu", "tanh", "softplus"):
            raise ValueError("non_linearity must be relu, tanh or softplus")
        if tensor_cores not in _MODES:
            raise ValueError("tensor_cores must be True, False, '3xtf32' or 'tf32'")
        self.dim, self.hidden, self.non_linearity, self.tensor_cores = int(dim), int(hidden), non_linearity, tensor_cores
        self.fc1 = nn.Linear(dim, hidden, dtype=dtype)
        self.fc2 = nn.Linear(hidden, hidden, dtype=dtype)
        self.fc3 = nn.Linear(hidden, dim, dtype=dtype)
        self.nfe = 0
        self.chain = chain

    def uses_tensor_cores(self, x):
        return (self._mode() is not None and x.is_cuda and x.dtype == torch.float32 and not torch.is_grad_enabled()
                and self.fc1.weight.dtype == torch.float32 and self.dim % 16 == 0 and self.hidden % 16 == 0
                and x.shape[-1] == self.dim)

    def chained(self):
        """One-launch form (``b2ode_mlp3``, single-pass TF32 only) when both widths fit the 128 KB activation tile."""
        return self._mode() == "tf32" and self.chain and self.dim <= 256 and self.hidden <= 256

    def _tail(self, h1):
        m = self._mode()
        h2 = dense_layer(h1, self.fc2.weight, self.fc2.bias, self.non_linearity, mode=m)
        return dense_layer(h2, self.fc3.weight, self.fc3.bias, "none", mode=m)

    def forward_from_stage(self, y0, ks, coefs, state_ptr, ystage):
        """First layer fed by the stage combine of y0 and the k's (all ``(batch, dim)`` fp32 CUDA tensors)."""
        self.nfe += 1
        if self.chained():
            return mlp3(y0, self.fc1, self.fc2, self.fc3, self.non_linearity, stage=(ks, coefs, state_ptr, ystage))
        h1 = dense_layer(y0, self.fc1.weight, self.fc1.bias, self.non_linearity, stage=(ks, coefs, state_ptr, ystage),
                         mode=self._mode())
        return self._tail(h1)

    def forward(self, t, x):
        self.nfe += 1
        if self.uses_tensor_cores(x):
            x2 = x.reshape(-1, self.dim)
            if not x2.is_contiguous():
                x2 = x2.contiguous()
            if self.chained():
                return mlp3(x2, self.fc1, self.fc2, self.fc3, self.non_linearity).reshape(x.shape)
            h1 = dense_layer(x2, self.fc1.weight, self.fc1.bias, self.non_linearity, mode=self._mode())
            return self._tail(h1).reshape(x.shape)
        act = {"relu": torch.relu, "tanh": torch.tanh, "softplus": torch.nn.functional.softplus}[self.non_linearity]
        return self.fc3(act(self.fc2(act(self.fc1(x)))))


def _linear_image(A, sign):
    """``b2ode_linear_f64``'s shared-memory image of ``sign * A`` (include/b2ode.h): a permutation of A's entries, rebuilt
    only when A changes.  Negation is exact, so the image of -A gives bit for bit the negated product."""
    def build(a):
        D = a.shape[0]
        a = a if sign > 0 else -a
        # rows 16 c + 4 t + 2 h + e, columns 8 n + g  ->  [c][n][h][g][t][e]
        return a.reshape(D // 16, 4, 2, 2, D // 8, 8).permute(0, 4, 2, 5, 1, 3).contiguous()
    return _CACHE.get("linear+" if sign > 0 else "linear-", (A,), build)


def linear_f64(x, A, sign=1.0, stage=None):
    """``x @ (sign * A)`` on the fp64 tensor cores (``b2ode_linear_f64``): ``x`` a contiguous ``[M, D]`` fp64 CUDA tensor.
    ``stage`` as in :func:`dense_layer`: Y = x + sum_j (dt * coefs[j]) * k_tensors[j] is formed inside the kernel (and
    stored to ``ystage`` if given), then multiplied."""
    import ctypes as C
    M, D = x.shape
    out = torch.empty_like(x)
    karr, carr, nk, state, ys = _stage_args(stage)

    def ptr(t):
        return C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(_lib.lib.b2ode_linear_f64(ptr(x), karr, carr, nk, C.c_void_p(state) if state else None, ptr(ys),
                                         ptr(_linear_image(A, sign)), ptr(out), M, D,
                                         C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
    return out


class LinearODE(nn.Module):
    """The linear system ``y' = y @ A`` (the reference's test problem, tests/problems.py:43-68, batched over rows): ``A``
    is a ``(D, D)`` ``nn.Parameter`` and the state any ``(..., D)`` tensor, its leading axes flattened into rows.  For
    the column form ``y' = A y`` pass ``A.T``.  Counts ``nfe`` like :class:`DenseMLP`.

    Under ``torch.no_grad()`` -- which is how ``odeint`` evaluates ``func`` -- on a CUDA fp64 state with D a multiple of
    16 in [16, 128], the product runs on the fp64 tensor cores (``b2ode_linear_f64``), and the adaptive Runge-Kutta
    solvers form each stage input inside that kernel instead of writing it to HBM and reading it back.  Every evaluation
    of a solve then goes through the same kernel, so the fused and unfused paths give identical bits.  Other widths,
    fp32 states, CPU tensors and autograd-enabled calls (training, ``odeint_adjoint``'s VJPs) are plain torch."""

    def __init__(self, A, dtype=torch.float64):
        super(LinearODE, self).__init__()
        A = torch.as_tensor(A, dtype=dtype).detach().clone()
        if A.dim() != 2 or A.shape[0] != A.shape[1]:
            raise ValueError("A must be a square (D, D) matrix")
        self.dim = int(A.shape[0])
        self.A = nn.Parameter(A)
        self.nfe = 0

    def uses_tensor_cores(self, y):
        D = self.dim
        return (y.is_cuda and y.dtype == torch.float64 and self.A.dtype == torch.float64 and self.A.device == y.device
                and not torch.is_grad_enabled() and D % 16 == 0 and 16 <= D <= 128 and y.dim() >= 1
                and y.shape[-1] == D and y.numel() > 0)

    def invalidate_tensor_core_cache(self):
        _CACHE.invalidate(self.A)

    def forward_from_stage(self, y0, ks, coefs, state_ptr, ystage, sign=1.0):
        """``f`` at the stage input ``y0 + sum_j (dt * coefs[j]) * ks[j]`` (dt in the solver's device state), formed inside
        the kernel and also stored to ``ystage`` if given; ``sign = -1`` evaluates the reverse-time system
        ``-f(-t, y)``.  All tensors are contiguous fp64 CUDA tensors of the state's shape."""
        self.nfe += 1
        D = self.dim
        rows = [k.reshape(-1, D) for k in ks]
        ys = ystage.view(-1, D) if ystage is not None else None
        out = linear_f64(y0.reshape(-1, D), self.A, sign, stage=(rows, coefs, state_ptr, ys))
        return out.reshape(y0.shape)

    def forward(self, t, y):
        self.nfe += 1
        if self.uses_tensor_cores(y):
            y2 = y.reshape(-1, self.dim)
            if not y2.is_contiguous() or y2.data_ptr() % 16:
                # the kernel loads 16 bytes at a time; a view at an odd element offset is copied (same bits)
                y2 = y2.clone(memory_format=torch.contiguous_format)
            return linear_f64(y2, self.A).reshape(y.shape)
        return y @ self.A


class Conv2dODEFunc(_TensorCoreFunc):
    """The reference's ``Conv2dODEFunc`` (tfdiffeq/models/conv_odenet.py:45-143, BASELINE config 4): conv 1x1 -> act ->
    conv 3x3 'same' -> act -> conv 1x1 on an NHWC state ``(batch, height, width, channels)`` -- TensorFlow's default
    image layout, which is also what makes the 1x1 convolutions plain GEMMs over ``M = batch * height * width`` rows.

    Under ``torch.no_grad()`` on a CUDA fp32 state the two 1x1 convolutions run on the tensor cores (wgmma) through the
    same dense-layer kernel as :class:`DenseMLP` (``b2ode_dense_layer_x3`` / ``b2ode_dense_layer``), the first one fed
    straight from the Runge-Kutta stage combine; the 3x3 convolution stays on cuDNN (channels-last, no layout copies:
    the NHWC buffer *is* a channels-last NCHW tensor), with TF32 disabled in the accurate mode.  ``time_dependent=True``
    (conv_odenet.py:11-42: time appended as an extra input channel of every convolution) runs in plain torch.
    ``channels`` must be given up front (the reference builds conv3 lazily from the first input, :118-128)."""

    def __init__(self, num_filters, channels=None, time_dependent=False, non_linearity="relu", tensor_cores=True,
                 dtype=torch.float32):
        super(Conv2dODEFunc, self).__init__()
        if non_linearity not in ("relu", "tanh", "softplus"):
            raise ValueError("non_linearity must be relu, tanh or softplus")
        if tensor_cores not in _MODES:
            raise ValueError("tensor_cores must be True, False, '3xtf32' or 'tf32'")
        channels = num_filters if channels is None else channels
        self.num_filters, self.channels, self.time_dependent = int(num_filters), int(channels), bool(time_dependent)
        self.non_linearity, self.tensor_cores = non_linearity, tensor_cores
        extra = 1 if time_dependent else 0
        self.conv1 = nn.Conv2d(self.channels + extra, self.num_filters, 1, dtype=dtype)
        self.conv2 = nn.Conv2d(self.num_filters + extra, self.num_filters, 3, padding=1, dtype=dtype)
        self.conv3 = nn.Conv2d(self.num_filters + extra, self.channels, 1, dtype=dtype)
        self.nfe = 0

    def uses_tensor_cores(self, x):
        return (self._mode() is not None and not self.time_dependent and x.is_cuda and x.dtype == torch.float32
                and x.dim() == 4 and not torch.is_grad_enabled() and self.conv1.weight.dtype == torch.float32
                and self.channels % 16 == 0 and self.num_filters % 16 == 0 and x.shape[-1] == self.channels)

    def _act(self, v):
        return {"relu": torch.relu, "tanh": torch.tanh, "softplus": torch.nn.functional.softplus}[self.non_linearity](v)

    def _conv3x3(self, h):
        """h: NHWC contiguous -> NHWC contiguous; cuDNN channels-last, activation applied by the caller."""
        w = _CACHE.get("cl", (self.conv2.weight,), lambda w: w.contiguous(memory_format=torch.channels_last))
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=(self._mode() == "tf32")):
            o = torch.nn.functional.conv2d(h.permute(0, 3, 1, 2), w, self.conv2.bias, padding=1)
        o = o.permute(0, 2, 3, 1)
        return o if o.is_contiguous() else o.contiguous()

    def _tail(self, h1):
        m = self._mode()
        h2 = self._act(self._conv3x3(h1))
        return dense_layer(h2, self.conv3.weight, self.conv3.bias, "none", mode=m)

    def forward_from_stage(self, y0, ks, coefs, state_ptr, ystage):
        self.nfe += 1
        h1 = dense_layer(y0, self.conv1.weight, self.conv1.bias, self.non_linearity, stage=(ks, coefs, state_ptr, ystage),
                         mode=self._mode())
        return self._tail(h1)

    def forward(self, t, x):
        self.nfe += 1
        if self.uses_tensor_cores(x):
            xc = x if x.is_contiguous() else x.contiguous()
            h1 = dense_layer(xc, self.conv1.weight, self.conv1.bias, self.non_linearity, mode=self._mode())
            return self._tail(h1)
        v = x.permute(0, 3, 1, 2)

        def tcat(u):
            if not self.time_dependent:
                return u
            tt = torch.ones_like(u[:, :1]) * t.to(u.dtype)                      # conv_odenet.py:30-40
            return torch.cat([tt, u], 1)
        out = self._act(self.conv1(tcat(v)))
        out = self._act(self.conv2(tcat(out)))
        out = self.conv3(tcat(out))
        return out.permute(0, 2, 3, 1)
