"""Multistep solvers behind the reference's solver protocol (SURVEY.md 8f-4):

* ``AdamsBashforthMoulton`` / ``AdamsBashforth``  -- tfdiffeq/fixed_adams.py:168-212 (``fixed_adams``, ``explicit_adams``)
* ``VariableCoefficientAdamsBashforth``            -- tfdiffeq/adams.py:22-211 (``adams``)

The step logic (derivative history, functional iteration, order selection, step-size control) is host code, as it
is in the reference; every tensor operation is a ``libb2ode`` launch -- ``b2ode_lincomb`` for the linear
combinations of stored derivatives, ``b2ode_reduce`` for the error norms and the convergence test, the fixed-grid
ops for the Runge-Kutta start-up steps and the output interpolation.  Host scalars are read back where the
reference's Python control flow reads them (once per functional iteration / per attempted step).
"""
import collections
import ctypes as C
import math
import sys
from fractions import Fraction

import numpy as np
import torch

from . import _lib
from .misc import _assert_increasing, _handle_unused_kwargs, _is_iterable, _tf_f64
from .solvers import FixedGridODESolver, _DT, _FuncOutputs, _Segments, _ptr_array, last_stats

_MAX_TERMS = 16


# ---- Adams coefficients as exact rationals -------------------------------------------------------------------------
def _poly_mul(a, b):
    out = [Fraction(0)] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            out[i + j] += x * y
    return out


_WEIGHT_CACHE = {}


def adams_weights(k, implicit):
    """(integer numerators, common divisor) of the k-point Adams-Bashforth (``implicit=False``: nodes t_n, t_n-1, ...)
    or Adams-Moulton (``implicit=True``: nodes t_n+1, t_n, ...) formula: the integral over one step of the Lagrange
    basis on those nodes.  Equal to the tables at tfdiffeq/fixed_adams.py:7-160 (checked in tests/test_lib_cpu.py)."""
    key = (k, bool(implicit))
    if key not in _WEIGHT_CACHE:
        nodes = [Fraction((1 if implicit else 0) - j) for j in range(k)]
        w = []
        for j in range(k):
            poly, den = [Fraction(1)], Fraction(1)
            for i in range(k):
                if i != j:
                    poly = _poly_mul(poly, [-nodes[i], Fraction(1)])
                    den *= nodes[j] - nodes[i]
            w.append(sum(c / (p + 1) for p, c in enumerate(poly)) / den)
        div = 1
        for x in w:
            div = div * x.denominator // math.gcd(div, x.denominator)
        _WEIGHT_CACHE[key] = ([int(x * div) for x in w], div)
    return _WEIGHT_CACHE[key]


# ---- thin wrappers over the two kernels ----------------------------------------------------------------------------
class _FlatPtrs(object):
    """A ready-made per-segment pointer array (e.g. a row of the output slab) where _Ops expects a buffer."""

    def __init__(self, arr):
        self.arr = arr


class _Ops(object):
    def __init__(self, seg):
        self.seg = seg
        self.dcode = _DT[seg.dtype]
        self.lens = _lib.LenArray(*seg.lens)
        self.sm = torch.cuda.get_device_properties(seg.device).multi_processor_count
        self.stream = torch.cuda.current_stream(seg.device)
        self.sptr = C.c_void_p(self.stream.cuda_stream)
        self.npdt = np.float32 if seg.dtype == torch.float32 else np.float64
        ws = int(_lib.lib.b2ode_reduce_workspace_bytes(self.sm))
        self.ws = torch.zeros(ws, dtype=torch.uint8, device=seg.device)
        self.red_out = torch.zeros(2 * _lib.MAXSEG, dtype=torch.float64, device=seg.device)
        self.launches = 0

    def ptrs(self, x):
        """x: engine flat buffer, a _FlatPtrs, or a list of per-segment tensors (func outputs)."""
        if isinstance(x, _FlatPtrs):
            return [x.arr[s] for s in range(self.seg.nseg)]
        if isinstance(x, torch.Tensor):
            return self.seg.ptrs(x)
        return [t.data_ptr() for t in x]

    def lincomb(self, out, base, scale, terms, coefs):
        """out = base + scale * sum coefs[j] * terms[j]  (state dtype, left to right)."""
        n = len(terms)
        assert 1 <= n <= _MAX_TERMS
        nseg = self.seg.nseg
        xs = (C.c_void_p * (n * nseg))()
        for j, tm in enumerate(terms):
            for s, p in enumerate(self.ptrs(tm)):
                xs[j * nseg + s] = p
        cf = (C.c_double * n)(*[float(c) for c in coefs])
        _lib.check(_lib.lib.b2ode_lincomb(self.dcode, nseg, self.lens, _ptr_array(self.ptrs(out)),
                                          _ptr_array(self.ptrs(base)) if base is not None else None, float(scale), n, xs, cf,
                                          self.sm, self.sptr))
        self.launches += 1

    def reduce(self, mode, a, b=None, p0=None, p1=None):
        nseg = self.seg.nseg
        arr = lambda v: (C.c_double * _lib.MAXSEG)(*([float(x) for x in v] + [0.0] * (_lib.MAXSEG - len(v))))   # noqa: E731
        _lib.check(_lib.lib.b2ode_reduce(self.dcode, mode, nseg, self.lens, _ptr_array(self.ptrs(a)),
                                         _ptr_array(self.ptrs(b)) if b is not None else None,
                                         arr(p0) if p0 is not None else None, arr(p1) if p1 is not None else None,
                                         C.c_void_p(self.red_out.data_ptr()), C.c_void_p(self.ws.data_ptr()), self.ws.numel(),
                                         self.sm, self.sptr))
        self.launches += 1
        return self.red_out[:2 * nseg].cpu().numpy().reshape(nseg, 2)           # the host decision point


# =====================================================================================================================
# fixed grid: Adams-Bashforth(-Moulton)
# =====================================================================================================================
class AdamsBashforthMoulton(FixedGridODESolver):
    """tfdiffeq/fixed_adams.py:168-212.  Quirks kept: orders below 4 are 3/8-rule Runge-Kutta steps that reuse the
    stored derivative as k1 (:188-191); the corrector's own derivative is never stored (:211 is a no-op because
    ``prev_t == t`` by then); a functional iteration that does not converge prints the reference's warning and drops
    the OLDEST stored derivative (:207-210)."""

    method, order = "adams", 4
    _MIN_ORDER, _MAX_ORDER, _MAX_ITERS = 4, 12, 4

    def __init__(self, func, y0, rtol=1e-3, atol=1e-4, implicit=True, max_iters=_MAX_ITERS, max_order=_MAX_ORDER, **kwargs):
        if kwargs.pop('independent_rows', False):
            raise ValueError("independent_rows is not supported by the multistep solvers")
        super(AdamsBashforthMoulton, self).__init__(func, y0, **kwargs)
        self.rtol, self.atol = rtol, atol
        self.implicit = implicit
        self.max_iters = max_iters
        self.max_order = int(min(max_order, self._MAX_ORDER))

    def _integrate(self, t, seg):
        lib, check = _lib.lib, _lib.check
        dev, dtype = seg.device, seg.dtype
        ops = _Ops(seg)
        npdt = ops.npdt
        t = t.to(dtype)                                                        # solvers.py:84
        time_grid = self.grid_constructor(self.func, self.y0, t)
        t_np = t.detach().cpu().numpy().astype(npdt)
        g_np = time_grid.detach().cpu().numpy().astype(npdt)
        assert g_np[0] == t_np[0] and g_np[-1] == t_np[-1]                     # solvers.py:86
        n_out, n_steps = int(t_np.shape[0]), int(g_np.shape[0]) - 1
        outs = [torch.empty((n_out,) + shp, dtype=dtype, device=dev) for shp in seg.shapes]
        for o, y in zip(outs, self.y0):
            o[0].copy_(y)
        item, nseg = seg.item, seg.nseg

        def fixed_op(code, out_p, y_p, a, b=None, c=None, d=None, dt=0.0, s1=0.0, s2=0.0):
            check(lib.b2ode_fixed_op(ops.dcode, code, nseg, ops.lens, out_p, y_p, a, b, c, d, float(dt), float(s1), float(s2),
                                     ops.sm, ops.sptr))

        def row_ptrs(j):
            return _ptr_array([o.data_ptr() + j * n * item for o, n in zip(outs, seg.lens)])

        # engine-owned storage: the derivative history (copies -- func may reuse its output storage), the stage /
        # corrector input, two dy buffers, delta, and two y1 scratch states for cells that do not end on an output
        depth = max(self.max_order - 1, 1)
        pool = [seg.new() for _ in range(depth + 1)]
        hist = collections.deque()                                             # newest first, at most `depth` entries
        S, DYa, DYb, DELTA, Y1a, Y1b = (seg.new() for _ in range(6))
        fo = _FuncOutputs(seg, tuple(pool) + (S, DYa, DYb, DELTA, Y1a, Y1b) + tuple(outs))
        s_views, s_ptrs = seg.views(S), _ptr_array(seg.ptrs(S))
        scratch = [(seg.views(Y1a), Y1a), (seg.views(Y1b), Y1b)]
        times_dev = torch.from_numpy(np.ascontiguousarray(np.stack(
            [g_np[:-1], g_np[:-1] + (g_np[1:] - g_np[:-1]) / npdt(3), g_np[:-1] + (g_np[1:] - g_np[:-1]) * npdt(2) / npdt(3),
             g_np[:-1] + (g_np[1:] - g_np[:-1])], 1).astype(npdt))).to(dev) if n_steps else None

        func = self.func
        y_p, y_views = row_ptrs(0), tuple(o[0] for o in outs)
        j, nfe, flip, not_converged = 1, 0, 0, 0
        prev_t = None
        for i in range(n_steps):
            t0, t1 = g_np[i], g_np[i + 1]
            dt = npdt(t1 - t0)
            j_hi = j
            while j_hi < n_out and t1 >= t_np[j_hi]:                           # solvers.py:97
                j_hi += 1
            ends_on_output = j_hi > j and t_np[j_hi - 1] == t1
            if ends_on_output:
                y1_p, y1_views = row_ptrs(j_hi - 1), tuple(o[j_hi - 1] for o in outs)
            else:
                y1_views, y1_flat = scratch[flip]
                y1_p = _ptr_array(seg.ptrs(y1_flat))
                flip ^= 1
            tv = times_dev[i]

            # ---- step_func (fixed_adams.py:187-212) -------------------------------------------------------------------
            f_now = fo.collect(func(tv[0], y_views), set())
            nfe += 1
            if prev_t is None or prev_t != t0:                                 # _update_history
                buf = pool.pop() if len(hist) < depth else hist.pop()
                ops.lincomb(buf, None, 1.0, [f_now], [1.0])                    # private copy of the derivative
                hist.appendleft(buf)
                prev_t = t0
            del f_now
            order = min(len(hist), self.max_order - 1)
            if order < self._MIN_ORDER - 1:
                # rk4_alt_step_func(func, t, dt, y, k1=prev_f[0])  (rk_common.py:73-81)
                p1 = _ptr_array(seg.ptrs(hist[0]))
                live = set()
                fixed_op(_lib.OP_RK4_S2, s_ptrs, y_p, p1, dt=dt)
                k2 = [x.clone() for x in fo.collect(func(tv[1], s_views), live)]
                p2 = _ptr_array([x.data_ptr() for x in k2])
                fixed_op(_lib.OP_RK4_S3, s_ptrs, y_p, p1, p2, dt=dt)
                k3 = [x.clone() for x in fo.collect(func(tv[2], s_views), live)]
                p3 = _ptr_array([x.data_ptr() for x in k3])
                fixed_op(_lib.OP_RK4_S4, s_ptrs, y_p, p1, p2, p3, dt=dt)
                k4 = fo.collect(func(tv[3], s_views), live)
                p4 = _ptr_array([x.data_ptr() for x in k4])
                fixed_op(_lib.OP_RK4_FINAL, y1_p, y_p, p1, p2, p3, p4, dt=dt)
                nfe += 3
                del k2, k3, k4
            else:
                ab, ab_div = adams_weights(order, False)
                terms = [hist[q] for q in range(order)]
                ab_coef = [(1 / ab_div) * c for c in ab]                       # misc.py:121 (scale * x), python floats
                if not self.implicit:
                    ops.lincomb(_FlatPtrs(y1_p), _FlatPtrs(y_p), dt, terms, ab_coef)          # y + dt * sum
                else:
                    am, am_div = adams_weights(order + 1, True)
                    dy, dy_other = DYa, DYb
                    ops.lincomb(dy, None, dt, terms, ab_coef)                                 # Bashforth predictor
                    ops.lincomb(DELTA, None, dt, terms, [(1 / am_div) * c for c in am[1:]])
                    c0 = npdt(dt * npdt(am[0] / am_div))                                      # dt * (m0 / div) in the state dtype
                    converged = False
                    for _ in range(self.max_iters):
                        ops.lincomb(S, _FlatPtrs(y_p), 1.0, [dy], [1.0])                      # y + dy
                        f = fo.collect(func(tv[3], s_views), set())
                        nfe += 1
                        ops.lincomb(dy_other, DELTA, 1.0, [f], [c0])                          # dt*(m0/div)*f + delta
                        del f
                        bad = ops.reduce(_lib.RED_NOT_CONVERGED, dy, dy_other, [self.rtol] * nseg, [self.atol] * nseg)
                        dy, dy_other = dy_other, dy
                        converged = not bool(bad[:, 0].sum() > 0)
                        if converged:
                            break
                    if not converged:
                        print('Warning: Functional iteration did not converge. Solution may be incorrect.', file=sys.stderr)
                        not_converged += 1
                        pool.append(hist.pop())
                    ops.lincomb(_FlatPtrs(y1_p), _FlatPtrs(y_p), 1.0, [dy], [1.0])           # y1 = y + dy (solvers.py:95)
            # ---- outputs inside this cell: linear interpolation (solvers.py:106-115) ------------------------------------
            for jj in range(j, j_hi - (1 if ends_on_output else 0)):
                fixed_op(_lib.OP_LERP, row_ptrs(jj), y_p, y1_p, s1=npdt(t1) - npdt(t0), s2=npdt(t_np[jj]) - npdt(t0))
            j = j_hi
            y_p, y_views = y1_p, y1_views
        self.stats = dict(n_accepted=n_steps, n_rejected=0, nfe=nfe, status=0, fused_rhs=False, not_converged=not_converged)
        last_stats.clear()
        last_stats.update(self.stats)
        ops.stream.synchronize()
        return tuple(outs)


class AdamsBashforth(AdamsBashforthMoulton):
    """tfdiffeq/fixed_adams.py:209-212"""

    def __init__(self, func, y0, **kwargs):
        super(AdamsBashforth, self).__init__(func, y0, implicit=False, **kwargs)


# =====================================================================================================================
# adaptive: variable-coefficient Adams-Bashforth-Moulton
# =====================================================================================================================
_GAMMA_STAR = [1, -1 / 2, -1 / 12, -1 / 24, -19 / 720, -3 / 160, -863 / 60480, -275 / 24192, -33953 / 3628800, -0.00789255,
               -0.00678585, -0.00592406, -0.00523669, -0.0046775, -0.00421495, -0.0038269]          # adams.py:16-19


def _optimal_step_size(last_step, error_ratio, safety, ifactor, dfactor, order):
    """tfdiffeq/misc.py:267-287 on host scalars (float64; the exponent is rounded through float32, :281-282)."""
    vals = [float(v) for v in error_ratio]
    m = float("nan") if any(v != v for v in vals) else max(vals)
    if m == 0:
        return last_step * ifactor
    if m < 1:
        dfactor = 1.0
    exponent = float(np.float64(np.float32(1.0 / order)))
    with np.errstate(all="ignore"):
        cand = np.float64(np.sqrt(np.float64(m))) ** np.float64(exponent) / np.float64(safety)
    if cand != cand:
        return last_step / float(cand)
    factor = max(1.0 / ifactor, min(float(cand), 1.0 / dfactor))
    return last_step / factor


class VariableCoefficientAdamsBashforth(object):
    """tfdiffeq/adams.py:79-211 (Hairer, Norsett & Wanner III.5), orders 1..12, behind solvers.py:10-35's protocol.

    Quirks kept: g lives in a float32 variable (:34); ``first_step`` is ignored (:112-115); the predictor uses
    ``max(1, order-1)`` terms (:144-147); the state carried forward is the PREDICTOR (:211); a reject keeps the order."""

    _MIN_ORDER, _MAX_ORDER = 1, 12

    def __init__(self, func, y0, rtol, atol, implicit=True, first_step=None, max_order=_MAX_ORDER, safety=0.9, ifactor=10.0,
                 dfactor=0.2, **unused_kwargs):
        unused_kwargs.pop('shared_step_group', None)
        unused_kwargs.pop('replicated_components', None)
        unused_kwargs.pop('host_output', None)       # (only the Runge-Kutta drivers deliver to host buffers)
        unused_kwargs.pop('cuda_graph', None)
        unused_kwargs.pop('fused_rhs', None)
        if unused_kwargs.pop('independent_rows', False):
            raise ValueError("independent_rows is not supported by the multistep solvers")
        _handle_unused_kwargs(self, unused_kwargs)
        del unused_kwargs
        self.func = func
        self.y0 = y0
        self.rtol = list(rtol) if _is_iterable(rtol) else [rtol] * len(y0)
        self.atol = list(atol) if _is_iterable(atol) else [atol] * len(y0)
        self.implicit = implicit
        self.first_step = first_step
        self.max_order = int(max(self._MIN_ORDER, min(max_order, self._MAX_ORDER)))
        self.safety, self.ifactor, self.dfactor = _tf_f64(safety), _tf_f64(ifactor), _tf_f64(dfactor)
        self.stats = {}

    def integrate(self, t):
        _assert_increasing(t)
        seg = _Segments(self.y0)
        with torch.cuda.device(seg.device), torch.no_grad():
            return self._integrate(t, seg)

    # -- `_select_initial_step(func, t0, y0, 2, rtol[0], atol[0], f0)` through the adaptive solver's native path ------
    def _initial_step(self, seg, ops, Y, F0, S, t0, fo, outs, t_dev):
        lib, check = _lib.lib, _lib.check
        d = _lib.AdaptiveDesc()
        d.dtype, d.nseg = ops.dcode, seg.nseg
        for i, n in enumerate(seg.lens):
            d.seg_len[i] = n
            d.rtol[i], d.atol[i] = float(self.rtol[i]), float(self.atol[i])
        d.n_k, d.fsal = 2, 0
        d.alpha[0] = 1.0
        d.beta[0][0] = 1.0
        d.c_sol[0], d.c_sol[1] = 0.5, 0.5
        d.c_error[0], d.c_error[1] = 0.5, -0.5
        d.dense_kind, d.controller = 0, _lib.CTRL_REFERENCE
        d.safety, d.ifactor, d.dfactor = self.safety, self.ifactor, self.dfactor
        d.exponent, d.max_num_steps, d.init_order, d.sm_count = 0.5, 1, 2, ops.sm      # adams.py:113: order 2
        tstage = torch.zeros(2, dtype=seg.dtype, device=seg.device)
        state_dev = torch.zeros(256, dtype=torch.uint8, device=seg.device)
        workspace = torch.empty(max(int(lib.b2ode_workspace_bytes(C.byref(d))), 32), dtype=torch.uint8, device=seg.device)
        handle = C.c_void_p()
        check(lib.b2ode_adaptive_create(C.byref(handle), C.byref(d)))
        try:
            buf = _lib.AdaptiveBuffers()
            buf.state, buf.workspace, buf.workspace_bytes = state_dev.data_ptr(), workspace.data_ptr(), workspace.numel()
            for i, (a, b, c) in enumerate(zip(seg.ptrs(Y), seg.ptrs(F0), seg.ptrs(S))):
                buf.y0[i], buf.f0[i], buf.ystage[i] = a, b, c
                buf.out[i] = outs[i].data_ptr()
            buf.tstage, buf.t_out, buf.n_out = tstage.data_ptr(), t_dev.data_ptr(), int(t_dev.numel())
            check(lib.b2ode_adaptive_bind(handle, C.byref(buf), ops.sptr))
            check(lib.b2ode_adaptive_init(handle, float(t0), float("nan")))
            check(lib.b2ode_initial_step_probe(handle))
            f1 = fo.collect(self.func(tstage[0], seg.views(S)), set())
            check(lib.b2ode_initial_step_finish(handle, fo.pointers(f1)))
            pinned = torch.empty(256, dtype=torch.uint8).pin_memory()
            check(lib.b2ode_poll_sync(handle, C.c_void_p(pinned.data_ptr())))
            st = _lib.State.from_buffer_copy(_lib.State.from_address(pinned.data_ptr()))
            return float(st.dt)
        finally:
            lib.b2ode_adaptive_destroy(handle)

    def _integrate(self, t, seg):
        dev, dtype = seg.device, seg.dtype
        ops = _Ops(seg)
        npdt = ops.npdt
        nseg = seg.nseg
        t_host = t.detach().to("cpu", torch.float64).numpy()                  # solvers.py:30
        t_dev = torch.from_numpy(t_host).to(dev)
        n_out = int(t_host.shape[0])
        outs = [torch.empty((n_out,) + shp, dtype=dtype, device=dev) for shp in seg.shapes]
        func = self.func
        numel = [max(n, 1) for n in seg.lens]

        Y, F0, S = seg.new(), seg.new(), seg.new()
        fo = _FuncOutputs(seg, (Y, F0, S))
        seg.fill(Y, self.y0)
        for o, y in zip(outs, self.y0):
            o[0].copy_(y)
        nfe = n_acc = n_rej = 0

        def tcast(x):       # tf.cast(t, y.dtype): the time handed to func
            return torch.tensor(float(npdt(x)), dtype=dtype, device=dev)

        def feval(tt, flat):
            """func at time tt on an engine buffer; the result is copied into a fresh engine buffer."""
            f = fo.collect(func(tcast(tt), seg.views(flat)), set())
            out = seg.new()
            ops.lincomb(out, None, 1.0, [f], [1.0])
            return out

        # ---- before_integrate (adams.py:100-118) ----------------------------------------------------------------------
        f0 = feval(t_host[0], Y)
        nfe += 1
        F0.copy_(f0)
        first_step = self._initial_step(seg, ops, Y, F0, S, t_host[0], fo, outs, t_dev)       # first_step option ignored (:112-115)
        nfe += 1
        prev_t = collections.deque([float(t_host[0])], maxlen=self.max_order + 1)
        phi = [f0]
        y_n, next_t, order = Y, float(t_host[0]) + first_step, 1

        def err_ratio(coef, x, tol):
            r = ops.reduce(_lib.RED_RATIO_SUMSQ, x, None, [coef] * nseg, tol)
            return [float(npdt(r[s, 0] / numel[s])) for s in range(nseg)]

        for i in range(1, n_out):
            final_t = float(t_host[i])
            while final_t > prev_t[0]:                                        # adams.py:123-126
                # ---- _adaptive_adams_step (adams.py:128-211) ----------------------------------------------------------
                if next_t > final_t:
                    next_t = final_t
                dt = next_t - prev_t[0]
                if not math.isfinite(dt):
                    # the reference spins forever here (`final_t > prev_t[0]` never changes once dt is NaN)
                    raise AssertionError('non-finite values in state `y` or step size: {}'.format(dt))
                dtc = npdt(dt)
                # g_and_explicit_phi (adams.py:29-59): g in float32, c and beta in float64
                k = order
                g32 = np.zeros(k + 1, dtype=np.float32)
                g32[0] = 1
                c = 1.0 / np.arange(1, k + 2).astype(np.float64)
                ephi = [phi[0]]
                beta = np.float64(1.0)
                with np.errstate(all="ignore"):
                    for q in range(1, k):
                        beta = (np.float64(next_t) - prev_t[q - 1]) / (np.float64(prev_t[0]) - prev_t[q]) * beta
                        e = seg.new()
                        ops.lincomb(e, None, 1.0, [phi[q]], [float(npdt(beta))])
                        ephi.append(e)
                        c = c[:-1] - c[1:] if q == 1 else c[:-1] - c[1:] * dt / (np.float64(next_t) - prev_t[q - 1])
                        g32[q] = np.float32(c[0])
                    c = c[:-1] - c[1:] * dt / (np.float64(next_t) - prev_t[k - 1])
                    g32[k] = np.float32(c[0])
                g = g32.astype(npdt)
                # predictor (adams.py:144-147)
                m = max(1, order - 1)
                p_next = seg.new()
                ops.lincomb(p_next, y_n, 1.0, ephi[:m], [float(dtc * g[q]) for q in range(m)])
                f_p = feval(next_t, p_next)
                nfe += 1
                # implicit phi with the predictor's derivative (adams.py:62-77, k = order + 1)
                iphi_p = [f_p]
                for q in range(1, min(len(ephi) + 1, order + 1)):
                    d_ = seg.new()
                    ops.lincomb(d_, iphi_p[q - 1], 1.0, [ephi[q - 1]], [-1.0])
                    iphi_p.append(d_)
                # corrector (adams.py:154-157)
                y_next = seg.new()
                ops.lincomb(y_next, p_next, 1.0, [iphi_p[order - 1]], [float(dtc * g[order - 1])])
                # error estimate (adams.py:160-167)
                mx = ops.reduce(_lib.RED_ABSMAX2, y_n, y_next)
                tol = []
                for s_ in range(nseg):
                    a0, a1 = mx[s_, 0], mx[s_, 1]
                    mm = float("nan") if (a0 != a0 or a1 != a1) else max(a0, a1)
                    tol.append(float(npdt(self.atol[s_]) + npdt(self.rtol[s_]) * npdt(mm)))
                error_k = err_ratio(float(dtc * (g[order] - g[order - 1])), iphi_p[order], tol)
                accept = all(e <= 1 for e in error_k)
                if not accept:
                    n_rej += 1
                    dt_next = _optimal_step_size(dt, error_k, self.safety, self.ifactor, self.dfactor, order)
                    next_t = prev_t[0] + dt_next                               # :172 same phi, same order
                    continue
                n_acc += 1
                f_c = feval(next_t, y_next)
                nfe += 1
                implicit_phi = [f_c]
                for q in range(1, min(len(ephi) + 1, order + 2)):
                    d_ = seg.new()
                    ops.lincomb(d_, implicit_phi[q - 1], 1.0, [ephi[q - 1]], [-1.0])
                    implicit_phi.append(d_)
                next_order = order
                if len(prev_t) <= 4 or order < 3:                              # :182-183
                    next_order = min(order + 1, 3, self.max_order)
                else:
                    e1 = err_ratio(float(dtc * (g[order - 1] - g[order - 2])), iphi_p[order - 1], tol)
                    e2 = err_ratio(float(dtc * (g[order - 2] - g[order - 3])), iphi_p[order - 2], tol)
                    if min(e1 + e2) < max(error_k):
                        next_order = order - 1
                    elif order < self.max_order:
                        ep = err_ratio(float(dtc * npdt(_GAMMA_STAR[order])), iphi_p[order], tol)
                        if max(ep) < max(error_k):
                            next_order = order + 1
                dt_next = dt if next_order > order else _optimal_step_size(dt, error_k, self.safety, self.ifactor,
                                                                            self.dfactor, order + 1)
                prev_t.appendleft(next_t)
                y_n, phi, order = p_next, implicit_phi, next_order             # :211 the predictor is carried on
                next_t = next_t + dt_next
            assert final_t == prev_t[0]
            seg_views = seg.views(y_n)
            for o, v in zip(outs, seg_views):
                o[i].copy_(v)
        self.stats = dict(n_accepted=n_acc, n_rejected=n_rej, nfe=nfe, status=0, fused_rhs=False, cuda_graph=False)
        last_stats.clear()
        last_stats.update(self.stats)
        ops.stream.synchronize()
        return tuple(outs)
