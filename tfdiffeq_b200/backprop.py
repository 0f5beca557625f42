"""``odeint(..., options={'backprop': True})``: reverse-mode gradients of the discrete solve.

The forward solve records, for every accepted step n, its start state y_n (one checkpoint slot of N elements), its
schedule (t_n, dt_n, the outputs it emitted) and the times at which its k's were evaluated; the backward pass walks the
accepted steps in reverse with that schedule held constant:

* recompute the stage inputs Y_i = y_n + sum_j (dt_n beta_ij) k_j with ``b2ode_bp_combine`` (the forward stage kernels'
  operation order; the fixed-grid rk4 with ``b2ode_fixed_op``'s OP_RK4_S2..S4, as its forward formed them) and
  k_{i+1} = func(tau_i, Y_i), once per stage, keeping each call's autograd graph;
* carry the cotangents of the step's outputs into y_n, y_{n+1} and the k's (``b2ode_bp_dense``: the quartic dense output
  of the adaptive tableaus, the linear interpolation of the fixed grid);
* sweep the stages backwards: mu_{i+1} = (dense) + sum_{l > i} (dt beta_{l,i+1}) nu_l + (dt b_{i+1} or beta_{s-2,i+1})
  lambda_{n+1} (``b2ode_bp_combine``), nu_i = J(tau_i, Y_i)^T mu_{i+1} (torch autograd of func, parameter cotangents
  included), lambda_n = (dense) + sum nu_i + lambda_{n+1} (+ J^T mu_0 when f0 is an evaluation at y_n).

A built-in right-hand side (rhs.Lorenz, LotkaVolterra, Kepler, CubicMLP, LatentODEFunc) takes neither forward nor
autograd: its k's and vector-Jacobian products come from ``b2ode_bp_rhs``, which rebuilds Y_i in registers and, for a
trainable CubicMLP or LatentODEFunc, sums the parameter cotangents in fp64 in a fixed order.

f0 of step n: for FSAL tableaus and the fixed grid it is an evaluation at y_n (for FSAL at the previous step's last
stage time t_{n-1} + dt_{n-1}, not at t_n); for adaptive Heun (no FSAL) it is the previous step's last k, whose
cotangent is carried into that step.  The step size controller, the initial step, the interpolation abscissae and the
rejected attempts are constants of the schedule: they contribute nothing.

With ``independent_rows`` (a built-in right-hand side, an adaptive method) every row has its own schedule.  The forward
solve is k_rows_adaptive's recording variant (``b2ode_rows_solve_record``): each row writes, per accepted step, y_n,
(t_n, dt_n) in float64 and, for adaptive Heun, f0 -- slot-major, into a record of ROWS_INITIAL_SLOTS slots per row (fewer
when that would exceed ROWS_INITIAL_BYTES); if a row accepted more steps the forward runs once more with exactly
max(row steps) slots.  The backward pass is one launch of ``b2ode_rows_bp``: one thread per row runs the sweep above
over its own steps in registers, so row r's gradient is that of the shared-step path on row r alone, bit for bit, and a
trainable CubicMLP's or LatentODEFunc's weight gradients are the sum over rows (fp64, fixed order) of the per-row ones.
"""
import ctypes as C

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib
from . import rhs as _rhs
from . import solvers as _solvers

_ADAPTIVE = ("dopri5", "bosh3", "adaptive_heun", "dopri8")
_FIXED = ("euler", "midpoint", "rk4", "heun", "huen")
_REFUSED_KEYS = ("shared_step_group", "cuda_graph", "host_output")

# initial record of an independent-rows solve: slots per row, and the most bytes it may take (at least one slot per row)
ROWS_INITIAL_SLOTS = 256
ROWS_INITIAL_BYTES = 1 << 30

# the fixed-grid methods as stage recipes: Y_i = y + sum_j (dt beta_ij) k_j, y1 = y + sum_j (dt b_j) k_j
_FIXED_TAB = {
    "euler": ((), (1.0,)),
    "midpoint": (((0.5,),), (0.0, 1.0)),
    "heun": (((1.0,),), (0.5, 0.5)),
    "rk4": (((1.0 / 3.0,), (-1.0 / 3.0, 1.0), (1.0, -1.0, 1.0)), (0.125, 0.375, 0.375, 0.125)),
}

_STEP = C.sizeof(_lib.BpStep)

# statistics of the most recent backward pass
last_stats = {}


def check_options(method, options, t):
    """Raise ValueError for everything options={'backprop': True} does not support; returns the options without the key."""
    m = "dopri5" if method is None else method
    if m == "tsit5":
        raise ValueError("backprop: tsit5's dense output is k-based and not supported; use dopri5, bosh3, adaptive_heun, "
                         "dopri8 or a fixed-grid method")
    if m not in _ADAPTIVE + _FIXED:
        raise ValueError("backprop supports %s, got %r" % (", ".join(_ADAPTIVE + _FIXED), m))
    for key in _REFUSED_KEYS:
        v = options.get(key)
        if v is not None and v is not False:
            raise ValueError("backprop cannot be combined with %s" % key)
    if isinstance(t, torch.Tensor) and t.requires_grad:
        raise ValueError("backprop holds t constant; for gradients with respect to t use odeint_adjoint")
    # the rows of a fixed grid are independent already: the flag is dropped, as odeint drops it without backprop
    drop = ("backprop", "independent_rows") if m in _FIXED else ("backprop",)
    return {k: v for k, v in options.items() if k not in drop}


def check_rows(func, options):
    """independent_rows with backprop differentiates built-in right-hand sides only (b2ode_rows_bp)."""
    if options.get("independent_rows") and not isinstance(func, _rhs.BuiltinRHS):
        raise ValueError("backprop with independent_rows needs a built-in right-hand side (tfdiffeq_b200.rhs)")


def check_builtin(func, options):
    """A built-in right-hand side differentiated by the kernels (b2ode_bp_rhs): its trainable parameters must be ones
    the kernels know -- all four weights of a CubicMLP, all six of a LatentODEFunc, or none."""
    if not isinstance(func, _rhs.BuiltinRHS) or options.get("fused_rhs", True) is False:
        return
    params = list(func.parameters())
    if func.trainable_weights is not None:
        count, names = func.trainable_weights
        if not _rhs.weights_all_or_none(func):
            raise ValueError("backprop differentiates a %s whose %s weights (%s) are all trainable or all frozen, and no "
                             "other parameters; use fused_rhs=False for anything else"
                             % (type(func).__name__, count, ", ".join(names)))
    elif any(p.requires_grad for p in params):
        raise ValueError("backprop: %s has trainable parameters the kernels do not know; use fused_rhs=False"
                         % type(func).__name__)


def _trainable(func):
    return tuple(p for p in func.parameters() if p.requires_grad) if isinstance(func, nn.Module) else ()


def needs_grad(func, y0):
    if not torch.is_grad_enabled():
        return False
    ys = (y0,) if isinstance(y0, torch.Tensor) else tuple(y0)
    return any(y.requires_grad for y in ys) or len(_trainable(func)) > 0


class Record(object):
    """What the forward solve leaves for the backward pass.  Device memory: (steps + 1) N state elements of checkpoints
    (twice that for adaptive Heun, whose f0 is not a function of y_n), a 40-byte log entry and n_k stage times per step."""

    def __init__(self):
        self.fixed = False
        self.n_steps = 0
        self.builtin = None       # the built-in right-hand side the forward evaluated in the stage kernels, if any

    # ---- adaptive driver -----------------------------------------------------------------------
    def start_adaptive(self, seg, tab, t0_state):
        self.seg, self.tab, self.nk, self.fsal = seg, tab, tab.n_k, tab.fsal
        self.beta, self.c_sol = tab.beta, tab.c_sol
        self.cap = 0
        self.ckpt = self.ckpt_f0 = self.log = self.tau = None
        self._grow(16)
        self.tau[0, 0] = t0_state

    def _grow(self, need):
        cap = max(need, 2 * self.cap)
        seg = self.seg
        ckpt = torch.empty((cap, seg.total), dtype=seg.dtype, device=seg.device)
        f0 = None if self.fsal else torch.empty((cap, seg.total), dtype=seg.dtype, device=seg.device)
        log = torch.zeros((cap, _STEP), dtype=torch.uint8, device=seg.device)
        tau = torch.zeros((cap + 1, self.nk), dtype=seg.dtype, device=seg.device)
        if self.cap:
            # stream-ordered behind every record launch so far: no host synchronisation
            ckpt[:self.cap].copy_(self.ckpt)
            log[:self.cap].copy_(self.log)
            tau[:self.cap + 1].copy_(self.tau)
            if f0 is not None:
                f0[:self.cap].copy_(self.ckpt_f0)
        self.ckpt, self.ckpt_f0, self.log, self.tau, self.cap = ckpt, f0, log, tau, cap
        d = _lib.BpRecordDesc()
        d.ckpt = ckpt.data_ptr()
        d.ckpt_f0 = f0.data_ptr() if f0 is not None else None
        d.slot_elems = seg.total
        for i, o in enumerate(seg.offs):
            d.seg_off[i] = o
        d.capacity = cap
        d.log, d.tau = log.data_ptr(), tau.data_ptr()
        self._desc = d

    def record_attempt(self, handle, n_enq):
        """After attempt n_enq's finalize: accepted steps are n_acc <= n_enq, so n_enq slots always suffice."""
        if n_enq > self.cap:
            self._grow(n_enq)
        _lib.check(_lib.lib.b2ode_bp_record(handle, C.byref(self._desc)))

    def finish_adaptive(self, n_acc):
        self.n_steps = int(n_acc)

    # ---- fixed grid ----------------------------------------------------------------------------
    def start_fixed(self, seg, method, times, n_steps):
        import numpy as np
        self.fixed, self.seg, self.n_steps = True, seg, n_steps
        self.rk4 = method == "rk4"
        self.dt_host = [0.0] * n_steps
        self.beta, self.c_sol = _FIXED_TAB[method]
        self.nk, self.fsal = len(self.c_sol), False
        self.ckpt = torch.empty((max(n_steps, 1), seg.total), dtype=seg.dtype, device=seg.device)
        self.ckpt_f0 = None
        self.tau = torch.from_numpy(np.ascontiguousarray(times)).to(seg.device) if n_steps else None
        self._log_host = np.zeros((max(n_steps, 1), _STEP), dtype=np.uint8)

    def record_fixed_step(self, i, y_views, t0, t1, dt, j0, j1, ends):
        self.seg.fill(self.ckpt[i], y_views)
        self.dt_host[i] = float(dt)
        e = _lib.BpStep(float(t0), float(t1), float(dt), int(j0), int(j1), 1 if ends else 0, 0)
        self._log_host[i] = memoryview(bytes(e))

    def finish_fixed(self):
        self.log = torch.from_numpy(self._log_host).to(self.seg.device)
        del self._log_host


class RowsRecord(object):
    """What an independent-rows forward solve leaves for the backward pass: per row and accepted step, y_n (D elements),
    (t_n, dt_n) (16 bytes) and, without FSAL, f0 (D elements), slot-major [slot][row]."""

    def start(self, seg, tab, desc, base, rows):
        """Called by the rows driver before the recording launch: allocates the initial record."""
        self.seg, self.tab, self.desc_adaptive, self.base, self.rows = seg, tab, desc, base, rows
        self.dim = base.dim
        self.rerun = False
        item = seg.dtype.itemsize
        per_slot = rows * (self.dim * item * (1 if tab.fsal else 2) + 16)
        self._alloc(max(1, min(ROWS_INITIAL_SLOTS, ROWS_INITIAL_BYTES // per_slot)))

    def _alloc(self, cap):
        seg, shape = self.seg, (cap, self.rows, self.dim)
        self.ckpt = self.ckpt_f0 = self.sched = None          # free the old record before the new one is allocated
        self.ckpt = torch.empty(shape, dtype=seg.dtype, device=seg.device)
        self.ckpt_f0 = None if self.tab.fsal else torch.empty(shape, dtype=seg.dtype, device=seg.device)
        self.sched = torch.empty((cap, self.rows, 2), dtype=torch.float64, device=seg.device)
        self.capacity = cap
        d = _lib.RowsRecordDesc()
        d.ckpt = self.ckpt.data_ptr()
        d.ckpt_f0 = self.ckpt_f0.data_ptr() if self.ckpt_f0 is not None else None
        d.sched, d.capacity = self.sched.data_ptr(), cap
        self.desc = d

    def grow(self, need):
        self.rerun = True
        self._alloc(int(need))

    def finish(self, row_acc, total, most):
        self.row_acc, self.n_steps, self.max_steps = row_acc, int(total), int(most)


def _rows_backward(solver, rec, t_dev, gs, params):
    """One launch of b2ode_rows_bp: (dL/dy0, flat float64 parameter gradients or None, launches)."""
    seg, g = rec.seg, gs[0]
    if rec.max_steps == 0:
        return g[0], None, 0
    dev = seg.device
    rows, n_out = rec.rows, int(t_dev.shape[0])
    P = sum(p.numel() for p in params)
    grad_y0 = torch.empty(seg.shapes[0], dtype=seg.dtype, device=dev)
    pgrad = torch.empty(P, dtype=torch.float64, device=dev) if P else None
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    d = _lib.RowsBpDesc()
    d.rhs, weights = rec.base.rhs_desc(seg.dtype, dev, float(solver.func._b2ode_sign))
    nbytes = int(_lib.lib.b2ode_rows_bp_workspace_bytes(C.byref(d.rhs), rows, P, sm))
    if nbytes == 0:
        _lib.check(-1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    d.ckpt = rec.ckpt.data_ptr()
    d.ckpt_f0 = rec.ckpt_f0.data_ptr() if rec.ckpt_f0 is not None else None
    d.sched, d.capacity, d.n_acc = rec.sched.data_ptr(), rec.capacity, rec.row_acc.data_ptr()
    d.t_out, d.n_out = t_dev.data_ptr(), n_out
    d.grad_out, d.grad_y0 = g.data_ptr(), grad_y0.data_ptr()
    d.n_params = P
    d.param_grad = pgrad.data_ptr() if pgrad is not None else None
    d.workspace, d.workspace_bytes = ws.data_ptr(), nbytes
    d.sm_count, d.cuda_stream = sm, torch.cuda.current_stream(dev).cuda_stream
    _lib.check(_lib.lib.b2ode_rows_bp(C.byref(rec.desc_adaptive), C.byref(d)))
    return grad_y0, pgrad, 1


class _Backward(object):
    """The reverse sweep over the recorded steps (see the module docstring)."""

    def __init__(self, func, rec, t_dev, params):
        self.func, self.rec, self.t_dev, self.params = func, rec, t_dev, params
        seg = rec.seg
        self.seg, self.dcode = seg, _solvers._DT[seg.dtype]
        self.sm = torch.cuda.get_device_properties(seg.device).multi_processor_count
        self.stream = torch.cuda.current_stream(seg.device).cuda_stream
        self.launches = 0
        self.calls = 0
        # a built-in right-hand side that the forward solve evaluated in the stage kernels: its k's and vector-Jacobian
        # products come from b2ode_bp_rhs, with no forward or autograd call
        self.builtin = rec.builtin
        self.param_acc = None
        if self.builtin is not None:
            self.rd, self._weights = self.builtin.rhs_desc(seg.dtype, seg.device, float(getattr(func, "_b2ode_sign", 1.0)))
            if params:
                P = sum(p.numel() for p in params)
                self.param_acc = torch.zeros(P, dtype=torch.float64, device=seg.device)
                nbytes = int(_lib.lib.b2ode_bp_rhs_workspace_bytes(C.byref(self.rd), seg.lens[0], P, self.sm))
                if nbytes == 0:
                    _lib.check(-1)
                self.rhs_ws = torch.zeros(nbytes, dtype=torch.uint8, device=seg.device)

    def combine(self, out, base, terms, step):
        """out = base + sum (dt_n c) x over (coef, flat) terms; returns False (and writes nothing) with no terms."""
        seg = self.seg
        terms = [(c, x) for c, x in terms if c != 0.0]
        if not terms:
            return False
        d = _lib.BpCombineDesc()
        d.dtype, d.nseg = self.dcode, seg.nseg
        for i, n in enumerate(seg.lens):
            d.seg_len[i] = n
        for i, p in enumerate(seg.ptrs(out)):
            d.out[i] = p
        if base is not None:
            for i, p in enumerate(seg.ptrs(base)):
                d.base[i] = p
        d.nterms = len(terms)
        for j, (c, x) in enumerate(terms):
            d.coef[j] = c
            for i, p in enumerate(seg.ptrs(x)):
                d.x[j][i] = p
        d.step = step
        d.sm_count, d.cuda_stream = self.sm, self.stream
        _lib.check(_lib.lib.b2ode_bp_combine(C.byref(d)))
        self.launches += 1
        return True

    def rk4_stage(self, out, y_n, ks, dt):
        """out = the fixed-grid rk4 stage input after k_1 .. k_len(ks), with the forward's formula (b2ode_fixed_op)."""
        seg = self.seg
        op = (_lib.OP_RK4_S2, _lib.OP_RK4_S3, _lib.OP_RK4_S4)[len(ks) - 1]
        ops = [_lib.PtrArray(*seg.ptrs(x)) for x in ks] + [None] * (4 - len(ks))
        _lib.check(_lib.lib.b2ode_fixed_op(self.dcode, op, seg.nseg, _lib.LenArray(*seg.lens), _lib.PtrArray(*seg.ptrs(out)),
                                           _lib.PtrArray(*seg.ptrs(y_n)), *ops, float(dt), 0.0, 0.0, self.sm,
                                           C.c_void_p(self.stream)))
        self.launches += 1

    def stage_k(self, tau, y_n, terms, step, rk4_dt=None):
        """k = func(tau, Y), Y = y_n + sum (dt_n c) k_j (rk4_dt given: the rk4 stage input of the k's, dt_n = rk4_dt):
        returns (k, what stage_vjp needs)."""
        terms = [(c, x) for c, x in terms if c != 0.0]
        rk4 = rk4_dt is not None and len(terms) > 0
        if self.builtin is not None:
            k = self.seg.new()
            self.rhs_launch(_lib.BP_EVAL, tau, y_n, terms, None, [], k, step, rk4)
            return k, (tau, terms, rk4)
        if rk4:
            Y = self.seg.new()
            self.rk4_stage(Y, y_n, [x for _, x in terms], rk4_dt)
        elif terms:
            Y = self.seg.new()
            self.combine(Y, y_n, terms, step)
        else:
            Y = y_n
        k, outs, leaf = self.evaluate(tau, Y)
        return k, (outs, leaf)

    def stage_vjp(self, y_n, handle, base, terms, step, pgrads):
        """J^T mu at the evaluation `handle`, mu = base + sum (dt_n c) x (None when mu is absent)."""
        if self.builtin is not None:
            terms = [(c, x) for c, x in terms if c != 0.0]
            if not terms and base is None:
                return None
            nu = self.seg.new()
            tau, yterms, rk4 = handle
            self.rhs_launch(_lib.BP_VJP, tau, y_n, yterms, base, terms, nu, step, rk4)
            return nu
        mu = self.seg.new()
        if not self.combine(mu, base, terms, step):
            mu = base
        if mu is None:
            return None
        return self.vjp(handle[0], handle[1], mu, pgrads)

    def rhs_launch(self, mode, tau, y_n, yterms, base, mterms, out, step, rk4=False):
        d = _lib.BpRhsDesc()
        d.dtype, d.mode, d.rhs, d.n = self.dcode, mode, self.rd, self.seg.lens[0]
        d.step, d.t_scalar, d.y = step, tau.data_ptr(), y_n.data_ptr()
        d.ny, d.rk4_stage = len(yterms), 1 if rk4 else 0
        for j, (c, x) in enumerate(yterms):
            d.cy[j], d.ky[j] = c, x.data_ptr()
        d.base = base.data_ptr() if base is not None else None
        d.nm = len(mterms)
        for j, (c, x) in enumerate(mterms):
            d.cm[j], d.xm[j] = c, x.data_ptr()
        d.out = out.data_ptr()
        if self.param_acc is not None:
            d.n_params, d.param_acc = self.param_acc.numel(), self.param_acc.data_ptr()
            d.workspace, d.workspace_bytes = self.rhs_ws.data_ptr(), self.rhs_ws.numel()
        d.sm_count, d.cuda_stream = self.sm, self.stream
        _lib.check(_lib.lib.b2ode_bp_rhs(C.byref(d)))
        self.launches += 1

    def evaluate(self, tau, y_flat):
        """k = func(tau, Y) with Y a fresh leaf: returns (k as an engine buffer, the call's outputs, the leaf)."""
        seg = self.seg
        leaf = y_flat.detach().requires_grad_(True)
        with torch.enable_grad():
            outs = self.func(tau, seg.views(leaf))
        self.calls += 1
        if isinstance(outs, torch.Tensor):
            outs = (outs,)
        k = seg.new()
        seg.fill(k, [o.detach() for o in outs])
        return k, outs, leaf

    def vjp(self, outs, leaf, mu, pgrads):
        """J^T mu at the call that produced `outs`; accumulates the parameter cotangents into pgrads."""
        seg = self.seg
        live = [(o, m) for o, m in zip(outs, seg.views(mu)) if isinstance(o, torch.Tensor) and o.requires_grad]
        if not live:
            return None
        wrt = (leaf,) + self.params
        gs = torch.autograd.grad([o for o, _ in live], wrt, [m.reshape(o.shape) for o, m in live], allow_unused=True)
        for i, g in enumerate(gs[1:]):
            if g is not None:
                pgrads[i] = g if pgrads[i] is None else pgrads[i] + g
        return gs[0]

    def run(self, grad_out):
        rec, seg = self.rec, self.seg
        nk, beta, c_sol, fsal = rec.nk, rec.beta, rec.c_sol, rec.fsal
        pgrads = [None] * len(self.params)
        lam = seg.new().zero_()
        carry = None
        g_ptrs = [g.data_ptr() for g in grad_out]
        quartic = not rec.fixed
        if quartic:
            tab = rec.tab
            mask = 1 | (1 << (nk - 1))
            for j in range(nk):
                if tab.c_mid[j] != 0.0:
                    mask |= 1 << j
        else:
            mask = 0
        mu_dense = [seg.new() if (mask >> j) & 1 else None for j in range(nk)]
        g0 = seg.new()
        for n in range(rec.n_steps - 1, -1, -1):
            step = rec.log.data_ptr() + _STEP * n
            y_n = rec.ckpt[n]
            tau = rec.tau[n]
            fresh0 = rec.fixed or fsal or n == 0
            # ---- recompute the stages of step n -----------------------------------------------------
            if fresh0:
                k0, h0 = self.stage_k(tau[0], y_n, [], step)
            else:
                k0, h0 = rec.ckpt_f0[n], None
            ks, calls = [k0], []
            rk4_dt = rec.dt_host[n] if rec.fixed and rec.rk4 else None
            for i in range(nk - 1):
                k, h = self.stage_k(tau[i + 1], y_n, [(beta[i][j], ks[j]) for j in range(i + 1)], step, rk4_dt)
                ks.append(k)
                calls.append(h)
            # ---- dense output -----------------------------------------------------------------------
            d = _lib.BpDenseDesc()
            d.dtype, d.nseg, d.n_k = self.dcode, seg.nseg, nk
            d.kind = _lib.BP_QUARTIC if quartic else _lib.BP_LINEAR
            for i, ln in enumerate(seg.lens):
                d.seg_len[i] = ln
                d.grad_out[i] = g_ptrs[i]
            for i, p in enumerate(seg.ptrs(g0)):
                d.grad_y0[i] = p
            for i, p in enumerate(seg.ptrs(lam)):
                d.grad_y1[i] = p
            d.k_mask = mask
            for j in range(nk):
                if mu_dense[j] is not None:
                    d.c_mid[j] = tab.c_mid[j]
                    for i, p in enumerate(seg.ptrs(mu_dense[j])):
                        d.grad_k[j][i] = p
            d.step, d.t_out = step, self.t_dev.data_ptr()
            d.sm_count, d.cuda_stream = self.sm, self.stream
            _lib.check(_lib.lib.b2ode_bp_dense(C.byref(d)))
            self.launches += 1
            if carry is not None:
                # adaptive Heun: this step's last k is the next step's f0
                self.combine(mu_dense[nk - 1], mu_dense[nk - 1], [(1.0, carry)], None)
            # ---- reverse stage sweep ----------------------------------------------------------------
            # lambda (the cotangent of y_{n+1}) enters k_j with dt b_j -- for FSAL y_{n+1} is the last stage input,
            # whose row of beta is b
            lam_coef = beta[nk - 2] if fsal else c_sol
            nus = [None] * (nk - 1)
            for i in range(nk - 2, -1, -1):
                j = i + 1
                terms = [(beta[l][j], nus[l]) for l in range(j, nk - 1) if nus[l] is not None]
                if j < len(lam_coef):
                    terms.append((lam_coef[j], lam))
                nus[i] = self.stage_vjp(y_n, calls[i], mu_dense[j], terms, step, pgrads)
            terms = [(beta[l][0], nus[l]) for l in range(nk - 1) if nus[l] is not None] + [(lam_coef[0], lam)]
            xi0 = None
            if fresh0:
                xi0 = self.stage_vjp(y_n, h0, mu_dense[0], terms, step, pgrads)
                carry = None
            else:
                carry = seg.new()
                if not self.combine(carry, mu_dense[0], terms, step):
                    carry = mu_dense[0]
            # ---- lambda_n = dense + sum nu_i + lambda_{n+1} (+ J^T mu_0) ---------------------------
            new = seg.new()
            self.combine(new, g0, [(1.0, v) for v in nus + [xi0] if v is not None] + [(1.0, lam)], None)
            lam = new
            del calls, ks, h0
        if self.param_acc is not None:
            off = 0
            for i, p in enumerate(self.params):
                pgrads[i] = self.param_acc[off:off + p.numel()].reshape(p.shape)
                off += p.numel()
        return lam, pgrads


class _OdeintBackprop(torch.autograd.Function):

    @staticmethod
    def forward(ctx, solver, t_dev, n_params, *args):
        flat_params, y0 = args[0], args[1:]
        rec = RowsRecord() if getattr(solver, "independent_rows", False) else Record()
        solver.bp_record = rec
        _rhs._FORCE_ACCURATE[0] += 1
        try:
            with torch.no_grad():
                sol = solver.integrate(t_dev)
        finally:
            _rhs._FORCE_ACCURATE[0] -= 1
            solver.bp_record = None
        if isinstance(rec, Record) and not rec.fixed:
            rec.finish_adaptive(solver.stats["n_accepted"])
        # output times on the device in float64: k_bp_dense reads them there
        ctx.solver, ctx.rec = solver, rec
        ctx.t_dev = t_dev.detach().to(device=y0[0].device, dtype=torch.float64).contiguous()
        return tuple(sol)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grad_out):
        rec, solver = ctx.rec, ctx.solver
        seg = rec.seg
        gs = [torch.zeros((ctx.t_dev.shape[0],) + shp, dtype=seg.dtype, device=seg.device) if g is None
              else g.to(seg.dtype).contiguous() for g, shp in zip(grad_out, seg.shapes)]
        params = _trainable(solver.func_module) if solver.func_module is not None else ()
        global last_stats
        if isinstance(rec, RowsRecord):
            with torch.cuda.device(seg.device), torch.no_grad():
                grad, pflat, launches = _rows_backward(solver, rec, ctx.t_dev, gs, params)
            last_stats = dict(rows=rec.rows, steps=rec.n_steps, launches=launches, func_calls=0, rerun=rec.rerun)
            if params and pflat is None:
                pflat = torch.zeros(sum(p.numel() for p in params), dtype=torch.float64, device=seg.device)
            flat = pflat.to(params[0].dtype) if params else None
            return (None, None, None, flat, grad)
        if rec.n_steps == 0:
            grads, pgrads = [g[0] for g in gs], [None] * len(params)
            last_stats = dict(steps=0, launches=0, func_calls=0)
        else:
            _rhs._FORCE_ACCURATE[0] += 1
            try:
                with torch.cuda.device(seg.device), torch.no_grad():
                    bw = _Backward(solver.func, rec, ctx.t_dev, params)
                    lam, pgrads = bw.run(gs)
                    grads = [v + g[0] for v, g in zip(seg.views(lam), gs)]
            finally:
                _rhs._FORCE_ACCURATE[0] -= 1
            last_stats = dict(steps=rec.n_steps, launches=bw.launches, func_calls=bw.calls)
        if params:
            flat = torch.cat([(torch.zeros_like(p) if g is None else g).reshape(-1).to(p.dtype) for g, p in zip(pgrads, params)])
        else:
            flat = None
        return (None, None, None, flat) + tuple(grads)


def integrate(solver, func, y0, t):
    """solver.integrate(t) with the result attached to autograd through _OdeintBackprop."""
    from .adjoint import _FlatParamsGrad
    params = _trainable(func)
    solver.func_module = func if isinstance(func, nn.Module) else None
    flat = _FlatParamsGrad.apply(*params) if params else torch.zeros(0, dtype=y0[0].dtype, device=y0[0].device)
    return _OdeintBackprop.apply(solver, t, len(params), flat, *y0)
