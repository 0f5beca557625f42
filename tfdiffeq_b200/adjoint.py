"""``odeint_adjoint``: O(1)-memory gradients by solving the augmented system backwards in time.

Caller of the hot path (SURVEY.md 8(f)-1): the reference implements it as a ``tf.custom_gradient`` around
``odeint`` (tfdiffeq/adjoint.py:35-180); here it is a ``torch.autograd.Function`` with the same algorithm.
The backward pass runs the same sm_90a kernels on the augmented tuple state
``(y, adj_y, adj_t, adj_params)`` -- components of unequal shapes, per-component error norms -- and takes
the vector-Jacobian products of ``func`` from PyTorch autograd (the reference uses a ``GradientTape``,
adjoint.py:77-96).
"""
import torch
import torch.nn as nn

from . import _lib
from . import rhs as _rhs
from .odeint import odeint


def _flatten(seq):
    flat = [p.reshape(-1) for p in seq]
    return torch.cat(flat) if len(flat) > 0 else torch.tensor([])


# statistics of the most recent odeint_adjoint call: the forward solve and every backward (augmented) solve
last_stats = {"forward": None, "backward": []}


def _group_of(options):
    return (options or {}).get("shared_step_group") if isinstance(options, dict) else None


def _all_reduce_sum(x, group):
    """Sum over the ranks of a shared-step group (NCCL on the current stream).  Batch-summed quantities of the
    adjoint -- a^T df/dtheta, a^T df/dt, dL/dt_i -- are sums over ALL trajectories of the system, i.e. over all shards."""
    import torch.distributed as dist
    if x.numel():
        dist.all_reduce(x, group=group.group)
    return x


def _augmented_dynamics(func, n_tensors, f_params, dtype, dev, group):
    """The backward pass's func (adjoint.py:71-107): ``(f, -a^T df/dy, -a^T df/dt, -a^T df/dtheta)`` of the tuple state
    ``(*y, *adj_y, adj_t, adj_params)``, with the vector-Jacobian products from torch autograd of ``func``."""

    def augmented_dynamics(tt, y_aug):
        y, adj_y = y_aug[:n_tensors], y_aug[n_tensors:2 * n_tensors]
        with torch.enable_grad():
            tt_ = tt.detach().requires_grad_(True)
            y_ = tuple(v.detach().requires_grad_(True) for v in y)
            func_eval = func(tt_, y_)
            # outputs that depend on none of (t, y, theta) -- a constant field, a component func passes through
            # detached -- have no graph: their VJP is zero (the reference asks for UnconnectedGradients.ZERO,
            # adjoint.py:88-96) and autograd.grad must not see them
            live = [(f, -a) for f, a in zip(func_eval, adj_y) if f.requires_grad]
            wrt = (tt_,) + y_ + f_params
            if live:
                vjps = torch.autograd.grad([f for f, _ in live], wrt, [a for _, a in live], allow_unused=True)
            else:
                vjps = (None,) * len(wrt)
        vjp_t, vjp_y, vjp_params = vjps[0], vjps[1:1 + n_tensors], vjps[1 + n_tensors:]
        vjp_t = torch.zeros_like(tt_) if vjp_t is None else vjp_t
        vjp_y = tuple(torch.zeros_like(v) if g is None else g for g, v in zip(vjp_y, y_))
        if len(f_params) == 0:
            vjp_p = torch.zeros((), dtype=dtype, device=dev)                              # adjoint.py:103-105
        else:
            vjp_p = _flatten([torch.zeros_like(p) if g is None else g for g, p in zip(vjp_params, f_params)])
            vjp_p = vjp_p.to(dtype)
        vjp_t = vjp_t.to(dtype)
        if group is not None:
            vjp_t = _all_reduce_sum(vjp_t.contiguous(), group)
            if len(f_params):
                vjp_p = _all_reduce_sum(vjp_p.contiguous(), group)
        return (*(f.detach() for f in func_eval), *vjp_y, vjp_t, vjp_p)
    return augmented_dynamics


class _FusedAugmentedDynamics(object):
    """The augmented dynamics of a built-in right-hand side with ``fused_vjp``: a marker the adaptive solvers recognise
    (solvers._adjoint_rhs) and evaluate in the stage kernels (b2ode_adjoint_rhs_eval / b2ode_rk_stage_adjoint_rhs).  It
    is never called per evaluation."""

    def __init__(self, module):
        self.adjoint_rhs = module

    def __call__(self, t, y_aug):
        raise RuntimeError("fused_vjp: the augmented dynamics of %s are evaluated by the stage kernels only"
                           % type(self.adjoint_rhs).__name__)


def _check_fused_vjp(func, y0, adjoint_method, adjoint_options):
    """Raise ValueError unless the backward solves of odeint_adjoint(func, y0, ...) can run with fused_vjp."""
    from .odeint import _ADAPTIVE_RK
    if not isinstance(func, _rhs.BuiltinRHS):
        raise ValueError("fused_vjp needs a built-in right-hand side (tfdiffeq_b200.rhs.Lorenz, LotkaVolterra, Kepler, "
                         "CubicMLP or LatentODEFunc), got %s" % type(func).__name__)
    if not isinstance(y0, torch.Tensor):
        raise ValueError("fused_vjp needs a single-tensor state, not a tuple")
    if y0.dim() < 1 or y0.numel() == 0 or y0.shape[-1] % func.dim:
        raise ValueError("fused_vjp needs a non-empty state whose last axis holds whole rows of %d" % func.dim)
    method = "dopri5" if adjoint_method is None else adjoint_method
    if method not in _ADAPTIVE_RK:
        raise ValueError("fused_vjp runs the adaptive Runge-Kutta stage kernels; adjoint_method %r is not one of %s"
                         % (method, sorted(_ADAPTIVE_RK)))
    ao = adjoint_options if isinstance(adjoint_options, dict) else {}
    fr = ao.get("fused_rhs", True)
    if fr is not True:
        raise ValueError("fused_vjp evaluates the right-hand side in the stage kernels; it cannot be combined with "
                         "fused_rhs=%r" % (fr,))
    if ao.get("shared_step_group") is not None:
        raise ValueError("fused_vjp cannot be combined with shared_step_group")
    params = list(func.parameters())
    if func.trainable_weights is not None:
        count, names = func.trainable_weights
        if not _rhs.weights_all_or_none(func):
            raise ValueError("fused_vjp supports a %s whose %s weights (%s) are all trainable or all frozen, and no other "
                             "parameters" % (type(func).__name__, count, ", ".join(names)))
    elif any(p.requires_grad for p in params):
        raise ValueError("fused_vjp: %s has trainable parameters the kernels do not know" % type(func).__name__)


_ROWS_METHODS = ("dopri5", "bosh3", "adaptive_heun", "dopri8")


def _check_independent_rows(func, method, adjoint_method, rtol, atol):
    """Raise ValueError unless the rows of odeint_adjoint(func, ...) can be differentiated one by one (independent_rows
    with fused_vjp; the fused_vjp checks have run)."""
    for name, m in (("method", method), ("adjoint_method", adjoint_method)):
        m = "dopri5" if m is None else m
        if m not in _ROWS_METHODS:
            raise ValueError("independent_rows in odeint_adjoint supports %s for %s, got %r" % (", ".join(_ROWS_METHODS), name, m))
    if any(p.requires_grad for p in func.parameters()):
        raise ValueError("independent_rows in odeint_adjoint takes a right-hand side with frozen parameters: the per-row "
                         "parameter adjoint of a trainable %s does not fit one thread" % type(func).__name__)
    for name, tol in (("rtol", rtol), ("atol", atol)):
        if isinstance(tol, (list, tuple)) or (isinstance(tol, torch.Tensor) and tol.numel() > 1):
            raise ValueError("independent_rows takes one scalar %s for every row, not per-component values" % name)


def _rows_backward(t, ans, grad_output, opts):
    """The backward pass of odeint_adjoint with independent_rows: (dL/dy0, dL/dt).  The adjoint method's solver is built
    as odeint builds it -- on the augmented state of the last interval, reverse-time wrapper included -- so its option
    parsing, first_step, max_num_steps, controller factors and warnings are odeint's; it then runs every row and every
    interval in one launch (solvers.AdaptiveStepsizeODESolver.integrate_adjoint_rows)."""
    from . import solvers as _solvers
    from .misc import _check_inputs
    from .odeint import SOLVERS
    module = opts["tensor_func"]
    T = ans.shape[0]
    if T == 1:
        last_stats["backward"] = dict(independent_rows=True, fused_vjp=True, rows=grad_output[0].numel() // module.dim,
                                      intervals=0, n_accepted=0, n_rejected=0, nfe=0, status=0)
        return grad_output[0].clone(), torch.zeros_like(t)
    dtype, dev = ans.dtype, ans.device
    zero = torch.zeros((), dtype=dtype, device=dev)
    aug_y0 = (ans[-1], grad_output[-1], zero, zero)                                          # adjoint.py:146
    _, func, aug_y0, _ = _check_inputs(_FusedAugmentedDynamics(module), aug_y0, torch.stack([t[-1], t[-2]]))
    method = opts["adjoint_method"]
    solver = SOLVERS["dopri5" if method is None else method](func, aug_y0, rtol=opts["adjoint_rtol"],
                                                             atol=opts["adjoint_atol"], **(opts["adjoint_options"] or {}))
    try:
        grad_y0, t_grad = solver.integrate_adjoint_rows(ans, grad_output, t)
    finally:
        # also when rows failed: the per-row status tells which
        last_stats["backward"] = dict(_solvers.last_stats) if solver.stats else {}
    return grad_y0, t_grad.to(t.dtype)


class _OdeintAdjoint(torch.autograd.Function):
    """tfdiffeq/adjoint.py:35-180"""

    @staticmethod
    def forward(ctx, func, n_tensors, options, t, flat_params, *y0):
        ctx.func, ctx.options, ctx.n_tensors = func, options, n_tensors
        # a tensor state is solved on the caller's module and tensor, not on the 1-tuple wrapper: odeint then recognises a
        # built-in right-hand side (persistent kernel, stage kernels) or a tensor-core func (stage-combine producer) exactly
        # as it does outside the adjoint.  The backward pass keeps the tuple form.
        base = options["tensor_func"]
        _rhs._FORCE_ACCURATE[0] += 1
        try:
            with torch.no_grad():
                kw = dict(rtol=options["rtol"], atol=options["atol"], method=options["method"], options=options["options"])
                if base is not None:
                    ans = (odeint(base, y0[0], t, **kw),)
                else:
                    ans = odeint(func, tuple(y0), t, **kw)                                    # adjoint.py:54
        finally:
            _rhs._FORCE_ACCURATE[0] -= 1
        from . import solvers as _solvers
        last_stats["forward"] = dict(_solvers.last_stats)
        last_stats["backward"] = []
        ctx.save_for_backward(t, flat_params, *ans)
        return ans

    @staticmethod
    def backward(ctx, *grad_output):
        t, flat_params, *ans = ctx.saved_tensors
        func, opts, n_tensors = ctx.func, ctx.options, ctx.n_tensors
        f_params = tuple(p for p in func.parameters() if p.requires_grad)
        dev, dtype = ans[0].device, ans[0].dtype
        grad_output = tuple(g if g is not None else torch.zeros_like(a) for g, a in zip(grad_output, ans))
        # Shards of one system on several GPUs (options={'shared_step_group': g}): y and adj_y are sharded like the
        # batch; adj_t and adj_params are sums over the whole batch, so their derivatives are all-reduced on every
        # evaluation and the two components are *replicated* (bit-identical on every rank, counted once in the norm)
        adj_options = opts["adjoint_options"]
        group = _group_of(adj_options)
        if group is not None and group.world > 1:
            adj_options = dict(adj_options, replicated_components=(2 * n_tensors, 2 * n_tensors + 1))
        else:
            group = None
        if opts["fused_vjp"]:
            # the same augmented system, evaluated on the device by the stage kernels (built-in right-hand sides)
            augmented_dynamics = _FusedAugmentedDynamics(opts["tensor_func"])
        else:
            augmented_dynamics = _augmented_dynamics(func, n_tensors, f_params, dtype, dev, group)

        if opts["independent_rows"]:
            with torch.no_grad():
                grad_y0, time_vjps = _rows_backward(t, ans[0], grad_output[0], opts)
            return (None, None, None, time_vjps, None, grad_y0)

        T = ans[0].shape[0]
        _rhs._FORCE_ACCURATE[0] += 1
        try:
            with torch.no_grad():
                adj_y = tuple(g[-1] for g in grad_output)                                     # adjoint.py:110-113
                adj_params = torch.zeros_like(flat_params, dtype=dtype) if flat_params.numel() else \
                    torch.zeros((), dtype=dtype, device=dev)
                adj_time = torch.zeros((), dtype=dtype, device=dev)
                time_vjps = []
                for i in range(T - 1, 0, -1):                                                 # adjoint.py:118
                    ans_i = tuple(a[i] for a in ans)
                    grad_i = tuple(g[i] for g in grad_output)
                    func_i = func(t[i].to(dtype), ans_i)
                    # effect of moving the current measurement time (adjoint.py:133-139)
                    dLd_cur_t = sum(torch.dot(f.reshape(-1), g.reshape(-1)).reshape(1) for f, g in zip(func_i, grad_i))
                    if group is not None:
                        dLd_cur_t = _all_reduce_sum(dLd_cur_t.contiguous(), group)
                    adj_time = adj_time - dLd_cur_t.reshape(())
                    time_vjps.append(dLd_cur_t)
                    aug_y0 = (*ans_i, *adj_y, adj_time, adj_params)                           # adjoint.py:146
                    aug_ans = odeint(augmented_dynamics, aug_y0, torch.stack([t[i], t[i - 1]]),
                                     rtol=opts["adjoint_rtol"], atol=opts["adjoint_atol"], method=opts["adjoint_method"],
                                     options=adj_options)                                     # adjoint.py:148-153
                    from . import solvers as _solvers
                    last_stats["backward"].append(dict(_solvers.last_stats))
                    adj_y = tuple(a[1] for a in aug_ans[n_tensors:2 * n_tensors])
                    adj_time = aug_ans[2 * n_tensors][1]
                    adj_params = aug_ans[2 * n_tensors + 1][1]
                    adj_y = tuple(a + g[i - 1] for a, g in zip(adj_y, grad_output))           # adjoint.py:164
                    del aug_y0, aug_ans
                time_vjps.append(adj_time.reshape(1))
                time_vjps = torch.cat(time_vjps[::-1]).to(t.dtype)                            # adjoint.py:169
                grad_params = adj_params if flat_params.numel() else None
        finally:
            _rhs._FORCE_ACCURATE[0] -= 1
        return (None, None, None, time_vjps, grad_params, *adj_y)


class _TupleFunc(nn.Module):
    """adjoint.py:205-212"""

    def __init__(self, base_func):
        super(_TupleFunc, self).__init__()
        self.base_func = base_func

    def forward(self, t, y):
        return (self.base_func(t, y[0]),)


class _FlatParamsGrad(torch.autograd.Function):
    """Routes the flat parameter gradient produced by the adjoint back onto the individual parameters."""

    @staticmethod
    def forward(ctx, *params):
        ctx.shapes = [p.shape for p in params]
        return _flatten(params) if params else torch.tensor([])

    @staticmethod
    def backward(ctx, g):
        out, off = [], 0
        for shp in ctx.shapes:
            n = 1
            for d in shp:
                n *= d
            out.append(g[off:off + n].reshape(shp))
            off += n
        return tuple(out)


def odeint_adjoint(func, y0, t, rtol=1e-6, atol=1e-12, method=None, options=None, adjoint_method=None,
                   adjoint_rtol=None, adjoint_atol=None, adjoint_options=None):
    """tfdiffeq/adjoint.py:183-224.  ``func`` must be an ``nn.Module`` (the reference demands a
    ``tf.keras.Model``, :187) so that its parameters can be found.

    The reference accepts ``adjoint_rtol`` / ``adjoint_atol`` but silently discards them and integrates the
    adjoint with ``rtol`` / ``atol`` (adjoint.py:18-19, :63-64).  That behaviour is reproduced.

    A state of n tensors integrates an augmented state of 2n + 2 components backwards; the engine carries at most
    ``B2ODE_MAXSEG`` = 12 components, i.e. n <= 5 (the reference has no such limit); a larger state raises
    ``ValueError`` before the forward solve.  Tensor-core funcs
    (``rhs.DenseMLP`` / ``rhs.Conv2dODEFunc``) run both passes in their fp32-accurate mode so that the forward solve,
    the backward reconstruction of y and the autograd VJPs see the same dynamics.  With
    ``options={'shared_step_group': g}`` (batch shards on several GPUs) the returned parameter and time gradients are
    already summed over all shards and identical on every rank.

    ``adjoint_options={'fused_vjp': True}`` (opt-in; also read from ``options`` when ``adjoint_options`` is not given):
    for a built-in right-hand side (``rhs.Lorenz``, ``LotkaVolterra``, ``Kepler``, ``CubicMLP``, ``LatentODEFunc``) on a
    single-tensor state,
    the backward solves evaluate the augmented dynamics in the stage kernels, vector-Jacobian products included, with no
    ``forward`` or ``autograd.grad`` call per evaluation.  The algorithm, step schedule and error norms are unchanged.
    Lorenz, Lotka-Volterra and Kepler give the same bits as the default path; ``CubicMLP`` and ``LatentODEFunc`` sum their
    parameter cotangents over the rows in a fixed order of their own, so their gradients agree with the default path to
    rounding.  Tuple states,
    other funcs, a fixed-grid or multistep ``adjoint_method``, ``fused_rhs=False``/``'stages'``, ``shared_step_group``
    and a partially frozen ``CubicMLP`` or ``LatentODEFunc`` raise ``ValueError`` before the forward solve.  Each entry of
    ``last_stats['backward']`` then carries ``fused_vjp=True``.

    ``options={'independent_rows': True, 'fused_vjp': True}`` (the flag in both ``options`` and ``adjoint_options``, which
    inherits it): gradients of a per-row solve (see ``odeint``).  Row r of ``y0.grad`` is what ``odeint_adjoint`` gives for
    the row ``y0.reshape(-1, func.dim)[r]`` alone, with the same methods, tolerances and options; ``t.grad`` is the sum
    over rows of each row's time gradient, formed in float64 in a fixed order.  The whole backward pass -- every row,
    every interval, the ``dL/dt_i`` terms -- is one kernel launch plus one for the time-gradient sums, with no ``forward``
    call.  Built-in ``Lorenz``, ``LotkaVolterra``, ``Kepler`` and a ``CubicMLP`` or ``LatentODEFunc`` with all weights
    frozen; ``dopri5``,
    ``bosh3``, ``adaptive_heun`` and ``dopri8`` forward and backward; scalar ``rtol``/``atol``.  The flag without
    ``fused_vjp``, in only one of ``options`` / ``adjoint_options``, a trainable ``CubicMLP`` or ``LatentODEFunc``, and everything
    ``independent_rows`` or ``fused_vjp`` refuse raise ``ValueError`` before the forward solve.  ``last_stats['backward']``
    is then ONE dict: totals, ``intervals``, and per-row CUDA tensors ``row_accepted`` / ``row_rejected`` (summed over the
    intervals), ``row_dt_next`` / ``row_error_ratio`` (after the last attempt of the interval ending at ``t[0]``) and
    ``row_status``.  A failed row raises ``AssertionError`` with that row's message and ``[row r; k of n rows failed]``.
    """
    if not isinstance(func, nn.Module):
        raise ValueError('func is required to be an instance of nn.Module')
    for o in (options, adjoint_options):
        if isinstance(o, dict) and "backprop" in o:
            raise ValueError("backprop is an option of odeint; odeint_adjoint computes the continuous adjoint instead")
    if adjoint_method is None:
        adjoint_method = method
    if adjoint_options is None:
        adjoint_options = options
    rows_fwd, rows_bwd = (bool(o.get("independent_rows")) if isinstance(o, dict) else False for o in (options, adjoint_options))
    if rows_fwd != rows_bwd:
        raise ValueError("independent_rows must be in both options and adjoint_options: a per-row forward solve needs a "
                         "per-row adjoint and the other way round")
    # fused_vjp belongs to the backward solves: neither the forward nor the backward odeint sees the key
    fused_vjp = bool(adjoint_options.get("fused_vjp", False)) if isinstance(adjoint_options, dict) else False
    if rows_bwd and not fused_vjp:
        raise ValueError("independent_rows in odeint_adjoint needs adjoint_options={'fused_vjp': True, ...}: there is no "
                         "per-row backward pass through torch autograd")
    if isinstance(options, dict) and "fused_vjp" in options:
        options = {k: v for k, v in options.items() if k != "fused_vjp"}
    if isinstance(adjoint_options, dict) and "fused_vjp" in adjoint_options:
        adjoint_options = {k: v for k, v in adjoint_options.items() if k != "fused_vjp"}
    if fused_vjp:
        _check_fused_vjp(func, y0, adjoint_method, adjoint_options)
    if rows_bwd:
        _check_independent_rows(func, method, adjoint_method, rtol, atol)
    tensor_input, base_func = False, None
    if isinstance(y0, torch.Tensor):
        tensor_input, base_func = True, func
        y0 = (y0,)
        func = _TupleFunc(func)
    if len(y0) > (_lib.MAXSEG - 2) // 2:
        raise ValueError("odeint_adjoint supports at most %d state tensors (the backward pass integrates 2n + 2 <= %d "
                         "components), got %d" % ((_lib.MAXSEG - 2) // 2, _lib.MAXSEG, len(y0)))
    params = tuple(p for p in func.parameters() if p.requires_grad)
    flat_params = _FlatParamsGrad.apply(*params) if params else torch.zeros(0, device=y0[0].device, dtype=y0[0].dtype)
    opts = dict(rtol=rtol, atol=atol, method=method, options=options, adjoint_method=adjoint_method,
                adjoint_rtol=rtol, adjoint_atol=atol, adjoint_options=adjoint_options, tensor_func=base_func,
                fused_vjp=fused_vjp, independent_rows=rows_bwd)
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(t)
    t = t.to(y0[0].device)
    ys = _OdeintAdjoint.apply(func, len(y0), opts, t, flat_params, *y0)
    if tensor_input:
        ys = ys[0]
    return ys
