"""Public entry point with the reference's signature and dispatch (tfdiffeq/odeint.py:11-81)."""
from .misc import _check_inputs
from .multistep import AdamsBashforth, AdamsBashforthMoulton, VariableCoefficientAdamsBashforth
from .solvers import (AdaptiveHeunSolver, Bosh3Solver, Dopri5Solver, Dopri8Solver, Euler, Heun, Midpoint, RK4,
                      Tsit5Solver)

# method name -> solver class; the names (including the historical 'huen' spelling) are the reference's
# (tfdiffeq/odeint.py:11-25)
_ADAPTIVE_RK = dict(dopri5=Dopri5Solver, dopri8=Dopri8Solver, bosh3=Bosh3Solver, tsit5=Tsit5Solver,
                    adaptive_heun=AdaptiveHeunSolver)
_FIXED_GRID = dict(euler=Euler, midpoint=Midpoint, rk4=RK4, heun=Heun, huen=Heun)
_MULTISTEP = dict(adams=VariableCoefficientAdamsBashforth, fixed_adams=AdamsBashforthMoulton, explicit_adams=AdamsBashforth)
SOLVERS = dict(_ADAPTIVE_RK, **_FIXED_GRID, **_MULTISTEP)


def odeint(func, y0, t, rtol=1e-7, atol=1e-9, method=None, options=None):
    """Integrate ``dy/dt = func(t, y), y(t[0]) = y0`` and return ``y`` at every time in ``t``.

    Same contract as the reference (tfdiffeq/odeint.py:28-81): ``y0`` is a tensor of any shape or a tuple of
    tensors, ``t`` a strictly monotone 1-D tensor (decreasing ``t`` integrates backwards, misc.py:318-321),
    the result has shape ``(len(t), *y0.shape)`` (a tuple of such for tuple states) in ``y0``'s dtype.
    ``func(t, y)`` is any callable on torch CUDA tensors, typically an ``nn.Module``; ``t`` reaches it as a
    0-dim device tensor.  Raises ``ValueError`` if ``options`` is given without ``method``, ``KeyError`` for
    an unknown ``method``, ``TypeError`` for non-numeric inputs, ``AssertionError`` for non-monotone ``t``,
    step-size underflow, non-finite states or ``max_num_steps``; unknown option keys only warn.

    ``options={'independent_rows': True}`` (``dopri5``, ``bosh3``, ``adaptive_heun``, ``dopri8``; a built-in right-hand
    side of ``tfdiffeq_b200.rhs``; a single fp32/fp64 tensor state; scalar ``rtol``/``atol``): every row
    ``y0.reshape(-1, func.dim)[r]`` is solved as its own system, exactly as ``odeint`` would solve that row alone -- its own
    initial step, error norm over the row, accept decisions, step counts and ``max_num_steps`` -- in one kernel launch for
    a batch of any size.  If any row fails, ``AssertionError`` carries the message of the first failed row and the number
    of failed rows.  ``last_stats`` then holds totals over rows plus per-row CUDA tensors ``row_accepted``,
    ``row_rejected``, ``row_dt_next``, ``row_error_ratio`` and ``row_status``.  Other adaptive methods, other ``func`` s,
    tuple states, per-component tolerances, ``fused_rhs=False``/``'stages'`` and ``shared_step_group`` raise
    ``ValueError``; fixed-grid methods accept the flag and ignore it (their rows are already independent).
    ``odeint_adjoint`` differentiates such a solve row by row when ``fused_vjp`` is also given (see its docstring).

    ``options={'backprop': True}`` differentiates through the solve itself: when autograd needs the result (grad mode on
    and ``y0`` or a trainable parameter of an ``nn.Module`` ``func`` requires grad) the returned tensors have a
    ``grad_fn`` whose backward pass is the exact reverse-mode derivative of the computation the solver performed, with
    the step schedule held constant -- every accepted step's t_n and dt_n, the initial step and the interpolation
    abscissae are constants and rejected attempts contribute nothing (what torchdiffeq and a tape around the oracle's
    solver compute, without the tape's derivative of the controller's dt).  Gradients reach every component of ``y0``
    and the trainable parameters of ``func`` when it is an ``nn.Module`` (a plain callable gets ``y0`` gradients only);
    ``t`` is held constant.  ``dopri5``, ``bosh3``, ``adaptive_heun``, ``dopri8``, ``euler``, ``midpoint``, ``rk4`` and
    ``heun``/``huen``.  The forward solve keeps one checkpoint of the state per accepted step ((steps + 1) N elements;
    2x for ``adaptive_heun``) until the graph is freed; the backward pass calls ``func`` once per stage per step (with
    autograd) and launches the stage combines and the dense-output VJP.  Built-in right-hand sides run the stage kernels
    (not the persistent kernel) in the forward solve and ``b2ode_bp_rhs`` in the backward pass, with no ``forward`` or
    autograd call (a CubicMLP trains with all four weights or none, a LatentODEFunc with all six or none; a partly frozen
    one raises ``ValueError``, as does a
    built-in with other trainable parameters); tensor-core funcs run their fp32-accurate mode.  ``tsit5``, the
    multistep methods, ``shared_step_group``, ``cuda_graph``, ``host_output`` and a ``t`` that requires grad raise
    ``ValueError`` before anything runs.  If autograd does not need the result the solve is the one made without the flag.

    ``options={'independent_rows': True, 'backprop': True}`` (a built-in right-hand side, an adaptive method above) gives
    every row the gradient ``backprop`` gives that row solved alone: ``y0.grad[r]`` is bit for bit that of
    ``y0.reshape(-1, dim)[r:r+1]`` with ``backprop``, and a CubicMLP or LatentODEFunc whose weights are trainable gets the sum over
    rows of the per-row weight gradients (in fp64, in a fixed order).  The forward solve is the plain rows solve (same
    solution, counts and failures) that also records every row's accepted steps -- y_n, t_n and dt_n per step, and f0
    for ``adaptive_heun`` -- and runs once more if a row outgrew the initial record (``backprop.last_stats['rerun']``);
    the backward pass is one kernel launch.  A func that is not a built-in raises ``ValueError``, as does everything
    either option refuses on its own.  Fixed-grid methods drop ``independent_rows`` with ``backprop`` as they do without.
    """
    backprop = isinstance(options, dict) and bool(options.get("backprop", False))
    if isinstance(options, dict) and "backprop" in options:
        from . import backprop as _bp
        options = _bp.check_options(method, options, t) if backprop else {k: v for k, v in options.items() if k != "backprop"}
        if backprop:
            _bp.check_rows(func, options)
            _bp.check_builtin(func, options)
        backprop = backprop and _bp.needs_grad(func, y0)
    user_func = func
    tensor_input, func, y0, t = _check_inputs(func, y0, t)
    if options is not None and method is None:
        raise ValueError('cannot supply `options` without specifying `method`')      # odeint.py:72-73
    solver_cls = SOLVERS['dopri5' if method is None else method]                     # unknown name: KeyError (:77)
    odeint.last_solver = solver = solver_cls(func, y0, rtol=rtol, atol=atol, **(options or {}))
    if backprop:
        solution = _bp.integrate(solver, user_func, y0, t)
    else:
        solution = solver.integrate(t)
    return solution[0] if tensor_input else solution


odeint.last_solver = None
