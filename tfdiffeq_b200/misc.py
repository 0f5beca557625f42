"""Host-side input handling with the reference's semantics (``tfdiffeq/misc.py``), on torch tensors."""
import warnings

import numpy as np
import torch


def _is_iterable(inputs):
    """tfdiffeq/misc.py:162-167"""
    try:
        iter(inputs)
        return True
    except TypeError:
        return False


def _handle_unused_kwargs(solver, unused_kwargs):
    """tfdiffeq/misc.py:178-181: unknown option keys warn, they do not raise."""
    if len(unused_kwargs) > 0:
        warnings.warn('{}: Unexpected arguments {}'.format(solver.__class__.__name__, unused_kwargs))


def _decreasing(t):
    """tfdiffeq/misc.py:153-155 (an empty comparison is True, so a length-1 ``t`` counts as decreasing)."""
    return bool(torch.all(t[1:] < t[:-1]))


def _assert_increasing(t):
    """tfdiffeq/misc.py:158-159"""
    assert bool(torch.all(t[1:] > t[:-1])), 't must be strictly increasing or decrasing'


def _tf_f64(value):
    """``_convert_to_tensor(a, dtype=tf.float64)`` (tfdiffeq/misc.py:137-144): a python float goes through
    ``tf.convert_to_tensor`` first, i.e. through float32.  safety=0.9 really is 0.8999999761581421."""
    if isinstance(value, float):
        return float(np.float64(np.float32(value)))
    if isinstance(value, torch.Tensor):
        return float(value.to(torch.float64))
    return float(value)


def _is_numeric(x):
    return isinstance(x, torch.Tensor) and (x.dtype.is_floating_point or x.dtype.is_complex or x.dtype in (
        torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8))


def _check_inputs(func, y0, t):
    """tfdiffeq/misc.py:290-329: tensor -> 1-tuple wrap, reverse-time wrap, dtype checks."""
    tensor_input = False
    base, sign = func, 1.0
    if isinstance(y0, torch.Tensor):
        tensor_input = True
        y0 = (y0,)
        _base_nontuple_func_ = func
        func = lambda t, y: (_base_nontuple_func_(t, y[0]),)          # noqa: E731
    assert isinstance(y0, tuple), 'y0 must be either a torch.Tensor or a tuple'
    for y0_ in y0:
        assert isinstance(y0_, torch.Tensor), 'each element must be a torch.Tensor but received {}'.format(type(y0_))
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(t)
    if _decreasing(t):
        t = -t
        _base_reverse_func = func
        func = lambda t, y: tuple(-f_ for f_ in _base_reverse_func(-t, y))   # noqa: E731
        sign = -1.0
    for y0_ in y0:
        if not _is_numeric(y0_):
            raise TypeError('`y0` must be a floating point Tensor but is a {}'.format(y0_.dtype))
    if not _is_numeric(t):
        raise TypeError('`t` must be a floating point Tensor but is a {}'.format(t.dtype))
    if tensor_input or getattr(base, "adjoint_rhs", None) is not None:
        # lets a solver recognise a built-in right-hand side behind the wrappers (tfdiffeq_b200/rhs.py), and, for tuple
        # states, odeint_adjoint's augmented dynamics of one (options fused_vjp)
        try:
            func._b2ode_base, func._b2ode_sign = base, sign
        except AttributeError:
            pass
    return tensor_input, func, y0, t
