"""Axis plans of the K7 sums and running sums (np.sum / np.cumsum / np.cumulative_sum along any axis).

A C-ordered array is viewed as (O, R, I) around the axis being reduced or scanned: R is its length, O the product of the
axes before it, I the product of the axes after it.  Pure Python (no torch), so that the operator hooks of
mpyc_b200.resident can decide whether a call is covered before any device work; mpyc_b200.device runs the plans.
"""
import numpy as np


def _prod(xs):
    n = 1
    for x in xs:
        n *= x
    return n


def _axis_index(ndim, a):
    if isinstance(a, (bool, np.bool_)) or not isinstance(a, (int, np.integer)):
        raise TypeError(f'axis must be an integer, not {type(a).__name__}')
    a = int(a)
    if not -ndim <= a < ndim:
        raise ValueError(f'axis {a} is out of bounds for array of dimension {ndim}')
    return a % ndim


def normalize_axes(ndim, axis):
    """None / int / tuple of ints -> sorted tuple of distinct axes in range(ndim); TypeError / ValueError otherwise."""
    if axis is None:
        return tuple(range(ndim))
    items = axis if isinstance(axis, tuple) else (axis,)
    axes = [_axis_index(ndim, a) for a in items]
    if len(set(axes)) != len(axes):
        raise ValueError('duplicate value in axis')
    return tuple(sorted(axes))


def sum_plan(shape, axis=None, keepdims=False):
    """(passes, out_shape) of np.sum(a, axis, keepdims): passes is a list of (O, R, I), run in order on the result of the
    previous pass.  Axes that are adjacent in the shape collapse into one R; other axis sets are reduced one run at a
    time, the largest reduction first (initial belongs to the last pass).  axis=() is one pass with R = 1."""
    shape = tuple(int(s) for s in shape)
    axes = normalize_axes(len(shape), axis)
    runs = []
    for a in axes:
        if runs and runs[-1][1] == a:
            runs[-1][1] = a + 1
        else:
            runs.append([a, a + 1])
    runs.sort(key=lambda r: -_prod(shape[r[0]:r[1]]))
    work = list(shape)
    passes = [] if runs else [(_prod(shape), 1, 1)]
    for lo, hi in runs:
        passes.append((_prod(work[:lo]), _prod(work[lo:hi]), _prod(work[hi:])))
        work[lo:hi] = [1] * (hi - lo)
    out_shape = tuple(work) if keepdims else tuple(s for k, s in enumerate(shape) if k not in axes)
    return passes, out_shape


def scan_plan(shape, axis=None, include_initial=False):
    """((O, R, I), out_shape) of np.cumsum(a, axis) (axis=None: the flattened array) and
    np.cumulative_sum(a, axis=axis, include_initial=...) (one more row along the axis, a zero)."""
    shape = tuple(int(s) for s in shape)
    inc = 1 if include_initial else 0
    if axis is None:
        n = _prod(shape)
        return (1, n, 1), (n + inc,)
    k = _axis_index(len(shape), axis)
    out_shape = shape[:k] + (shape[k] + inc,) + shape[k + 1:]
    return (_prod(shape[:k]), shape[k], _prod(shape[k + 1:])), out_shape
