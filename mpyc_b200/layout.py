"""Layout plans of the K8 copies (NumPy views, joins, reorders and broadcasts of field arrays).

Every plan turns a NumPy operation on C-ordered arrays into copies between strided views (`View`: element offset,
extents, signed element strides, optionally one axis whose offsets come from an index table), with NumPy's own rules for
keys, axes and shapes.  A plan that NumPy would reject, or that the kernels do not cover, is None ("not covered"): the
caller then leaves the operation to NumPy, which raises its own error.  Pure Python (no torch), so that the operator
hooks of mpyc_b200.resident can decide whether a call is covered before any device work; mpyc_b200.device runs the plans.
"""
import numpy as np
from numpy.lib.array_utils import normalize_axis_index, normalize_axis_tuple

MAX_RANK = 6          # MPYC_B200_VIEW_RANK: views have at most this many axes after collapsing


def _prod(xs):
    n = 1
    for x in xs:
        n *= x
    return n


def c_strides(shape):
    st, acc = [], 1
    for s in reversed(shape):
        st.append(acc)
        acc *= s
    return tuple(reversed(st))


class View:
    """Element (c_0, .., c_{r-1}) of the view is at offset + sum_k o_k * strides[k], o_k = index[c_k] on index_axis, else
    c_k."""

    __slots__ = ('offset', 'shape', 'strides', 'index_axis', 'index')

    def __init__(self, offset, shape, strides, index_axis=-1, index=None):
        self.offset, self.shape, self.strides = int(offset), tuple(int(s) for s in shape), tuple(int(s) for s in strides)
        self.index_axis, self.index = index_axis, index

    @classmethod
    def full(cls, shape, offset=0):
        """The C-ordered array of `shape` starting at element `offset`."""
        return cls(offset, shape, c_strides(shape))

    @property
    def size(self):
        return _prod(self.shape)

    def run(self):
        """(start, stop) when the view is one contiguous run of elements in C order, else None."""
        if self.index_axis >= 0:
            return None
        n = self.size
        if n == 0:
            return (0, 0)
        if all(st == c for st, c, e in zip(self.strides, c_strides(self.shape), self.shape) if e != 1):
            return (self.offset, self.offset + n)
        return None

    def axis_range(self, axis, start, stop):
        """The sub-view with coordinates [start, stop) on `axis` (no index axis there)."""
        shape = list(self.shape)
        shape[axis] = stop - start
        return View(self.offset + start * self.strides[axis], shape, self.strides, self.index_axis, self.index)

    def __repr__(self):
        ix = f', index_axis={self.index_axis}' if self.index_axis >= 0 else ''
        return f'View({self.offset}, {self.shape}, {self.strides}{ix})'


# ---- collapsing ---------------------------------------------------------------------------------------------------------

def collapse(*views):
    """Views of equal extents with extent-1 axes dropped and adjacent axes merged where every view is contiguous across
    them (an index axis is never merged).  None if the result has more than MAX_RANK axes."""
    shape = views[0].shape
    if 0 in shape:
        return tuple(View(0, (0,), (1,)) for _ in views)
    offs = [v.offset for v in views]
    keep = []
    for k, e in enumerate(shape):
        if e == 1:
            for j, v in enumerate(views):        # a length-1 axis adds its one offset
                offs[j] += (int(v.index[0]) if k == v.index_axis else 0) * v.strides[k]
        else:
            keep.append(k)
    ext = [shape[k] for k in keep]
    strides = [[v.strides[k] for k in keep] for v in views]
    ix = [keep.index(v.index_axis) if v.index_axis in keep else -1 for v in views]
    k = len(ext) - 2
    while k >= 0:
        if all(ix[j] not in (k, k + 1) and strides[j][k] == strides[j][k + 1] * ext[k + 1] for j in range(len(views))):
            ext[k:k + 2] = [ext[k] * ext[k + 1]]
            for j in range(len(views)):
                strides[j][k:k + 2] = [strides[j][k + 1]]
                if ix[j] > k:
                    ix[j] -= 1
        k -= 1
    if len(ext) > MAX_RANK:
        return None
    return tuple(View(offs[j], ext, strides[j], ix[j], views[j].index if ix[j] >= 0 else None) for j in range(len(views)))


def pieces(items):
    """[(source number, src View, dst View)] collapsed pairwise; None if one does not fit MAX_RANK axes."""
    out = []
    for i, s, d in items:
        c = collapse(s, d)
        if c is None:
            return None
        out.append((i,) + c)
    return out


# ---- indexing -----------------------------------------------------------------------------------------------------------

def _int_key(x):
    return isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))


def _index_array(x):
    """A 1-D integer array / list as int64, False for any other array-like key (not covered), None for a non-array."""
    if isinstance(x, list):
        if not x:
            return np.zeros(0, dtype=np.int64)
        if not all(_int_key(v) for v in x):
            return False
        return np.array(x, dtype=np.int64)
    if isinstance(x, np.ndarray):
        if x.ndim != 1 or x.dtype.kind not in 'iu':
            return False
        return x.astype(np.int64)
    return None


def getitem_plan(shape, key):
    """(src View of the selection, result shape, scalar) of a[key] for a C-ordered a of `shape`, key a NumPy basic-indexing
    key (ints, slices of any step, Ellipsis, None) with at most one 1-D integer array or list; scalar: NumPy returns an
    element rather than a 0-d array.  None if not covered (boolean keys, several arrays, anything NumPy rejects)."""
    shape = tuple(int(s) for s in shape)
    items = list(key) if isinstance(key, tuple) else [key]
    arrays = 0
    for j, x in enumerate(items):
        if x is None or x is Ellipsis or isinstance(x, slice) or _int_key(x):
            continue
        a = _index_array(x)
        if a is None or a is False:
            return None
        items[j] = a
        arrays += 1
    if arrays > 1 or sum(x is Ellipsis for x in items) > 1:
        return None
    if any(isinstance(x, slice) and not all(v is None or _int_key(v) for v in (x.start, x.stop, x.step)) for x in items):
        return None
    used = sum(1 for x in items if x is not None and x is not Ellipsis)
    if used > len(shape):
        return None
    ellipsis = any(x is Ellipsis for x in items)
    if ellipsis:
        j = next(j for j, x in enumerate(items) if x is Ellipsis)
        items[j:j + 1] = [slice(None)] * (len(shape) - used)
    else:
        items += [slice(None)] * (len(shape) - used)
    strides = c_strides(shape)
    offset, d = 0, 0
    out_shape, out_strides, adv = [], [], []
    index, index_pos = None, -1
    for j, x in enumerate(items):
        if x is None:
            out_shape.append(1)
            out_strides.append(0)
            continue
        n = shape[d]
        if isinstance(x, slice):
            if x.step == 0:
                return None
            start, stop, step = x.indices(n)
            ln = len(range(start, stop, step))
            if ln:
                offset += start * strides[d]
            out_shape.append(ln)
            out_strides.append(step * strides[d])
        elif isinstance(x, np.ndarray):
            if x.size and (x.min() < -n or x.max() >= n):
                return None
            index = np.where(x < 0, x + n, x)
            index_pos = len(out_shape)
            out_shape.append(len(x))
            out_strides.append(strides[d])
            adv.append(j)
        else:
            i = int(x)
            if not -n <= i < n:
                return None
            offset += (i % n) * strides[d]
            adv.append(j)
        d += 1
    scalar = not out_shape and not ellipsis
    if index is None:
        return View(offset, out_shape, out_strides), tuple(out_shape), scalar
    # one index array: NumPy puts its axis where the (array and int) indices stand when they are adjacent, else first
    if adv[-1] - adv[0] + 1 != len(adv):
        out_shape.insert(0, out_shape.pop(index_pos))
        out_strides.insert(0, out_strides.pop(index_pos))
        index_pos = 0
    return View(offset, out_shape, out_strides, index_pos, index), tuple(out_shape), False


# ---- axis permutations and reorders -------------------------------------------------------------------------------------

def permuted(shape, perm):
    """The view of a C-ordered array of `shape` with its axes in the order `perm` (a transpose)."""
    st = c_strides(shape)
    return View(0, [shape[k] for k in perm], [st[k] for k in perm])


def transpose_axes(ndim, axes=None):
    """NumPy's axis order of a.transpose(*axes) / np.transpose(a, axes); ValueError / TypeError as NumPy."""
    if axes is None or axes == ():
        return tuple(reversed(range(ndim)))
    if len(axes) == 1 and isinstance(axes[0], (tuple, list)):
        axes = tuple(axes[0])
    if len(axes) == 1 and axes[0] is None:
        return tuple(reversed(range(ndim)))
    if len(axes) != ndim:
        raise ValueError("axes don't match array")
    perm = normalize_axis_tuple(tuple(axes), ndim)
    return perm


def swapaxes_axes(ndim, a1, a2):
    a1, a2 = normalize_axis_index(a1, ndim), normalize_axis_index(a2, ndim)
    perm = list(range(ndim))
    perm[a1], perm[a2] = a2, a1
    return tuple(perm)


def moveaxis_axes(ndim, source, destination):
    """np.moveaxis's axis order."""
    source = normalize_axis_tuple(source, ndim, 'source')
    destination = normalize_axis_tuple(destination, ndim, 'destination')
    if len(source) != len(destination):
        raise ValueError('`source` and `destination` arguments must have the same number of elements')
    order = [n for n in range(ndim) if n not in source]
    for dest, src in sorted(zip(destination, source)):
        order.insert(dest, src)
    return tuple(order)


def flip_view(shape, axis=None):
    """np.flip(a, axis): negative strides on the flipped axes."""
    shape = tuple(shape)
    axes = tuple(range(len(shape))) if axis is None else normalize_axis_tuple(axis, len(shape))
    st = list(c_strides(shape))
    offset = 0
    for k in axes:
        if shape[k]:
            offset += (shape[k] - 1) * st[k]
        st[k] = -st[k]
    return View(offset if 0 not in shape else 0, shape, st)


def roll_plan(shape, shift, axis=None):
    """np.roll(a, shift, axis) for an int shift and axis None / int: [(0, src, dst)] copies into a new array of `shape`
    (two per rolled axis, one when the shift is a multiple of the length)."""
    shape = tuple(shape)
    if axis is None:
        return roll_plan((_prod(shape),), shift, 0)
    k = normalize_axis_index(axis, len(shape))
    n = shape[k]
    s = int(shift) % n if n else 0
    src, dst = View.full(shape), View.full(shape)
    out = [(0, src.axis_range(k, 0, n - s), dst.axis_range(k, s, n))]
    if s:
        out.append((0, src.axis_range(k, n - s, n), dst.axis_range(k, 0, s)))
    return out


# ---- joins --------------------------------------------------------------------------------------------------------------

def concatenate_plan(shapes, axis=0):
    """(out shape, [(i, src, dst)]) of np.concatenate(arrays of `shapes`, axis): each input is one copy into its slab of the
    output.  axis=None joins the flattened inputs.  ValueError / AxisError as NumPy."""
    shapes = [tuple(s) for s in shapes]
    if not shapes:
        raise ValueError('need at least one array to concatenate')
    if axis is None:
        shapes, axis = [(_prod(s),) for s in shapes], 0
    nd = len(shapes[0])
    if nd == 0:
        raise ValueError('zero-dimensional arrays cannot be concatenated')
    if any(len(s) != nd for s in shapes):
        raise ValueError('all the input array dimensions except for the concatenation axis must match exactly')
    k = normalize_axis_index(axis, nd)
    if any(s[:k] + s[k + 1:] != shapes[0][:k] + shapes[0][k + 1:] for s in shapes):
        raise ValueError('all the input array dimensions except for the concatenation axis must match exactly')
    out_shape = shapes[0][:k] + (sum(s[k] for s in shapes),) + shapes[0][k + 1:]
    dst = View.full(out_shape)
    items, at = [], 0
    for i, s in enumerate(shapes):
        items.append((i, View.full(s), dst.axis_range(k, at, at + s[k])))
        at += s[k]
    return out_shape, items


def stack_plan(shapes, axis=0):
    """np.stack: input i goes to the output with coordinate i on the new axis."""
    shapes = [tuple(s) for s in shapes]
    if not shapes:
        raise ValueError('need at least one array to stack')
    if any(s != shapes[0] for s in shapes):
        raise ValueError('all input arrays must have the same shape')
    k = normalize_axis_index(axis, len(shapes[0]) + 1)
    out_shape = shapes[0][:k] + (len(shapes),) + shapes[0][k:]
    st = c_strides(out_shape)
    sub = st[:k] + st[k + 1:]
    return out_shape, [(i, View.full(s), View(i * st[k], s, sub)) for i, s in enumerate(shapes)]


def vstack_shapes(shapes):
    """The shapes np.vstack joins along axis 0 (np.atleast_2d)."""
    return [(1, 1) if len(s) == 0 else ((1,) + tuple(s) if len(s) == 1 else tuple(s)) for s in shapes]


def hstack_axis(shapes):
    """(shapes, axis) np.hstack joins (np.atleast_1d; axis 0 when every input is 1-D, else 1)."""
    shapes = [(1,) if len(s) == 0 else tuple(s) for s in shapes]
    return shapes, 0 if shapes and all(len(s) == 1 for s in shapes) else 1


# ---- broadcasting and reshapes ------------------------------------------------------------------------------------------

def broadcast_views(sa, sb):
    """(out shape, view of a, view of b) of a (op) b under NumPy broadcasting: stride 0 on the broadcast axes."""
    out = np.broadcast_shapes(tuple(sa), tuple(sb))

    def view(s):
        s = tuple(s)
        st = (0,) * (len(out) - len(s)) + c_strides(s)
        s = (1,) * (len(out) - len(s)) + s
        return View(0, out, [0 if e == 1 and o != 1 else t for e, o, t in zip(s, out, st)])
    return out, view(sa), view(sb)


def reshaped(shape, func, *args, **kwargs):
    """The shape np.expand_dims / np.squeeze give an array of `shape` (the elements and their order do not change), with
    NumPy's own argument checks: they run on a stand-in whose every element is one byte of a 1-byte buffer."""
    probe = np.lib.stride_tricks.as_strided(np.zeros(1, np.uint8), tuple(shape), (0,) * len(shape))
    return func(probe, *args, **kwargs).shape
