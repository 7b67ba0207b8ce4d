"""Limb-resident field arrays behind the reference's own FiniteFieldArray objects.

MPyC's field arrays keep a NumPy dtype=object array of Python ints in their `value` slot
(mpyc/finfields.py:695-725) and every protocol step of runtime.py -- local product (`c = a * b`,
runtime.py:1133), `_reshare` (:603-689: np_random_split, pickle, np_recombine), the next product -- goes through
that representation, i.e. through ~40 ns per element of int <-> limb conversion on each side of every kernel.
This module lets the SAME objects carry their elements as limb buffers instead:

  * `LimbValue` is what `array.value` holds while the elements live as limbs (in HBM as a DeviceArray, or in host
    memory as the uint64 (n, L) / uint8 (n,) array the wire delivered).  It answers the questions runtime.py asks
    of `.value` on the protocol path -- shape, reshape(-1), len, pickle -- without creating a single Python int;
    ANY other use (indexing, arithmetic on the raw value as in runtime.py:860-872,3656-3671, iteration, NumPy
    functions through __array__) materialises the object array once and from then on the LimbValue is a plain
    delegate to it: behaviour identical to the reference's, at the reference's cost.
  * install(operators=True) (mpyc_b200/install.py) turns FiniteFieldArray.value into a property over the original
    slot: only the code that is known to treat `.value` as an opaque handle -- runtime._reshare / output /
    _distribute and FiniteFieldArray.reshape / ravel / flatten / copy / shape / ndim / size / __len__ -- ever sees a
    LimbValue; for any other reader the property first settles the slot to the real object ndarray, so raw values
    that escape into isinstance checks, in-place updates or C-level NumPy calls are exactly what the reference has.
    It also wraps FiniteFieldArray.__init__ so that a LimbValue / ShareRow is stored as is, and `+ - * neg @` (finfields.py:1056-1146) so that limb-backed operands -- or plain object
    arrays of at least `min_size` elements -- are combined by the K1 / K1c kernels, the result being limb-backed
    again.  Broadcasting, mixed operand kinds and everything below the threshold stay with the reference's code.
  * with `resident = True` np_recombine / np_pseudorandom_share return limb-backed arrays and np_random_split
    accepts them, so a chain input -> multiply -> reshare -> multiply -> ... -> output creates Python ints only at
    input and at output.
  * `ModValue` (with `resident` and `local_algebra`): Runtime.np_random_bits / np_trunc / np_sgn / np_to_bits -- recognised
    by the hash of their source -- compute on RAW share values between two openings (runtime.py:856-872, 3644-3694,
    4243-4273, 4413-4433).  Their `.value` reads get a ModValue, which evaluates those NumPy expressions mod p on the
    K1 / K6 kernels (csrc/local.cuh) instead of settling; see the class docstring for why that is exact.  The hooks
    around them (<< >>, contiguous __getitem__, np.concatenate(axis=0), == / != with a scalar, matrix/vector row
    broadcast) keep np_prod's halving loop and np_is_zero_public limb-backed as well.  Runtime.np_reciprocal / np_lsb /
    _np_is_zero / np_from_bits get ModValues too: `== 0`, np.count_nonzero and np.where (k_select) run on the limbs.
  * Division, reciprocal, ** by an int, sqrt (Blum primes), is_sqr and np.where of field arrays run on K11 / K1b
    (`divide`, `reciprocal`, `power`, `sqrt`, `is_sqr`, `where` below).

All arithmetic runs on the GPU through the C ABI (`backend` below); there is no CPU path.  tests/oracle_device.py
replaces `backend` by the oracle to exercise this module's host logic where no GPU exists.
"""
import numpy as np

from mpyc_b200 import _cabi, axes, codec, layout
from mpyc_b200.field import context_for, context_of_field
from mpyc_b200.wire import ShareRow, _poly_type

import sys

resident = False      # np_recombine / PRSS results stay limb-backed (set by install(resident=True))
min_size = 1024       # plain object-array operands of fewer elements are left to the reference's operators
public_matmul = False  # @ / np.matmul with a NumPy integer ndarray run on K14 (set by install(public_matmul=True))
calls = {'limb_ops': 0, 'materialised': 0, 'packed': 0, 'mod_values': 0, 'pow_exp': 0, 'prod': 0,
         'matmul_int': 0, 'gf_local': 0}    # counters (tests, profiling); gf_local: K15 calls


# ---------------------------------------------------------------------------------------------
# backend: where the limbs live and which kernels combine them
# ---------------------------------------------------------------------------------------------

class CudaBackend:
    """Stores are mpyc_b200.device.DeviceArray (1-D, n elements) on `device`; host limb arrays are uploaded on
    first use.  torch is imported lazily (device memory and streams only)."""

    def __init__(self, device=0):
        self.device = device

    def _dev(self):
        import torch
        from mpyc_b200 import device as dev
        return dev, torch.device('cuda', self.device)

    def to_store(self, ctx, limbs):
        dev, where = self._dev()
        if isinstance(limbs, dev.DeviceArray):
            return limbs
        return dev.DeviceArray.from_limbs(ctx, np.ascontiguousarray(limbs), where)

    def to_host(self, ctx, store):
        if isinstance(store, np.ndarray):
            return store
        return np.ascontiguousarray(store.to_limbs())

    def binop(self, ctx, op, a, b):
        a, b = self.to_store(ctx, a), self.to_store(ctx, b)
        return a._binop(b, op)

    def binop_scalar(self, ctx, op, a, scalar):
        return self.to_store(ctx, a)._binop(int(scalar), op)

    def neg(self, ctx, a):
        return -self.to_store(ctx, a)

    def matmul(self, ctx, a, b, r, k, c):
        dev, _ = self._dev()
        return dev.matmul(ctx, self.to_store(ctx, a), self.to_store(ctx, b), r, k, c)

    def split(self, ctx, sec, t, m, coeffs=None):
        """sec: store of n secrets -> host limb array (m, n, L) / (m, n): the rows leave for the wire anyway."""
        dev, where = self._dev()
        sec = self.to_store(ctx, sec)
        if coeffs is not None:
            C = dev.DeviceMatrix.empty(ctx, t, sec.n, where) if t else None
            import torch
            for j in range(t):
                src = np.ascontiguousarray(coeffs[j])
                C.t[j].copy_(torch.from_numpy(src if ctx.binary else src.view(np.int64)))
            out = dev.shamir_split(ctx, sec, C, t, m)
        else:
            out = dev.shamir_split_generate(ctx, sec, t, m)
        a = out.t.contiguous().cpu().numpy()
        return a if ctx.binary else a.view(np.uint64)

    def recombine(self, ctx, xs, rows, pts):
        """rows: stores (host limb arrays or DeviceArrays) -> list of len(pts) stores."""
        dev, _ = self._dev()
        rows = [self.to_store(ctx, r) for r in rows]
        out = dev.shamir_recombine(ctx, xs, rows, list(pts))
        return [out.row(r) for r in range(len(pts))]

    # ---- protocol-local algebra (csrc/local.cuh), used by ModValue ----
    def fma(self, ctx, a, b, c):
        dev, _ = self._dev()
        return dev.fma(self.to_store(ctx, a), None if b is None else self.to_store(ctx, b), self.to_store(ctx, c))

    def axpb(self, ctx, a, s, t):
        dev, _ = self._dev()
        return dev.axpb(self.to_store(ctx, a), s, t)

    def low_bits(self, ctx, a, nbits):
        dev, _ = self._dev()
        return dev.low_bits(self.to_store(ctx, a), nbits)

    def nonzero(self, ctx, a, want_mask=True):
        """(bool ndarray a != 0, count); want_mask=False: (None, count), nothing but the count crosses to the host"""
        dev, _ = self._dev()
        mask, count = dev.nonzero(self.to_store(ctx, a), want_mask)
        return (mask.cpu().numpy() if want_mask else None), count

    def bits_compose(self, ctx, bits, n, f, descending):
        dev, _ = self._dev()
        return dev.bits_compose(self.to_store(ctx, bits), n, f, descending)

    def sqrt(self, ctx, a, INV):
        return self.to_store(ctx, a).sqrt(INV=INV)

    def bits_decompose(self, ctx, c, l, descending):
        """store of l*n elements, row-major (l, n)"""
        dev, _ = self._dev()
        return dev.bits_decompose_flat(self.to_store(ctx, c), l, descending)

    def transpose(self, ctx, a, rows, cols):
        dev, _ = self._dev()
        return dev.transpose(self.to_store(ctx, a), rows, cols)

    def cumsum_rows(self, ctx, a, rows, cols):
        dev, _ = self._dev()
        return dev.cumsum_rows(self.to_store(ctx, a), rows, cols)

    def binop_rows(self, ctx, op, a, b, rows, cols, reflected):
        dev, _ = self._dev()
        return dev.binop_rows(self.to_store(ctx, a), self.to_store(ctx, b), op, rows, cols, reflected)

    def sum_axis(self, ctx, a, shape, axis, keepdims, initial):
        """store of the elements of np.sum(a.reshape(shape), axis, keepdims=keepdims, initial=initial) mod p"""
        dev, _ = self._dev()
        return dev.sum_axis(self.to_store(ctx, a), shape, axis, keepdims, initial)[0]

    def cumsum_axis(self, ctx, a, shape, axis, include_initial):
        dev, _ = self._dev()
        return dev.cumsum_axis(self.to_store(ctx, a), shape, axis, include_initial)[0]

    def copy_view(self, ctx, n, base, items):
        """A new store of n elements: a copy of the store `base` (None: uninitialised), then dst_view <- src_view for each
        (src store, src View, dst View) of `items` (K8; views of mpyc_b200.layout)."""
        dev, where = self._dev()
        if base is not None:
            out = dev.DeviceArray(ctx, self.to_store(ctx, base).t.clone())
        else:
            out = dev.DeviceArray.empty(ctx, n, where)
        for st, sv, dv in items:
            dev.copy_view(self.to_store(ctx, st), sv, out, dv)
        return out

    def binop_view(self, ctx, op, a, a_view, b, b_view):
        """store of a[a_view] (op) b[b_view] in C order of the views' (broadcast) extents (K8)"""
        dev, _ = self._dev()
        return dev.binop_view(self.to_store(ctx, a), a_view, self.to_store(ctx, b), b_view, op)

    def det(self, ctx, a, batch, n):
        """store of the batch determinants of a (batch x n x n) (K9)"""
        dev, _ = self._dev()
        return dev.det(self.to_store(ctx, a), batch, n)

    def solve(self, ctx, a, n, b, nrhs):
        """store of X (n x nrhs) with a X = b; b None: the inverse of a.  ZeroDivisionError for a singular a (K9)"""
        dev, _ = self._dev()
        return dev.solve(self.to_store(ctx, a), None if b is None else self.to_store(ctx, b), n, nrhs)

    def matrix_power(self, ctx, a, n, e):
        dev, _ = self._dev()
        return dev.matrix_power(self.to_store(ctx, a), n, e)

    def convolve(self, ctx, a, m, b, n, lo, count):
        """store of full[lo : lo + count] of the convolution of a (m) and b (n) (K10)"""
        dev, _ = self._dev()
        return dev.convolve(ctx, self.to_store(ctx, a), m, self.to_store(ctx, b), n, lo, count)

    # ---- K11 and K1b, used by the division / selection hooks and ModValue ----
    def divide(self, ctx, num, den):
        """store of num / den elementwise (ZeroDivisionError for a zero in den)"""
        dev, _ = self._dev()
        return dev.divide(self.to_store(ctx, num), self.to_store(ctx, den))

    def inverse(self, ctx, a):
        return self.to_store(ctx, a).reciprocal()

    def power(self, ctx, a, e):
        """store of a ** e for a Python int e (negative: of the inverse; ZeroDivisionError for a zero then)"""
        return self.to_store(ctx, a) ** e

    def is_sqr(self, ctx, a):
        """bool ndarray: a is a square (0 counts as one), K1b"""
        return self.to_store(ctx, a).is_sqr().cpu().numpy()

    def select(self, ctx, mask, x, x_map, y, y_map, n):
        """store of mask ? x * sx + tx : y * sy + ty (x_map = (sx, tx), y_map = (sy, ty); a side None: its constant t).
        mask: a host bool ndarray of n entries (uploaded), or a store whose nonzero elements select x -- that mask is built
        by k_nonzero on the device and never crosses to the host."""
        dev, _ = self._dev()
        if not (isinstance(mask, np.ndarray) and mask.dtype == bool):
            mask = dev.nonzero_mask(self.to_store(ctx, mask))
        x = None if x is None else self.to_store(ctx, x)
        y = None if y is None else self.to_store(ctx, y)
        return dev.select(mask, x, x_map, y, y_map, n)

    # ---- K12, used by the per-element exponent hooks ----
    def pow_exp(self, ctx, base, exps, signs, bits):
        """store of base(h)^e[h]: base a store (one base per element, signs None) or a Python int (one public base);
        exps, signs, bits as codec.exponents_to_limbs returns them (ZeroDivisionError for a zero int base with signs)"""
        dev, where = self._dev()
        if not isinstance(base, int):
            base = self.to_store(ctx, base)
        return dev.pow_exp(ctx, base, exps, signs, bits, device=where)

    # ---- K13, used by the np.prod / np.cumprod / np.all / np.any hooks ----
    def prod_axis(self, ctx, a, shape, axis, keepdims, initial):
        """store of the elements of np.prod(a.reshape(shape), axis, keepdims=keepdims, initial=initial) mod p"""
        dev, _ = self._dev()
        return dev.prod_axis(self.to_store(ctx, a), shape, axis, keepdims, initial)[0]

    def cumprod_axis(self, ctx, a, shape, axis, include_initial):
        dev, _ = self._dev()
        return dev.cumprod_axis(self.to_store(ctx, a), shape, axis, include_initial)[0]

    def all_any_axis(self, ctx, a, shape, axis, keepdims, any):
        """store of np.all / np.any (any) of a.reshape(shape) along axis as elements 0 / 1"""
        dev, _ = self._dev()
        return dev.all_any_axis(self.to_store(ctx, a), shape, axis, keepdims, any)[0]

    # ---- K14, used by matmul with an integer ndarray operand ----
    def matmul_int(self, ctx, x, w, r, k, c, w_left):
        """store of x @ w (w_left: w @ x) mod p, x a store of r*k (w_left: k*c) elements, w a NumPy integer array"""
        dev, _ = self._dev()
        return dev.matmul_int(ctx, self.to_store(ctx, x), w, r, k, c, w_left)

    # ---- K15, used by the GF(2^8) hooks and ModValue in np_to_bits / np_from_bits ----
    def gf_bits_compose(self, ctx, bits, n, l):
        """store of sum_j bits[i l + j] X^j mod poly for i < n"""
        dev, _ = self._dev()
        return dev.gf_bits_compose(self.to_store(ctx, bits), n, l)

    def gf_binop_view(self, ctx, op, a, a_view, b, b_view):
        """store of a[a_view] (op) b[b_view] over GF(2^8) in C order of the views' (broadcast) extents"""
        dev, _ = self._dev()
        return dev.gf_binop_view(self.to_store(ctx, a), a_view, self.to_store(ctx, b), b_view, op)

    def gf_matmul_batched(self, ctx, a, a_stacked, b, b_stacked, batch, r, k, c):
        """store of the batch products A[b] @ B[b]; a side that is not stacked holds one matrix for every b"""
        dev, _ = self._dev()
        return dev.gf_matmul_batched(self.to_store(ctx, a), a_stacked, self.to_store(ctx, b), b_stacked, batch, r, k, c)

    def conv2d(self, ctx, X, W, B, k, r, m, n, v, s):
        dev, _ = self._dev()
        return dev.conv2d(self.to_store(ctx, X), self.to_store(ctx, W), self.to_store(ctx, B), k, r, m, n, v, s)

    def slice(self, ctx, store, start, stop):
        if isinstance(store, np.ndarray):
            return store[start:stop]
        dev, _ = self._dev()
        return dev.DeviceArray(ctx, store.t[start:stop])

    def concat(self, ctx, stores):
        """One store holding the elements of `stores` back to back (device-to-device copies; torch is the allocator)."""
        dev, _ = self._dev()
        parts = [self.to_store(ctx, st) for st in stores]
        out = dev.DeviceArray.empty(ctx, sum(p.n for p in parts), parts[0].t.device)
        at = 0
        for p in parts:                       # contiguous device-to-device copies (cudaMemcpyAsync)
            out.t[at:at + p.n].copy_(p.t)
            at += p.n
        return out


backend = CudaBackend()


# ---------------------------------------------------------------------------------------------
# LimbValue
# ---------------------------------------------------------------------------------------------

def _norm_shape(n, shape):
    if len(shape) == 1 and isinstance(shape[0], (tuple, list)):
        shape = tuple(shape[0])
    shape = tuple(int(s) for s in shape)
    if shape.count(-1) > 1:
        raise ValueError('can only specify one unknown dimension')
    if -1 in shape:
        known = 1
        for s in shape:
            if s != -1:
                known *= s
        if known == 0 or n % known:
            raise ValueError(f'cannot reshape array of size {n} into shape {shape}')
        shape = tuple(n // known if s == -1 else s for s in shape)
    size = 1
    for s in shape:
        size *= s
    if size != n:
        raise ValueError(f'cannot reshape array of size {n} into shape {shape}')
    return shape


class LimbValue:
    """The `value` of a field array whose elements live as limbs (see module docstring).

    store: DeviceArray or host limb array holding prod(shape) elements in C order; immutable by convention (every
    operation produces a new store), so reshape / ravel / copy share it."""

    __slots__ = ('ctx', 'shape', 'store', '_ints', '_poly')
    __array_priority__ = 0.0
    __hash__ = None

    def __init__(self, ctx, store, shape=None, poly_type=None):
        self.ctx = ctx
        self.store = store
        n = len(store)
        self.shape = (n,) if shape is None else tuple(shape)
        self._ints = None
        self._poly = poly_type

    # ---- what the protocol path of runtime.py asks of `.value` (no Python ints are created) -------------
    @property
    def limb_backed(self):
        return self.store is not None

    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        n = 1
        for s in self.shape:
            n *= s
        return n

    dtype = np.dtype(object)

    def __len__(self):
        if not self.shape:
            raise TypeError('len() of unsized object')
        return self.shape[0]

    def reshape(self, *shape, **kwargs):
        # order='C' (Runtime.np_reshape passes it, runtime.py:2746) is the order the limbs are in
        if self.store is None or (kwargs and kwargs != {'order': 'C'}):
            return self._materialise().reshape(*shape, **kwargs)
        return LimbValue(self.ctx, self.store, _norm_shape(self.size, shape), self._poly)

    def ravel(self, *args, **kwargs):
        if self.store is None or args or kwargs:
            return self._materialise().ravel(*args, **kwargs)
        return LimbValue(self.ctx, self.store, (self.size,), self._poly)

    def flatten(self, *args, **kwargs):
        if self.store is None or args or kwargs:
            return self._materialise().flatten(*args, **kwargs)
        return LimbValue(self.ctx, self.store, (self.size,), self._poly)

    def copy(self, *args, **kwargs):
        if self.store is None:
            return self._ints.copy(*args, **kwargs)
        return LimbValue(self.ctx, self.store, self.shape, self._poly)

    def host_limbs(self):
        """The elements as a host limb array (n, L) / (n,) (one D2H copy when they are in HBM)."""
        return backend.to_host(self.ctx, self.store)

    def __reduce__(self):
        if self.store is None:
            return _from_ints, (self._ints,)
        return _from_wire, (self.ctx.modulus, self.ctx.binary, self.shape, codec.limbs_to_wire(self.host_limbs(), self.ctx))

    # ---- everything else: become the object array the reference would have had ---------------------------
    def _materialise(self):
        if self._ints is None:
            vals = codec.limbs_to_ints(self.host_limbs(), self.ctx)
            if self.ctx.binary:
                tp = self._poly or _poly_type()
                out = np.empty(len(vals), dtype=object)
                out[:] = [tp(int(v)) for v in vals]
                vals = out
            self._ints = vals.reshape(self.shape)
            self.store = None        # the ints may be modified in place from here on: the limbs are dropped
            calls['materialised'] += 1
        return self._ints

    def __array__(self, dtype=None, copy=None):
        a = self._materialise()
        if dtype is not None and dtype != object:
            return a.astype(dtype)
        return a.copy() if copy else a

    def __getattr__(self, name):
        if name.startswith('__') and name.endswith('__'):
            raise AttributeError(name)
        return getattr(self._materialise(), name)

    def __repr__(self):
        if self.store is None:
            return repr(self._ints)
        where = 'host' if isinstance(self.store, np.ndarray) else 'device'
        return f'LimbValue(shape={self.shape}, {where}, {self.ctx!r})'


def _delegate(name):
    def method(self, *args, **kwargs):
        return getattr(self._materialise(), name)(*args, **kwargs)
    method.__name__ = name
    return method


for _name in ('getitem', 'setitem', 'iter', 'contains', 'add', 'radd', 'iadd', 'sub', 'rsub', 'isub', 'mul', 'rmul', 'imul',
              'matmul', 'rmatmul', 'imatmul', 'mod', 'rmod', 'imod', 'floordiv', 'rfloordiv', 'ifloordiv', 'truediv',
              'rtruediv', 'itruediv', 'pow', 'rpow', 'ipow', 'neg', 'pos', 'abs', 'invert', 'lshift', 'rlshift', 'ilshift',
              'rshift', 'rrshift', 'irshift', 'and', 'rand', 'iand', 'or', 'ror', 'ior', 'xor', 'rxor', 'ixor', 'lt', 'le',
              'gt', 'ge', 'eq', 'ne', 'bool', 'int', 'index', 'float', 'divmod', 'rdivmod', 'str', 'format'):
    setattr(LimbValue, f'__{_name}__', _delegate(f'__{_name}__'))



# ---------------------------------------------------------------------------------------------
# ModValue: raw-value algebra of whitelisted protocol functions, mod p on the device
# ---------------------------------------------------------------------------------------------

class ModValue:
    """What `array.value` returns to np_random_bits / np_trunc / np_sgn / np_to_bits (`_MOD_SOURCES`) while the elements are
    limbs.

    Those functions compute on raw share values with NumPy object arithmetic -- `_r.value**2 + z.value`,
    `np.sum(r_bits.value.reshape((n, f)) << np.arange(f), axis=1)`, `ar_modf + (1 << l-1) + (r_divf << f)`,
    `c.value & ((1<<f) - 1)`, `bits += 1; bits *= (p+1) >> 1` (mpyc/runtime.py:856-872, 3644-3658, 4252-4271) -- over
    the integers, and reduce when the result enters `Zp.array(...)`.  A ModValue runs the same expressions mod p on the
    K1 / K6 kernels: reduction is a ring homomorphism, so the field array that comes out is identical.  Operations that
    are not ring operations (`&`, `!= 0`, `%` by a power of two) are only accepted on EXACT values -- residues read
    straight from a field array (an opened value) -- where the canonical residue IS the reference's integer; on a
    modular intermediate they raise instead of returning something that could differ.

    Scalar steps are kept as a pending affine map (value = store * s + t) and applied by one k_axpb launch when the
    elements are needed.  Anything not covered here turns the value into the settled object array (canonical
    residues) and continues with NumPy, like LimbValue."""

    __slots__ = ('ctx', 'shape', 'store', '_s', '_t', '_sq', 'exact', '_ints')
    __hash__ = None
    dtype = np.dtype(object)
    # sectypes.SecureArray subclasses accept raw values only as `isinstance(value, np.ndarray)` (sectypes.py:1402,1440)
    # and then hand them to `field.array(value)` -- which is hooked and takes the limbs.  isinstance() consults
    # __class__; type() -- which every check in this package uses -- does not.  NumPy's C code is not fooled either
    # (PyArray_Check looks at the type), it goes through __array__ / __array_ufunc__ / __array_function__ below.
    __class__ = property(lambda self: np.ndarray)

    def __init__(self, ctx, store, shape, exact=False, s=1, t=0, sq=False):
        self.ctx, self.store, self.shape = ctx, store, tuple(shape)
        self._s, self._t, self._sq = s, t, sq
        self.exact = exact and s == 1 and t == 0 and not sq
        self._ints = None

    # ---- plumbing ---------------------------------------------------------------------------------
    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        n = 1
        for d in self.shape:
            n *= d
        return n

    def __len__(self):
        if not self.shape:
            raise TypeError('len() of unsized object')
        return self.shape[0]

    def _flush(self):
        """Apply the pending square / affine map; afterwards store holds the canonical residues of the value."""
        if self._sq:
            self.store = backend.binop(self.ctx, _cabi.OP_MUL, self.store, self.store)
            self._sq = False
            calls['limb_ops'] += 1
        if self._s != 1 or self._t != 0:
            self.store = backend.axpb(self.ctx, self.store, self._s, self._t)
            self._s, self._t = 1, 0
            calls['limb_ops'] += 1
        return self.store

    def limb_value(self):
        """The value as a LimbValue (for FiniteFieldArray.__init__), or None once it has become an object array."""
        if self.store is None:
            return None
        return LimbValue(self.ctx, self._flush(), self.shape)

    def _new(self, store, shape=None, exact=False, s=1, t=0, sq=False):
        return ModValue(self.ctx, store, self.shape if shape is None else shape, exact, s, t, sq)

    def _materialise(self):
        if self._ints is None:
            lv = LimbValue(self.ctx, self._flush(), self.shape)
            self._ints = lv._materialise()
            self.store = None
        return self._ints

    def __array__(self, dtype=None, copy=None):
        a = self._materialise()
        if dtype is not None and dtype != object:
            return a.astype(dtype)
        return a.copy() if copy else a

    def __getattr__(self, name):
        if name.startswith('__') and name.endswith('__'):
            raise AttributeError(name)
        return getattr(self._materialise(), name)

    def __repr__(self):
        if self.store is None:
            return repr(self._ints)
        return f'ModValue(shape={self.shape}, exact={self.exact}, {self.ctx!r})'

    def __reduce__(self):
        return _from_ints, (self._materialise(),)

    def reshape(self, *shape, **kwargs):
        if self.store is None or kwargs:
            return self._materialise().reshape(*shape, **kwargs)
        return self._new(self.store, _norm_shape(self.size, shape), self.exact, self._s, self._t, self._sq)

    @property
    def T(self):
        """`r_bits.T` (runtime.py:3661): a 2-D value is transposed on the device (k_transpose)."""
        if self.store is not None and len(self.shape) == 2 and not self.ctx.binary:
            r, c = self.shape
            calls['limb_ops'] += 1
            return self._new(backend.transpose(self.ctx, self._flush(), r, c), (c, r), self.exact)
        return self._materialise().T

    def ravel(self, *args, **kwargs):
        if self.store is None or args or kwargs:
            return self._materialise().ravel(*args, **kwargs)
        return self.reshape(-1)

    flatten = ravel

    def copy(self, *args, **kwargs):
        if self.store is None:
            return self._ints.copy(*args, **kwargs)
        return self._new(self.store, None, self.exact, self._s, self._t, self._sq)

    def __getitem__(self, key):
        if (self.store is not None and len(self.shape) == 1 and isinstance(key, slice) and key.step in (None, 1)):
            start, stop, _ = key.indices(self.shape[0])
            stop = max(stop, start)
            return self._new(backend.slice(self.ctx, self._flush(), start, stop), (stop - start,), self.exact)
        return self._materialise()[key]

    def __setitem__(self, key, value):
        self._materialise()[key] = value

    def __iter__(self):
        return iter(self._materialise())

    # ---- ring operations ----------------------------------------------------------------------------
    def _scalar(self, x):
        return int(x) if isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_)) else None

    def _other_store(self, other, shape=None):
        """Store of an array operand of the given shape (default: this value's), packed from ints if need be; else None."""
        shape = self.shape if shape is None else tuple(shape)
        if type(other) is ModValue:
            if other.store is None:
                other = other._ints
            elif other.ctx is self.ctx and other.shape == shape:
                return other._flush()
            else:
                return None
        if type(other) is LimbValue:
            if other.store is not None:
                return other.store if (other.ctx is self.ctx and other.shape == shape) else None
            other = other._ints
        if type(other) is np.ndarray and other.shape == shape and other.dtype.kind in 'Oiu' and other.size:
            calls['packed'] += 1
            if other.dtype != object:
                other = other.astype(object)
            return codec.ints_to_limbs(other.reshape(-1), self.ctx)      # reduces: raw values may be negative / >= p
        return None

    def _ring(self, other, op, reflected=False):
        """self (op) other, op in '+', '-', '*'; reflected: other (op) self."""
        if self.store is None:
            return _NUMPY_OPS[op](other, self._ints) if reflected else _NUMPY_OPS[op](self._ints, other)
        if self.ctx.binary:
            return self._gf_ring(other, op, reflected)
        p = self.ctx.modulus
        k = self._scalar(other)
        if k is not None:
            s, t = self._s, self._t
            if self._sq:
                self._flush()
                s, t = 1, 0
            if op == '+':
                t = (t + k) % p
            elif op == '-':
                s, t = ((-s) % p, (k - t) % p) if reflected else (s, (t - k) % p)
            else:
                s, t = (s * k) % p, (t * k) % p
            return self._new(self.store, None, False, s, t)
        b = self._other_store(other)
        if b is None:
            r = self._ring_rows(other, op, reflected)
            if r is not None:
                return r
            a = self._materialise()
            return _NUMPY_OPS[op](other, a) if reflected else _NUMPY_OPS[op](a, other)
        calls['limb_ops'] += 1
        if op == '+' and self._sq and self._s == 1 and self._t == 0:                      # a*a + c in one pass
            return self._new(backend.fma(self.ctx, self.store, None, b))
        a = self._flush()
        code = {'+': _cabi.OP_ADD, '-': _cabi.OP_SUB, '*': _cabi.OP_MUL}[op]
        x, y = (b, a) if reflected else (a, b)
        return self._new(backend.binop(self.ctx, code, x, y))

    def _gf_ring(self, other, op, reflected):
        """GF(2^8): + and - of two values of one shape are XOR (`field_array + r_modl`, runtime.py:4418); anything else
        settles."""
        if op in '+-' and type(other) in (ModValue, LimbValue) and other.store is not None and other.ctx is self.ctx \
                and other.shape == self.shape:
            calls['limb_ops'] += 1
            return self._new(backend.binop(self.ctx, _cabi.OP_ADD, self.store, other._flush() if type(other) is ModValue else other.store))
        a = self._materialise()
        return _NUMPY_OPS[op](other, a) if reflected else _NUMPY_OPS[op](a, other)

    def _ring_rows(self, other, op, reflected):
        """NumPy's row broadcast between a vector (C,) and a matrix (R, C) -- `s_sign - <matrix>` (runtime.py:3670)."""
        oshape = getattr(other, 'shape', None)
        if oshape is None or not self.shape:
            return None
        if len(self.shape) == 1 and len(oshape) == 2 and oshape[1] == self.shape[0]:
            vec, mat, vec_is_self = self, other, True
        elif len(self.shape) == 2 and len(oshape) == 1 and oshape[0] == self.shape[1]:
            vec, mat, vec_is_self = other, self, False
        else:
            return None
        R, C = mat.shape
        if R == 0 or C == 0:
            return None
        other_store = self._other_store(other, oshape)
        if other_store is None:
            return None
        mine = self._flush()
        mstore, vstore = (other_store, mine) if vec_is_self else (mine, other_store)
        code = {'+': _cabi.OP_ADD, '-': _cabi.OP_SUB, '*': _cabi.OP_MUL}[op]
        # kernel computes matrix (op) vector, or vector (op) matrix when `refl`
        refl = (vec_is_self and not reflected) or (not vec_is_self and reflected)
        calls['limb_ops'] += 1
        return ModValue(self.ctx, backend.binop_rows(self.ctx, code, mstore, vstore, R, C, refl), (R, C))

    def __add__(self, other):
        return self._ring(other, '+')

    __radd__ = __iadd__ = __add__

    def __sub__(self, other):
        return self._ring(other, '-')

    __isub__ = __sub__

    def __rsub__(self, other):
        return self._ring(other, '-', reflected=True)

    def __mul__(self, other):
        return self._ring(other, '*')

    __rmul__ = __imul__ = __mul__

    def __neg__(self):
        return self._ring(-1, '*')

    def __pos__(self):
        return self

    def __pow__(self, e):
        if self.store is not None and self._scalar(e) == 2 and not self._sq and not self.ctx.binary:
            self._flush()
            return self._new(self.store, None, False, sq=True)
        return self._materialise() ** e

    def __lshift__(self, k):
        if self.store is None:
            return self._ints << k
        n = self._scalar(k)
        if n is not None and n >= 0 and not self.ctx.binary:
            return self._ring(pow(2, n, self.ctx.modulus), '*')
        if (isinstance(k, np.ndarray) and type(k) is np.ndarray and k.ndim == 1 and k.dtype.kind in 'iu' and len(self.shape) >= 2
                and k.shape[0] == self.shape[-1] and k.shape[0] > 0 and self.size):
            f = k.shape[0]
            if np.array_equal(k, np.arange(f)):
                return _ShiftedBits(self, k, False)
            if np.array_equal(k, np.arange(f - 1, -1, -1)) and not self.ctx.binary:
                return _ShiftedBits(self, k, True)
        return self._materialise() << k

    __ilshift__ = __lshift__

    def sqrt(self, INV=False):
        """PrimeFieldArray._sqrt on the limbs (Blum primes; finfields.py:1424-1438): an exact value again."""
        return self._new(backend.sqrt(self.ctx, self._flush(), INV), None, True)

    # ---- operations that are not ring operations: exact values only -----------------------------------------
    def _need_exact(self, what):
        if not self.exact:
            raise AssertionError(f'mpyc_b200: {what} on a modular intermediate (only opened / stored residues are exact)')

    def __and__(self, mask):
        if self.store is None or self.ctx.binary:
            return self._materialise() & mask
        m = self._scalar(mask)
        if m is not None and m >= 0 and (m + 1) & m == 0:           # 2^b - 1
            self._need_exact('bit mask')
            calls['limb_ops'] += 1
            return self._new(backend.low_bits(self.ctx, self.store, m.bit_length()), None, True)
        self._need_exact('bitwise and')
        return self._materialise() & mask

    __rand__ = __and__

    def __mod__(self, q):
        if self.store is None or self.ctx.binary:
            return self._materialise() % q
        m = self._scalar(q)
        if m == self.ctx.modulus:
            return self if not self._sq and self._s == 1 and self._t == 0 else self._new(self._flush())
        if m is not None and m > 0 and m & (m - 1) == 0:
            return self & (m - 1)
        self._need_exact('%')
        return self._materialise() % q

    __imod__ = __mod__

    def __ne__(self, other):
        if self.store is not None and self.ctx.binary:
            return self._materialise() != other
        if self.store is not None and self._scalar(other) == 0:
            self._need_exact('!= 0')
            mask, _ = backend.nonzero(self.ctx, self.store)
            return np.asarray(mask, dtype=bool).reshape(self.shape)
        if self.store is not None:
            self._need_exact('comparison')
        return self._materialise() != other

    def __eq__(self, other):
        if self.store is not None and self.ctx.binary:
            return self._materialise() == other
        if self.store is not None and self._scalar(other) == 0:
            self._need_exact('== 0')                               # `c.value == 0` (runtime.py:3614)
            mask, _ = backend.nonzero(self.ctx, self.store)
            return ~np.asarray(mask, dtype=bool).reshape(self.shape)
        if self.store is not None:
            self._need_exact('comparison')
        return self._materialise() == other

    # ---- NumPy protocol: `ndarray (op) ModValue` and direct ufunc calls -----------------------------------------
    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        if method == '__call__' and len(inputs) == 2 and not kwargs and ufunc in _UFUNC_OPS:
            a, b = inputs
            if a is self:
                return self._ring(b, _UFUNC_OPS[ufunc]) if ufunc is not np.left_shift else self.__lshift__(b)
            if ufunc is not np.left_shift:
                return self._ring(a, _UFUNC_OPS[ufunc], reflected=True)
        if (method == 'outer' and ufunc is np.right_shift and len(inputs) == 2 and not kwargs and inputs[0] is self
                and self.store is not None and len(self.shape) == 1 and self.exact and not self.ctx.binary):
            k = inputs[1]
            if isinstance(k, np.ndarray) and type(k) is np.ndarray and k.ndim == 1 and k.dtype.kind in 'iu' and k.shape[0] > 0:
                l = k.shape[0]
                if np.array_equal(k, np.arange(l)):
                    return _OuterBits(self, k, False, False)
                if np.array_equal(k, np.arange(l - 1, -1, -1)):
                    return _OuterBits(self, k, True, False)
        if method in ('__call__', 'outer') and ufunc in (np.right_shift, np.bitwise_and, np.not_equal, np.equal, np.remainder):
            for x in inputs:
                if type(x) is ModValue and x.store is not None and not x.ctx.binary:
                    x._need_exact(ufunc.__name__)
        args = [x._materialise() if type(x) in (ModValue, LimbValue) else x for x in inputs]
        if 'out' in kwargs:
            kwargs['out'] = tuple(x._materialise() if type(x) in (ModValue, LimbValue) else x for x in kwargs['out'])
        return getattr(ufunc, method)(*args, **kwargs)

    def __array_function__(self, func, types, args, kwargs):
        """np.vstack / np.cumsum(axis=0) of 2-D values stay on the device (runtime.py:3667-3670); every other NumPy
        function gets the settled object arrays."""
        if self.ctx.binary:
            return func(*_settled(args), **_settled(kwargs))
        if func is np.vstack and len(args) == 1 and not kwargs:
            r = _vstack(self.ctx, args[0])
            if r is not None:
                return r
        elif (func is np.cumsum and len(args) == 1 and args[0] is self and kwargs == {'axis': 0} and self.store is not None
              and len(self.shape) == 2 and self.size):
            calls['limb_ops'] += 1
            return self._new(backend.cumsum_rows(self.ctx, self._flush(), self.shape[0], self.shape[1]))
        elif func is np.count_nonzero and len(args) == 1 and args[0] is self and not kwargs and self.store is not None:
            self._need_exact('np.count_nonzero')                   # `np.count_nonzero(ar.value)` (runtime.py:1282)
            calls['limb_ops'] += 1
            return _count_nonzero(self.ctx, self.store)
        elif func is np.where and len(args) == 3 and not kwargs:
            r = _where(self.ctx, None, *args)
            if r is not None:
                return r
        return func(*_settled(args), **_settled(kwargs))


def _count_nonzero(ctx, store):
    """The number of nonzero elements of a store (k_nonzero; only the count crosses when the backend has K11)."""
    if _divsel_backend():
        return backend.nonzero(ctx, store, want_mask=False)[1]
    return int(backend.nonzero(ctx, store)[1])


def _array_class(x):
    """type(x) when x is an array of a patched FiniteFieldArray class, else None."""
    return type(x) if _slot is not None and isinstance(x, _slot.__objclass__) else None


def _where_side(ctx, cls, x, shape):
    """(store or None, s, t) for one side of np.where: the side's value is store * s + t, or the constant t when store is
    None.  x: a ModValue (its pending affine map is passed on), a limb-backed value, an array of cls (limb-backed, or of
    Python ints when it has at least min_size elements), an int or a field element of cls (reduced mod p, as the
    reference's cls(.) does).  None for anything else."""
    p = ctx.modulus
    if type(x) is ModValue:
        if x.store is None or x.ctx is not ctx or x.shape != shape:
            return None
        if x._sq:
            x._flush()
        return x.store, x._s, x._t
    if type(x) is LimbValue:
        return (x.store, 1, 0) if x.store is not None and x.ctx is ctx and x.shape == shape else None
    xc = _array_class(x)
    if xc is not None:
        if cls is None:
            cls = xc
        if xc is not cls or _ctx_of(xc) is not ctx:
            return None
        lv = as_limb_value(raw_value(x))
        if lv is not None:
            return (lv.store, 1, 0) if lv.shape == shape else None
        if np.shape(raw_value(x)) != shape:
            return None
        op = _operand(ctx, cls, x)
        return None if op is None else (op[0], 1, 0)
    if cls is not None and isinstance(x, cls.field):
        x = x.value
    if type(x) is int:
        return None, 1, x % p
    return None


def _where(ctx, cls, cond, x, y):
    """np.where(cond, x, y) on k_select for a condition of the result's shape -- a host bool / integer ndarray, or an exact
    ModValue / limb-backed LimbValue whose != 0 mask k_nonzero builds on the device -- and sides of _where_side, at least
    one of them an array.  The result is what the reference returns: an array of the sides' FiniteFieldArray class when
    one side is such an array (FiniteFieldArray.__array_function__ wraps np.where's result, finfields.py:801-807), else a
    (non-exact) ModValue for the object ndarray np.where makes of raw values.  None leaves the call to NumPy on the
    settled values (and always without K11)."""
    if not _divsel_backend() or ctx.binary:
        return None
    if type(cond) is ModValue or type(cond) is LimbValue:
        if cond.store is None or cond.ctx is not ctx:
            return None
        if type(cond) is ModValue:
            cond._need_exact('np.where condition')
        shape, mask = cond.shape, cond.store
    elif type(cond) is np.ndarray and cond.dtype.kind in 'biu':
        shape, mask = cond.shape, (cond != 0).reshape(-1)
    else:
        return None
    n = layout._prod(shape)
    if n == 0:
        return None
    sides = [_where_side(ctx, cls, v, shape) for v in (x, y)]
    if any(sd is None for sd in sides) or all(sd[0] is None for sd in sides):
        return None
    calls['limb_ops'] += 1
    (xs, sx, tx), (ys, sy, ty) = sides
    store = backend.select(ctx, mask, xs, (sx, tx), ys, (sy, ty), n)
    out_cls = cls or _array_class(x) or _array_class(y)
    if out_cls is not None:
        return _wrap(out_cls, ctx, store, shape)
    return ModValue(ctx, store, shape)


def _settled(x):
    """x with every ModValue / LimbValue inside (tuples, lists, dicts) replaced by its object array."""
    if type(x) in (ModValue, LimbValue):
        return x._materialise()
    if type(x) is _OuterBits or type(x) is _ShiftedBits:
        return x._eval()
    if isinstance(x, tuple):
        return tuple(_settled(v) for v in x)
    if isinstance(x, list):
        return [_settled(v) for v in x]
    if isinstance(x, dict):
        return {k: _settled(v) for k, v in x.items()}
    return x


def _vstack(ctx, parts):
    """np.vstack of 2-D pieces with the same number of columns, at least one limb-backed: ModValue, else None."""
    parts = list(parts)
    stores, rows, cols = [], 0, None
    for part in parts:
        shape = getattr(part, 'shape', None)
        if shape is None or len(shape) != 2 or (cols is not None and shape[1] != cols) or shape[0] == 0 or shape[1] == 0:
            return None
        cols = shape[1]
        if type(part) is ModValue and part.store is not None and part.ctx is ctx:
            stores.append(part._flush())
        else:
            if type(part) in (ModValue, LimbValue):
                part = part._materialise()
            if type(part) is not np.ndarray or part.dtype.kind not in 'Oiu':
                return None
            calls['packed'] += 1
            stores.append(codec.ints_to_limbs(part.astype(object).reshape(-1), ctx))
        rows += shape[0]
    if not any(type(part) is ModValue for part in parts):
        return None
    calls['limb_ops'] += 1
    return ModValue(ctx, backend.concat(ctx, stores), (rows, cols))


import operator as _operator   # noqa: E402

_NUMPY_OPS = {'+': _operator.add, '-': _operator.sub, '*': _operator.mul}
_UFUNC_OPS = {np.add: '+', np.subtract: '-', np.multiply: '*', np.left_shift: '<<'}


def _delegate_mod(name):
    def method(self, *args, **kwargs):
        return getattr(self._materialise(), name)(*args, **kwargs)
    method.__name__ = name
    return method


for _name in ('contains', 'matmul', 'rmatmul', 'imatmul', 'rmod', 'floordiv', 'rfloordiv', 'ifloordiv', 'truediv', 'rtruediv',
              'itruediv', 'rpow', 'ipow', 'abs', 'invert', 'rlshift', 'rshift', 'rrshift', 'irshift', 'iand', 'or', 'ror', 'ior',
              'xor', 'rxor', 'ixor', 'lt', 'le', 'gt', 'ge', 'bool', 'int', 'index', 'float', 'divmod', 'rdivmod', 'str',
              'format'):
    setattr(ModValue, f'__{_name}__', _delegate_mod(f'__{_name}__'))


class _ShiftedBits:
    """`value << shifts` for a value of shape (..., f) and shifts = arange(f) or arange(f-1, -1, -1): summed along the last
    axis by the k_bits_compose kernel (runtime.py:860, 3650-3651, 4415); any other use evaluates the shift on the object
    array."""

    def __init__(self, base, shifts, descending):
        self.base, self.shifts, self.descending = base, shifts, descending

    def sum(self, axis=None, out=None, **kwargs):
        b = self.base
        if b.store is not None and axis in (len(b.shape) - 1, -1) and out is None and not kwargs:
            f = b.shape[-1]                              # the bit positions are the last axis (runtime.py:860, 4415)
            n = b.size // f
            calls['limb_ops'] += 1
            if b.ctx.binary:
                calls['gf_local'] += 1
                return b._new(backend.gf_bits_compose(b.ctx, b._flush(), n, f), b.shape[:-1])
            return b._new(backend.bits_compose(b.ctx, b._flush(), n, f, self.descending), b.shape[:-1])
        return self._eval().sum(axis=axis, out=out, **kwargs)

    def _eval(self):
        return self.base._materialise() << self.shifts

    def __array__(self, dtype=None, copy=None):
        return self._eval()

    def __getattr__(self, name):
        if name.startswith('__') and name.endswith('__'):
            raise AttributeError(name)
        return getattr(self._eval(), name)


class _OuterBits:
    """`np.right_shift.outer(c, shifts)` for an opened value c and shifts = arange(l) or arange(l-1, -1, -1): `.T & 1`
    (runtime.py:3660) is the k_bits_decompose kernel; any other use evaluates the shifts on the object array."""

    def __init__(self, base, shifts, descending, transposed):
        self.base, self.shifts, self.descending, self.transposed = base, shifts, descending, transposed

    @property
    def shape(self):
        n, l = self.base.shape[0], self.shifts.shape[0]
        return (l, n) if self.transposed else (n, l)

    @property
    def T(self):
        return _OuterBits(self.base, self.shifts, self.descending, not self.transposed)

    def __and__(self, mask):
        b = self.base
        if b.store is not None and isinstance(mask, (int, np.integer)) and not isinstance(mask, (bool, np.bool_)) and mask == 1:
            n, l = b.shape[0], self.shifts.shape[0]
            calls['limb_ops'] += 1
            bits = backend.bits_decompose(b.ctx, b._flush(), l, self.descending)         # (l, n)
            if self.transposed:
                return b._new(bits, (l, n), True)
            calls['limb_ops'] += 1
            return b._new(backend.transpose(b.ctx, bits, l, n), (n, l), True)
        return self._eval() & mask

    __rand__ = __and__

    def _eval(self):
        a = np.right_shift.outer(self.base._materialise(), self.shifts)
        return a.T if self.transposed else a

    def __array__(self, dtype=None, copy=None):
        return self._eval()

    def __getattr__(self, name):
        if name.startswith('__') and name.endswith('__'):
            raise AttributeError(name)
        return getattr(self._eval(), name)


def _from_wire(modulus, binary, shape, data):
    ctx = context_for(modulus, binary=binary)
    limbs = codec.wire_to_limbs(data, ctx)
    n = 1
    for s in shape:
        n *= s
    if limbs.shape[0] != n:
        raise ValueError('LimbValue: wire data does not hold the announced number of elements')
    return LimbValue(ctx, limbs, shape)


def _from_ints(ints):
    return ints


def as_limb_value(value):
    """LimbValue for a limb-backed LimbValue / ShareRow / ModValue, else None."""
    if type(value) is LimbValue:
        return value if value.store is not None else None
    if type(value) is ModValue:
        return value.limb_value()
    if type(value) is ShareRow and value._ints is None:
        return LimbValue(value.ctx, value.limbs, (len(value),), value._poly)
    return None


# ---------------------------------------------------------------------------------------------
# FiniteFieldArray.value as a property over the original slot (installed by mpyc_b200.install)
# ---------------------------------------------------------------------------------------------

_slot = None            # the member descriptor FiniteFieldArray.__dict__['value'] of the patched finfields module
_lazy_codes = set()     # code objects that may see a LimbValue (see module docstring)
_mod_codes = set()      # code objects that get a ModValue: their arithmetic on raw values runs mod p on the device
_gf_mod_codes = set()   # those of _mod_codes that get a ModValue over GF(2^8) as well (_GF_MOD_NAMES)
_runtime_seen = [False]
local_algebra = True    # hand ModValues to the functions below (install(local_algebra=...))

# Runtime methods whose raw-value algebra is known to be ring operations ending in `Zp.array(...)` (plus `&` / `!= 0` on
# opened, canonical values): sha256 of their source in lschoe/mpyc v0.11.2.  A function whose source differs is not
# whitelisted -- its `.value` reads settle to the reference's object arrays as for every other reader.
_MOD_SOURCES = {
    'np_random_bits': '26b092e612b3091d4ac89237593b4069fa5eee590abcbe21077d13b992bf3868',     # runtime.py:4187-4273
    'np_trunc': 'e6354dbb71d6369d8bef9b065bef0cb65b1dc55631634954792f7945e087e3ad',           # runtime.py:838-872
    'np_sgn': '936eb16da844a41f636537f44306b80fff9aea3834ba205e187e6ba5a24547ad',             # runtime.py:3622-3694
    'np_to_bits': 'fb87bacf263e7c49f50422bba78d6bbf24fb200bc068983a511619da6bd16c1a',         # runtime.py:4391-4441
    'np_reciprocal': '0ebb2c0f58c50e5229f2586b7f2db9e3ca18a1bed3486c7f28aa047095af0c00',      # runtime.py:1250-1294
    'np_lsb': '4307852ce433d97be6c3bd63dbcc6a9c644b6acfd986a7fbbbac3eaa90c31bfb',             # runtime.py:1800-1822
    '_np_is_zero': 'd2beb72e8b098a8e79dbdd2438f24e0972b9a6c46073fbad7a13bec0a6c761f0',        # runtime.py:3581-3620
    'np_from_bits': '64d71aeb3dbed028a8046d6176b2fd8c8b38661bcd831ee069d3d1749338956c',       # runtime.py:4475-4484
}
# Over GF(2^8) (with K15) only these get ModValues: their raw-value algebra there is `v << np.arange(l)` summed along the last
# axis (k_gf_bits_compose), `field_array + r_modl` (XOR) and reads of the opened `c` (runtime.py:4415-4423, 4483).
_GF_MOD_NAMES = ('np_to_bits', 'np_from_bits')


def raw_value(arr):
    """The content of arr's value slot without settling it (arr: a patched FiniteFieldArray, or any stand-in)."""
    if _slot is not None and isinstance(arr, _slot.__objclass__):
        return _slot.__get__(arr)
    return arr.value


def _collect_runtime_codes(finfields_module):
    """runtime._reshare / output / _distribute of the MPyC the patched finfields belongs to, once it is imported."""
    if _runtime_seen[0]:
        return
    pkg = finfields_module.__name__.rsplit('.', 1)[0]
    rt = sys.modules.get(pkg + '.runtime')
    if rt is None or not hasattr(rt, 'Runtime'):
        return
    for name in ('_reshare', 'output', '_distribute'):
        fn = getattr(rt.Runtime, name, None)
        fn = getattr(fn, '__wrapped__', fn)
        if fn is not None and hasattr(fn, '__code__'):
            _lazy_codes.add(fn.__code__)
    st = sys.modules.get(pkg + '.sectypes')
    fn = getattr(getattr(st, 'SecureArray', None), '__init__', None)
    if fn is not None and hasattr(fn, '__code__') and fn.__code__.co_names.count('value') and 'shape' in fn.__code__.co_names:
        _lazy_codes.add(fn.__code__)          # `shape = value.value.shape` (sectypes.py:1019): asks the shape only
    if local_algebra:
        import hashlib
        import inspect
        for name, digest in _MOD_SOURCES.items():
            fn = getattr(rt.Runtime, name, None)
            fn = getattr(fn, '__wrapped__', fn)
            try:
                if hashlib.sha256(inspect.getsource(fn).encode()).hexdigest() == digest:
                    _mod_codes.add(fn.__code__)
                    if name in _GF_MOD_NAMES:
                        _gf_mod_codes.add(fn.__code__)
            except (OSError, TypeError):
                pass
    _runtime_seen[0] = True


def make_value_property(finfields_module):
    global _slot
    cls = finfields_module.FiniteFieldArray
    _slot = cls.__dict__['value']
    slot_get, slot_set = _slot.__get__, _slot.__set__
    _lazy_codes.clear()
    _mod_codes.clear()
    _gf_mod_codes.clear()
    _runtime_seen[0] = False
    for name in ('reshape', 'ravel', 'flatten', 'copy', '__len__'):
        fn = cls.__dict__.get(name)
        if fn is not None and hasattr(fn, '__code__'):
            _lazy_codes.add(fn.__code__)
    for name in ('shape', 'ndim', 'size'):
        prop = cls.__dict__.get(name)
        fn = getattr(prop, 'fget', None)
        if fn is not None and hasattr(fn, '__code__'):
            _lazy_codes.add(fn.__code__)

    def get(self):
        v = slot_get(self)
        if type(v) is not LimbValue:
            return v
        if v.store is not None:
            if not _runtime_seen[0]:
                _collect_runtime_codes(finfields_module)
            code = sys._getframe(1).f_code
            if code in _lazy_codes:
                return v
            if code in _mod_codes and (not v.ctx.binary or (code in _gf_mod_codes and _gf_backend())):
                calls['mod_values'] += 1
                return ModValue(v.ctx, v.store, v.shape, exact=True)
        a = v._materialise()
        slot_set(self, a)           # settled: from here on this array is an ordinary reference array
        return a

    return property(get, slot_set, doc='array of field element values (mpyc_b200: limb-backed until looked at)')


def restore_value_slot(finfields_module):
    global _slot
    if _slot is not None:
        finfields_module.FiniteFieldArray.value = _slot
        _slot = None


# ---------------------------------------------------------------------------------------------
# operator hooks for FiniteFieldArray (installed by mpyc_b200.install)
# ---------------------------------------------------------------------------------------------

_MISS = object()


def _ctx_of(cls):
    try:
        return context_of_field(cls.field)
    except _cabi.UnsupportedFieldError:
        return None


def _operand(ctx, cls, x, any_size=False):
    """(store, shape) of an array operand as limbs, or None when it should stay with the reference's code.  An object array
    of Python ints is packed when it has at least min_size elements, or whatever its size with any_size; over GF(2^8) (with
    K15) an object array of BinaryPolynomial or non-negative int entries, each reduced by _gf2_mod."""
    if isinstance(x, cls):
        x = raw_value(x)
    lv = as_limb_value(x)
    if lv is not None:
        return (lv.store, lv.shape) if lv.ctx is ctx else None
    if type(x) is LimbValue or type(x) is ModValue:
        x = x._ints
    if isinstance(x, np.ndarray) and x.dtype == object and (any_size or x.size >= min_size):
        if not ctx.binary:
            calls['packed'] += 1
            return codec.ints_to_limbs(x.reshape(-1), ctx), x.shape
        store = _gf_bytes(ctx, x, type(cls.field.modulus)) if _gf_backend() else None
        if store is not None:
            calls['packed'] += 1
            return store, x.shape
    return None


def _gf_backend():
    """K15's hooks run only when the backend has its three methods.  CudaBackend always does; a substituted backend without
    them (a test stand-in) leaves GF(2^8) operands to the reference's code, as before K15 existed."""
    return all(hasattr(backend, m) for m in ('gf_bits_compose', 'gf_binop_view', 'gf_matmul_batched'))


def _gf_bytes(ctx, x, poly_type):
    """uint8 store of an object array of polynomial (poly_type: the field's BinaryPolynomial class) or non-negative int
    entries reduced mod the field polynomial (the reference's field.array reduces them so, finfields.py:724); None when
    another entry occurs."""
    out = np.empty(x.size, dtype=np.uint8)
    for i, v in enumerate(x.flat):
        if not (isinstance(v, poly_type) or
                (isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_)) and v >= 0)):
            return None
        out[i] = _gf2_mod(int(v), ctx.modulus)
    return out


def _qualifies(value):
    """The operand rule of the hooks: a raw value that is limb-backed, or an ndarray of at least min_size elements."""
    return as_limb_value(value) is not None or (isinstance(value, np.ndarray) and value.size >= min_size)


def _gf2_mod(a, f):
    """a mod f in GF(2)[X] (integer encodings): an int operand of a binary-field array is the polynomial with that
    encoding (gfpx's int coercion, mpyc/gfpx.py:73-81), reduced when the result is (finfields.py:724)."""
    fb = f.bit_length()
    while a.bit_length() >= fb:
        a ^= f << (a.bit_length() - fb)
    return a


def _scalar(ctx, cls, x):
    if isinstance(x, cls.field):
        x = x.value
    if ctx.binary:
        if type(x).__name__.endswith('Polynomial') or (isinstance(x, (int, np.integer)) and not isinstance(x, bool) and x >= 0):
            return _gf2_mod(int(x), ctx.modulus)
        return None
    if isinstance(x, (int, np.integer)) and not isinstance(x, bool):
        return int(x)
    return None


def _wrap(cls, ctx, store, shape):
    calls['limb_ops'] += 1
    poly = type(cls.field.modulus) if ctx.binary else None
    return cls(LimbValue(ctx, store, shape, poly), check=False)


def binop(self, other, op, reflected=False):
    """self (op) other on limbs when self is limb-backed or large; _MISS -> caller uses the reference's method.
    op: _cabi.OP_ADD / OP_SUB / OP_MUL.  reflected: other - self."""
    cls = type(self)
    ctx = _ctx_of(cls)
    if ctx is None:
        return _MISS
    if not _qualifies(raw_value(self)) and not (isinstance(other, cls) and as_limb_value(raw_value(other)) is not None):
        return _MISS
    a = _operand(ctx, cls, self)
    if a is None:
        return _MISS
    s = _scalar(ctx, cls, other)
    if s is not None:
        if reflected:          # s - a = (-a) + s
            neg = backend.neg(ctx, a[0])
            return _wrap(cls, ctx, backend.binop_scalar(ctx, _cabi.OP_ADD, neg, s), a[1])
        return _wrap(cls, ctx, backend.binop_scalar(ctx, op, a[0], s), a[1])
    if not isinstance(other, (cls, np.ndarray, LimbValue)):
        return _MISS
    b = _gf_int_operand(ctx, self, other, op) if _int_matrix(other) else _operand(ctx, cls, other)
    if b is None:
        return _MISS
    if b[1] != a[1]:
        # NumPy's row broadcast between a matrix (R, C) and a vector (C,) runs on k_binop_rows, any other broadcast on
        # K8's k_binop_view (K15's k_gf_binop_view over GF(2^8))
        if ctx.binary:
            return _broadcast_binop(cls, ctx, op, (b, a) if reflected else (a, b))
        if len(a[1]) == 2 and len(b[1]) == 1 and a[1][1] == b[1][0] and a[1][0] and a[1][1]:
            mat, vec, vec_first = a, b, reflected
        elif len(a[1]) == 1 and len(b[1]) == 2 and b[1][1] == a[1][0] and b[1][0] and b[1][1]:
            mat, vec, vec_first = b, a, not reflected
        else:
            return _broadcast_binop(cls, ctx, op, (b, a) if reflected else (a, b))
        R, C = mat[1]
        return _wrap(cls, ctx, backend.binop_rows(ctx, op, mat[0], vec[0], R, C, vec_first), (R, C))
    x, y = (b[0], a[0]) if reflected else (a[0], b[0])
    return _wrap(cls, ctx, backend.binop(ctx, op, x, y), a[1])


def _layout_backend():
    """K8's hooks run only when the backend has copy_view and binop_view.  CudaBackend always does; a substituted backend
    without them (a test stand-in) leaves views, joins and broadcasts to the reference's code, as before K8 existed."""
    return hasattr(backend, 'copy_view') and hasattr(backend, 'binop_view')


def _broadcast_binop(cls, ctx, op, operands):
    """x (op) y under NumPy broadcasting for stores x, y of two shapes (K8's k_binop_view; the broadcast operand is read in
    place); _MISS for incompatible shapes (NumPy raises) and views beyond the kernels' rank."""
    (x, sx), (y, sy) = operands
    if not (_gf_backend() if ctx.binary else _layout_backend()):
        return _MISS
    try:
        shape, vx, vy = layout.broadcast_views(sx, sy)
    except ValueError:
        return _MISS
    c = layout.collapse(vx, vy)
    if c is None:
        return _MISS
    view_op = backend.gf_binop_view if ctx.binary else backend.binop_view
    calls['gf_local'] += ctx.binary
    return _wrap(cls, ctx, view_op(ctx, op, x, c[0], y, c[1]), shape)


def _gf_int_operand(ctx, self, other, op):
    """(store, shape) of a NumPy integer ndarray added to a limb-backed GF(2^8) array -- np_to_bits' `c_bits + r_bits`
    (runtime.py:4423): entries in [0, 256) are the field elements with those encodings, uploaded as bytes.  None for other
    entries, other operations, prime fields and backends without K15."""
    if not ctx.binary or op != _cabi.OP_ADD or not _gf_backend() or as_limb_value(raw_value(self)) is None or not other.size:
        return None
    if other.min() < 0 or other.max() > 255:
        return None
    calls['packed'] += 1
    return np.ascontiguousarray(other, dtype=np.uint8).reshape(-1), other.shape


def _element(cls, ctx, store):
    """The field element held by a one-element store (finfields.py:1006-1007 returns elements for 0-d selections)."""
    calls['limb_ops'] += 1
    return cls.field(int(codec.limbs_to_ints(backend.to_host(ctx, store), ctx)[0]))


def _gather(cls, lv, items, out_shape):
    """A new limb-backed array of out_shape filled by the K8 copies `items` ([(source, src View, dst View)], sources: stores)
    after collapsing; _MISS when a view has more axes than the kernels take."""
    n = layout._prod(out_shape)
    plan = layout.pieces([(i, s, d) for i, (_, s, d) in enumerate(items)])
    if plan is None:
        return _MISS
    store = backend.copy_view(lv.ctx, n, None, [(items[i][0], s, d) for i, s, d in plan])
    return _wrap(cls, lv.ctx, store, out_shape)


def _view_result(cls, lv, view, out_shape):
    """lv's elements seen through `view`: shares the store when the view is one contiguous run, else one K8 copy."""
    run = view.run()
    if run is not None:
        return cls(LimbValue(lv.ctx, backend.slice(lv.ctx, lv.store, *run), out_shape, lv._poly), check=False)
    return _gather(cls, lv, [(lv.store, view, layout.View.full(out_shape))], out_shape)


def _axis0_run(shape, key):
    """key is an int (ndim >= 2) or a step-1 slice on axis 0: the contiguous selections that share the store without K8
    (np_prod's halving loop, runtime.py:2198-2204)."""
    if isinstance(key, tuple):
        if len(key) != 1:
            return False
        key = key[0]
    if isinstance(key, slice):
        return bool(shape) and key.step in (None, 1)
    return _plain_int(key) and len(shape) >= 2


def getitem(self, key):
    """self[key] for a limb-backed array (FiniteFieldArray.__getitem__, finfields.py:1004-1009) and any key of ints,
    slices, Ellipsis, None and at most one 1-D integer array (mpyc_b200.layout.getitem_plan).  A selection that is one
    contiguous run of the C-ordered elements shares the limbs (the reference returns a no-copy view; limb stores are
    immutable, a later write replaces the store of the array written to); any other covered key is one K8 copy; a 0-d
    selection is a field element.  _MISS for everything else (boolean masks, several index arrays, keys NumPy rejects),
    and, on a backend without K8, for every key but an int or step-1 slice on axis 0."""
    cls = type(self)
    lv = as_limb_value(raw_value(self))
    if lv is None:
        return _MISS
    plan = layout.getitem_plan(lv.shape, key)
    if plan is None:
        return _MISS
    view, out_shape, scalar = plan
    if not _layout_backend() and not _axis0_run(lv.shape, key):
        return _MISS
    if scalar:
        return _element(cls, lv.ctx, backend.slice(lv.ctx, lv.store, view.offset, view.offset + 1))
    return _view_result(cls, lv, view, out_shape)


def setitem(self, key, value):
    """self[key] = value (FiniteFieldArray.__setitem__, finfields.py:1011-1029; Runtime.np_update, runtime.py:2657-2679)
    for a limb-backed array: value is an array of the same class (limb-backed, or of Python ints), a field element or an
    int, broadcastable to the selection.  The array gets a new store -- a device copy of the old one with the value copied
    into the selected view (stride 0 on broadcast axes) -- so arrays sharing the old store do not change.  Returns None
    when done; _MISS leaves the write to the reference (uncovered keys and values, and an index array with repeated
    entries, whose write order NumPy decides)."""
    cls = type(self)
    ctx = _ctx_of(cls)
    lv = as_limb_value(raw_value(self))
    if lv is None or ctx is None or lv.ctx is not ctx or not _layout_backend():
        return _MISS
    plan = layout.getitem_plan(lv.shape, key)
    if plan is None:
        return _MISS
    view, sel_shape, _ = plan
    if view.index_axis >= 0 and len(np.unique(view.index)) != len(view.index):
        return _MISS
    if isinstance(value, cls):
        vv = raw_value(value)
        # a settled LimbValue in the slot is left to the reference, which settles the slot itself
        op = None if type(vv) is LimbValue and vv.store is None else _operand(ctx, cls, vv, any_size=True)
        if op is None:
            return _MISS
        vstore, vshape = op
    else:
        k = _scalar(ctx, cls, value)
        if k is None:
            return _MISS
        vstore, vshape = codec.ints_to_limbs([k if ctx.binary else k % ctx.modulus], ctx), ()
    try:
        out, vview, _ = layout.broadcast_views(vshape, sel_shape)
    except ValueError:
        return _MISS
    if out != sel_shape:
        return _MISS                      # the value does not broadcast to the selection: the reference raises
    plan = layout.pieces([(0, vview, view)])
    if plan is None:
        return _MISS
    store = backend.copy_view(ctx, lv.size, lv.store, [(vstore, s, d) for _, s, d in plan])
    _slot.__set__(self, LimbValue(ctx, store, lv.shape, lv._poly))
    calls['limb_ops'] += 1
    return None


def permute(self, order):
    """self.transpose(*axes) / swapaxes / T / np.transpose / np.swapaxes / np.moveaxis for a limb-backed array: `order(ndim)`
    gives NumPy's axis order (mpyc_b200.layout); one K8 copy, or the shared store when the order moves only length-1 axes.
    _MISS for bad axes (NumPy raises) and arrays that are not limb-backed."""
    cls = type(self)
    lv = as_limb_value(raw_value(self))
    if lv is None or not _layout_backend():
        return _MISS
    try:
        perm = order(len(lv.shape))
    except (TypeError, ValueError, IndexError):
        return _MISS
    view = layout.permuted(lv.shape, perm)
    return _view_result(cls, lv, view, view.shape)


def transpose(self, *axes):
    """self.transpose(*axes) (T is self.transpose(), finfields.py:1358-1368) on K8, as permute."""
    return permute(self, lambda nd: layout.transpose_axes(nd, axes))


def swapaxes(self, axis1, axis2):
    return permute(self, lambda nd: layout.swapaxes_axes(nd, axis1, axis2))


def _join_parts(cls, arrays):
    """[(shape, LimbValue or None)] of a join's pieces -- arrays of class cls, limb-backed or plain (None: Python ints, or
    over GF(2^8) with K15 polynomials, packed by _operand), at least one limb-backed -- or None."""
    if not isinstance(arrays, (list, tuple)) or not arrays or any(type(a) is not cls for a in arrays):
        return None
    ctx = _ctx_of(cls)
    vals = [raw_value(a) for a in arrays]
    lvs = [as_limb_value(v) for v in vals]
    if ctx is None or all(v is None for v in lvs) or any(v is not None and v.ctx is not ctx for v in lvs):
        return None
    parts = []
    for v, x in zip(lvs, vals):
        if v is not None:
            parts.append((v.shape, v))
        elif isinstance(x, np.ndarray) and x.dtype == object and (not ctx.binary or _gf_backend()):
            parts.append((x.shape, None))
        else:
            return None
    return parts


def _bind(names, args, kwargs):
    """{parameter: argument} of args and kwargs bound to the parameter names `names` in order; None for more args than
    names, and for a keyword that is unknown or repeats a positional argument."""
    if len(args) > len(names) or not set(kwargs) <= set(names[len(args):]):
        return None
    return dict(zip(names, args), **kwargs)


_LAYOUT_PARAMS = {'transpose': ('a', 'axes'), 'swapaxes': ('a', 'axis1', 'axis2'), 'moveaxis': ('a', 'source', 'destination'),
                  'concatenate': ('arrays', 'axis'), 'stack': ('arrays', 'axis'), 'vstack': ('tup',), 'hstack': ('tup',),
                  'flip': ('m', 'axis'), 'roll': ('a', 'shift', 'axis'), 'expand_dims': ('a', 'axis'), 'squeeze': ('a', 'axis')}
_LAYOUT_REQUIRED = {'swapaxes': 3, 'moveaxis': 3, 'roll': 2, 'expand_dims': 2}
LAYOUT_FUNCTIONS = tuple(getattr(np, name) for name in _LAYOUT_PARAMS)


def layout_function(cls, func, args, kwargs):
    """np.transpose / swapaxes / moveaxis / concatenate / stack / vstack / hstack / flip / roll / expand_dims / squeeze of
    field arrays (FiniteFieldArray.__array_function__, finfields.py:766-819) on K8: one copy per input (two per rolled
    axis), or none for expand_dims / squeeze and permutations of length-1 axes, which share the store.  Pieces must be
    arrays of class cls; anything else (public integer arrays in particular, which the reference reduces), unknown
    arguments, 0-d results and arguments NumPy rejects give _MISS."""
    name = func.__name__
    names = _LAYOUT_PARAMS.get(name)
    bound = None if names is None else _bind(names, args, kwargs)
    if bound is None or not _layout_backend() or len(bound) < _LAYOUT_REQUIRED.get(name, 1):
        return _MISS
    first = bound[names[0]]
    try:
        if name in ('concatenate', 'stack', 'vstack', 'hstack'):
            parts = _join_parts(cls, first)
            if parts is None:
                return _MISS
            shapes = [p[0] for p in parts]
            if name == 'concatenate':
                out_shape, items = layout.concatenate_plan(shapes, bound.get('axis', 0))
            elif name == 'stack':
                out_shape, items = layout.stack_plan(shapes, bound.get('axis', 0))
            elif name == 'vstack':
                out_shape, items = layout.concatenate_plan(layout.vstack_shapes(shapes), 0)
            else:
                out_shape, items = layout.concatenate_plan(*layout.hstack_axis(shapes))
            if not out_shape:
                return _MISS
            ctx = _ctx_of(cls)
            stores = [_operand(ctx, cls, a, any_size=True)[0] for a in first]
            poly = next(v._poly for _, v in parts if v is not None)
            lv = LimbValue(ctx, stores[0], shapes[0], poly)
            return _gather(cls, lv, [(stores[i], s, d) for i, s, d in items], out_shape)
        if type(first) is not cls:
            return _MISS
        lv = as_limb_value(raw_value(first))
        if lv is None:
            return _MISS
        shape = lv.shape
        if name == 'transpose':
            return transpose(first, bound.get('axes'))
        if name == 'swapaxes':
            return swapaxes(first, bound['axis1'], bound['axis2'])
        if name == 'moveaxis':
            return permute(first, lambda nd: layout.moveaxis_axes(nd, bound['source'], bound['destination']))
        if name in ('expand_dims', 'squeeze'):
            out_shape = layout.reshaped(shape, func, bound.get('axis'))
            if not out_shape:
                return _MISS
            return cls(LimbValue(lv.ctx, lv.store, out_shape, lv._poly), check=False)
        if not shape:
            return _MISS
        if name == 'flip':
            view = layout.flip_view(shape, bound.get('axis'))
            return _view_result(cls, lv, view, shape)
        shift, axis = bound['shift'], bound.get('axis')
        if not _plain_int(shift) or not (axis is None or _plain_int(axis)):
            return _MISS
        return _gather(cls, lv, [(lv.store, s, d) for _, s, d in layout.roll_plan(shape, int(shift), axis)], shape)
    except (TypeError, ValueError, IndexError):
        return _MISS


def concatenate(cls, args, kwargs):
    """np.concatenate(arrays, axis=0) of limb-backed arrays of one field (np_prod's odd step, runtime.py:2202) on a backend
    without K8, which layout_function covers; _MISS otherwise."""
    if len(args) != 1 or not set(kwargs) <= {'axis'} or _layout_backend():
        return _MISS
    arrays = list(args[0])
    if kwargs.get('axis', 0) != 0 or not arrays:
        return _MISS
    lvs = [as_limb_value(raw_value(a)) if isinstance(a, cls) else None for a in arrays]
    if any(v is None or v.ctx is not lvs[0].ctx or v.shape[1:] != lvs[0].shape[1:] or not v.shape for v in lvs):
        return _MISS
    ctx = lvs[0].ctx
    calls['limb_ops'] += 1
    store = backend.concat(ctx, [v.store for v in lvs])
    return cls(LimbValue(ctx, store, (sum(v.shape[0] for v in lvs),) + lvs[0].shape[1:], lvs[0]._poly), check=False)


def equals(self, other, negate):
    """self == other / self != other (FiniteFieldArray.__eq__ / __ne__, finfields.py:1030-1042) for a limb-backed array and
    an integer: a bool ndarray from the k_nonzero kernel (np_is_zero_public's `a == 0`, runtime.py:966); _MISS otherwise."""
    cls = type(self)
    ctx = _ctx_of(cls)
    lv = as_limb_value(raw_value(self))
    if ctx is None or ctx.binary or lv is None or lv.ctx is not ctx or not lv.size:
        return _MISS
    if not isinstance(other, (int, np.integer)) or isinstance(other, (bool, np.bool_)):
        return _MISS
    k = int(other) % ctx.modulus
    store = lv.store if k == 0 else backend.binop_scalar(ctx, _cabi.OP_SUB, lv.store, k)
    calls['limb_ops'] += 1
    mask, _ = backend.nonzero(ctx, store)
    mask = np.asarray(mask, dtype=bool).reshape(lv.shape)
    return mask if negate else ~mask


def shift(self, other, right):
    """self << n / self >> n for a limb-backed array and an integer n >= 0; _MISS otherwise."""
    cls = type(self)
    ctx = _ctx_of(cls)
    if ctx is None or ctx.binary or as_limb_value(raw_value(self)) is None:
        return _MISS
    if not isinstance(other, (int, np.integer)) or isinstance(other, (bool, np.bool_)) or other < 0:
        return _MISS
    k = pow(2, int(other), ctx.modulus)
    if right:
        k = pow(k, -1, ctx.modulus)
    a = _operand(ctx, cls, self)
    return _wrap(cls, ctx, backend.binop_scalar(ctx, _cabi.OP_MUL, a[0], k), a[1])


def negate(self):
    cls = type(self)
    ctx = _ctx_of(cls)
    if ctx is None or as_limb_value(raw_value(self)) is None:
        return _MISS
    a = _operand(ctx, cls, self)
    return _wrap(cls, ctx, backend.neg(ctx, a[0]), a[1])


def _int_matrix(x):
    """A plain ndarray of a NumPy integer dtype: K14's public operand."""
    return type(x) is np.ndarray and x.dtype.kind in 'iu'


def matmul(self, other, reflected=False, ufunc=False):
    """self @ other (reflected: other @ self) for 1-D / 2-D operands: through K14 when the other operand is an ndarray of a
    NumPy integer dtype, public_matmul is set and the backend has matmul_int, through K1c otherwise.  ufunc: the call is
    np.matmul through __array_ufunc__, whose 1-D @ 1-D result is a 0-d array (the reference's `cls(a)`,
    finfields.py:760-764) rather than a field element."""
    cls = type(self)
    ctx = _ctx_of(cls)
    if ctx is None:
        return _MISS
    A, B = (other, self) if reflected else (self, other)

    def shape_of(x):
        v = raw_value(x) if isinstance(x, cls) else x
        return getattr(v, 'shape', None)
    sa, sb = shape_of(A), shape_of(B)
    if sa is None or sb is None or not sa or not sb:
        return _MISS
    if len(sa) > 2 or len(sb) > 2:
        return _gf_matmul_stacked(cls, ctx, A, B, sa, sb) if ctx.binary and not _int_matrix(other) else _MISS
    r, k = (1, sa[0]) if len(sa) == 1 else sa
    k2, c = (sb[0], 1) if len(sb) == 1 else sb
    if k != k2:
        return _MISS                      # let NumPy raise its own error
    limbish = any(isinstance(x, cls) and as_limb_value(raw_value(x)) is not None for x in (A, B))
    if not limbish and r * k * c < min_size * 8:
        return _MISS
    public = _int_matrix(other)
    if public and (not public_matmul or ctx.binary or not hasattr(backend, 'matmul_int')):
        return _MISS
    if public:
        x = _operand(ctx, cls, self, any_size=True)
        if x is None:
            return _MISS
        calls['matmul_int'] += 1
        out = backend.matmul_int(ctx, x[0], other, r, k, c, reflected)
    else:
        a, b = _operand(ctx, cls, A, any_size=True), _operand(ctx, cls, B, any_size=True)
        if a is None or b is None:
            return _MISS
        out = backend.matmul(ctx, a[0], b[0], r, k, c)
    if len(sa) == 1 and len(sb) == 1:     # inner product: a field element (finfields.py:1134)
        calls['limb_ops'] += 1
        poly = type(cls.field.modulus) if ctx.binary else None
        v = LimbValue(ctx, out, (1,), poly)._materialise()[0]
        return cls(np.array(v, dtype=object), check=False) if ufunc else cls.field(v)
    shape = (c,) if len(sa) == 1 else ((r,) if len(sb) == 1 else (r, c))
    return _wrap(cls, ctx, out, shape)


def _gf_matmul_stacked(cls, ctx, A, B, sa, sb):
    """A @ B over GF(2^8) with an operand of more than two axes (NumPy's matmul of stacks, the S-box's `A @ x[..., None]`) on
    K15's k_gf_matmul_batched: each side's stack axes either match the broadcast stack shape or hold one matrix (stride 0).
    _MISS for partial broadcasts of the stack axes, empty results, mismatched shapes (NumPy raises), backends without K15 and
    plain operands below the size rule."""
    if not _gf_backend():
        return _MISS
    a2 = sa if len(sa) >= 2 else (1,) + sa
    b2 = sb if len(sb) >= 2 else sb + (1,)
    (r, k), (k2, c) = a2[-2:], b2[-2:]
    try:
        stack = np.broadcast_shapes(a2[:-2], b2[:-2])
    except ValueError:
        return _MISS
    batch = layout._prod(stack)
    if k != k2 or not batch * r * c:
        return _MISS
    stacked = []
    for s in (a2[:-2], b2[:-2]):
        full = (1,) * (len(stack) - len(s)) + tuple(s) == tuple(stack)
        if not full and layout._prod(s) != 1:
            return _MISS
        stacked.append(full and batch > 1)
    limbish = any(isinstance(x, cls) and as_limb_value(raw_value(x)) is not None for x in (A, B))
    if not limbish and batch * r * k * c < min_size * 8:
        return _MISS
    a, b = _operand(ctx, cls, A, any_size=True), _operand(ctx, cls, B, any_size=True)
    if a is None or b is None:
        return _MISS
    calls['gf_local'] += 1
    out = backend.gf_matmul_batched(ctx, a[0], stacked[0], b[0], stacked[1], batch, r, k, c)
    shape = tuple(stack) + ((r,) if len(sa) >= 2 else ()) + ((c,) if len(sb) >= 2 else ())
    return _wrap(cls, ctx, out, shape)


def _array_operand(a, ready, nonempty=False):
    """(cls, ctx, store, shape) of a prime-field array that meets the operand rule (_qualifies); None otherwise, when the
    backend lacks the hook's kernels (ready: the hook's capability gate) and, with nonempty, for an empty array."""
    cls = type(a)
    ctx = _ctx_of(cls)
    if ctx is None or ctx.binary or not ready or not _qualifies(raw_value(a)):
        return None
    op = _operand(ctx, cls, a)
    if op is None or (nonempty and not layout._prod(op[1])):
        return None
    return (cls, ctx) + op


def _sum_backend():
    """K7's hooks run only when the backend has sum_axis and cumsum_axis.  CudaBackend always does; a substituted backend
    without them (a test stand-in) leaves the call to the reference's code, as before K7 existed."""
    return hasattr(backend, 'cumsum_axis') and hasattr(backend, 'sum_axis')


def _plain_int(x):
    return isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))


def sum_(a, axis=None, keepdims=False, initial=0):
    """np.sum(a, axis, keepdims=keepdims, initial=initial) / a.sum(...) (finfields.py:766-819,1332-1337; Runtime.np_sum,
    runtime.py:3476-3506) on the K7 kernels: a field element for a 0-d result (finfields.py:818), else a limb-backed
    array.  _MISS for a non-int initial or keepdims, bad axes (NumPy raises its own error), binary fields and arrays that
    are neither limb-backed nor large."""
    if not _plain_int(initial) or not isinstance(keepdims, (bool, np.bool_)):
        return _MISS
    try:
        _, out_shape = axes.sum_plan(np.shape(raw_value(a)), axis, keepdims)
    except (TypeError, ValueError):
        return _MISS
    op = _array_operand(a, _sum_backend())
    if op is None:
        return _MISS
    cls, ctx, store, shape = op
    out = backend.sum_axis(ctx, store, shape, axis, bool(keepdims), int(initial) % ctx.modulus)
    return _element(cls, ctx, out) if out_shape == () else _wrap(cls, ctx, out, out_shape)


def cumsum(a, axis=None, include_initial=False):
    """np.cumsum(a, axis) (axis=None: flattened) and np.cumulative_sum(a, axis=axis, include_initial=...) on the K7 scan; a
    limb-backed array, or _MISS as for sum_."""
    try:
        _, out_shape = axes.scan_plan(np.shape(raw_value(a)), axis, include_initial)
    except (TypeError, ValueError):
        return _MISS
    op = _array_operand(a, _sum_backend())
    if op is None:
        return _MISS
    cls, ctx, store, shape = op
    return _wrap(cls, ctx, backend.cumsum_axis(ctx, store, shape, axis, bool(include_initial)), out_shape)


_PROD_METHODS = ('prod_axis', 'cumprod_axis', 'all_any_axis')


def _prod_backend():
    """K13's hooks run only when the backend has prod_axis, cumprod_axis and all_any_axis.  CudaBackend always does; a
    substituted backend without them (a test stand-in) leaves np.prod / np.cumprod / np.all / np.any to the reference's
    code, as before K13 existed."""
    return all(hasattr(backend, m) for m in _PROD_METHODS)


def prod_(a, axis=None, keepdims=False, initial=1):
    """np.prod(a, axis, keepdims=keepdims, initial=initial) / a.prod(...) (finfields.py:766-819,1339-1349) on the K13
    kernels: a field element for a 0-d result, else a limb-backed array.  initial: a Python int (the caller turns a field
    element into its value).  _MISS for bad axes (NumPy raises its own error), binary fields and arrays that are neither
    limb-backed nor large."""
    if type(initial) is not int or not isinstance(keepdims, (bool, np.bool_)):
        return _MISS
    try:
        _, out_shape = axes.sum_plan(np.shape(raw_value(a)), axis, keepdims)
    except (TypeError, ValueError):
        return _MISS
    op = _array_operand(a, _prod_backend())
    if op is None:
        return _MISS
    cls, ctx, store, shape = op
    calls['prod'] += 1
    out = backend.prod_axis(ctx, store, shape, axis, bool(keepdims), initial % ctx.modulus)
    return _element(cls, ctx, out) if out_shape == () else _wrap(cls, ctx, out, out_shape)


def cumprod(a, axis=None, include_initial=False):
    """np.cumprod(a, axis) (axis=None: flattened) and np.cumulative_prod(a, axis=axis, include_initial=...) on the K13
    running product; a limb-backed array, or _MISS as for prod_."""
    try:
        _, out_shape = axes.scan_plan(np.shape(raw_value(a)), axis, include_initial)
    except (TypeError, ValueError):
        return _MISS
    op = _array_operand(a, _prod_backend())
    if op is None:
        return _MISS
    cls, ctx, store, shape = op
    calls['prod'] += 1
    return _wrap(cls, ctx, backend.cumprod_axis(ctx, store, shape, axis, bool(include_initial)), out_shape)


def all_any(a, axis=None, keepdims=False, any=False):
    """np.all(a, axis, keepdims=keepdims) / np.any(...) (any) as the reference answers them (finfields.py:766-819): np.True_
    or np.False_ for a 0-d result -- from the device's count of nonzero elements, nothing else crosses to the host -- else
    a limb-backed array of 0 / 1 (the reference's `cls(bool_array)`) from the K13 kernels.  _MISS as for prod_."""
    if not isinstance(keepdims, (bool, np.bool_)):
        return _MISS
    try:
        _, out_shape = axes.sum_plan(np.shape(raw_value(a)), axis, keepdims)
    except (TypeError, ValueError):
        return _MISS
    op = _array_operand(a, _prod_backend())
    if op is None:
        return _MISS
    cls, ctx, store, shape = op
    calls['prod'] += 1
    if out_shape == ():
        _, count = backend.nonzero(ctx, store, want_mask=False)
        n = layout._prod(shape)
        return np.True_ if (count > 0 if any else count == n) else np.False_
    return _wrap(cls, ctx, backend.all_any_axis(ctx, store, shape, axis, bool(keepdims), bool(any)), out_shape)


def prod_method(self, *args, **kwargs):
    """FiniteFieldArray.prod(*args, **kwargs) (finfields.py:1339-1349), which turns initial into a field element first:
    an int or an element of the array's field is taken here, anything else (and initial or where given by position) stays
    with the reference."""
    bound = _bind(('axis', 'dtype', 'out', 'keepdims', 'initial', 'where'), args, kwargs) if len(args) <= 4 else None
    if bound is None or any(bound.get(k, None) is not None for k in ('dtype', 'out')) or 'where' in bound:
        return _MISS
    initial = bound.get('initial', 1)
    if isinstance(initial, type(self).field):
        initial = int(initial.value)
    elif type(initial) is not int:
        return _MISS
    return prod_(self, bound.get('axis', None), bound.get('keepdims', False), initial)


def outer(a, b):
    """np.outer(a, b) of two arrays of one prime field (Runtime.np_outer, runtime.py:2544-2578): c[i, j] = a_i b_j on the
    flattened operands, through K1c with k = 1.  _MISS for anything else -- a public integer operand in particular, whose
    values _operand would pack without reducing them."""
    cls = type(a)
    ctx = _ctx_of(cls)
    if ctx is None or ctx.binary or type(b) is not cls:
        return _MISS
    va, vb = raw_value(a), raw_value(b)
    limbish = as_limb_value(va) is not None or as_limb_value(vb) is not None
    na, nb = int(np.size(va)), int(np.size(vb))
    if not limbish and na * nb < min_size:
        return _MISS
    x, y = _operand(ctx, cls, a, any_size=True), _operand(ctx, cls, b, any_size=True)
    if x is None or y is None:
        return _MISS
    return _wrap(cls, ctx, backend.matmul(ctx, x[0], y[0], na, 1, nb), (na, nb))


_REDUCTION_PARAMS = {'sum': ('a', 'axis', 'dtype', 'out', 'keepdims', 'initial', 'where'), 'cumsum': ('a', 'axis', 'dtype', 'out'),
                     'outer': ('a', 'b', 'out'), 'prod': ('a', 'axis', 'dtype', 'out', 'keepdims', 'initial', 'where'),
                     'cumprod': ('a', 'axis', 'dtype', 'out'), 'all': ('a', 'axis', 'out', 'keepdims', 'where'),
                     'any': ('a', 'axis', 'out', 'keepdims', 'where'),
                     'cumulative_sum': ('x', 'axis', 'include_initial', 'dtype', 'out'),
                     'cumulative_prod': ('x', 'axis', 'include_initial', 'dtype', 'out')}
REDUCTION_FUNCTIONS = tuple(getattr(np, name) for name in _REDUCTION_PARAMS if hasattr(np, name))


def reduction_function(self, func, args, kwargs):
    """The NumPy functions routed to K7 / K1c by array_function and FiniteFieldArray.sum: np.sum, np.cumsum,
    np.cumulative_sum, np.outer, and to K13: np.prod, np.cumprod, np.cumulative_prod, np.all, np.any.  Arguments are bound
    as NumPy's signatures do (the cumulative ones take x by position only, the rest by keyword); dtype / out / where and
    unknown arguments leave the call to the reference (_MISS)."""
    name = func.__name__
    names = _REDUCTION_PARAMS[name]
    bound = None if name.startswith('cumulative_') and len(args) != 1 else _bind(names, args, kwargs)
    if bound is None or any(bound.get(k, None) is not None for k in ('dtype', 'out')) or \
            bound.get('where', np._NoValue) is not np._NoValue:
        return _MISS
    first = bound.get(names[0])
    if type(first) is not type(self):
        return _MISS
    opt = lambda k, default: default if bound.get(k, np._NoValue) is np._NoValue else bound[k]   # noqa: E731
    if name == 'sum':
        return sum_(first, opt('axis', None), opt('keepdims', False), opt('initial', 0))
    if name == 'cumsum':
        return cumsum(first, opt('axis', None))
    if name == 'outer':
        return outer(first, bound.get('b'))
    if name == 'prod':
        return prod_(first, opt('axis', None), opt('keepdims', False), opt('initial', 1))
    if name == 'cumprod':
        return cumprod(first, opt('axis', None))
    if name in ('all', 'any'):
        return all_any(first, opt('axis', None), opt('keepdims', False), name == 'any')
    axis = opt('axis', None)
    if axis is None and np.ndim(raw_value(first)) > 1:
        return _MISS                      # NumPy requires the axis of a multi-dimensional array
    scan = cumsum if name == 'cumulative_sum' else cumprod
    return scan(first, axis, bool(opt('include_initial', False)))


def array_function(self, func, args, kwargs):
    """FiniteFieldArray.__array_function__ (finfields.py:766-819) on the kernels, or _MISS for the reference's method.  The
    hooks are looked up when called and tried in this order: layout functions (K8), np.concatenate without K8, sums and
    products (K7, K1c, K13), linear algebra (K9), np.convolve (K10) and np.where (K11).  self is an array of the patched
    class or, for np.where only, a field element whose `array` is such a class: FiniteFieldElement.__array_function__
    hands the call over with self the element (finfields.py:83-85)."""
    cls = _array_class(self)
    if cls is None:
        klass = getattr(type(self), 'array', None)
        if func is np.where and isinstance(klass, type) and issubclass(klass, _slot.__objclass__):
            return where(klass, args, kwargs)
        return _MISS
    if func in LAYOUT_FUNCTIONS:
        r = layout_function(cls, func, args, kwargs)
        return concatenate(cls, args, kwargs) if r is _MISS and func is np.concatenate else r
    if func in REDUCTION_FUNCTIONS:
        return reduction_function(self, func, args, kwargs)
    if func in LINALG_FUNCTIONS:
        return linalg_function(cls, func, args, kwargs)
    if func is np.convolve:
        return convolve(cls, args, kwargs)
    if func is np.where:
        return where(cls, args, kwargs)
    return _MISS


# the parameter names of the reference's implementations, so that keywords it rejects stay with it
_LINALG_PARAMS = {'det': ('a',), 'solve': ('A', 'B'), 'inv': ('A',), 'matrix_power': ('A', 'n')}
LINALG_FUNCTIONS = tuple(getattr(np.linalg, name) for name in _LINALG_PARAMS)


def _linalg_backend():
    """K9's hooks run only when the backend has det and solve (and matrix_power for np.linalg.matrix_power).  CudaBackend
    always does; a substituted backend without them (a test stand-in) leaves linear algebra to the reference's code."""
    return hasattr(backend, 'det') and hasattr(backend, 'solve')


def linalg_function(cls, func, args, kwargs):
    """np.linalg.det / solve / inv / matrix_power of prime-field arrays (FiniteFieldArray.gauss_det / gauss_solve /
    gauss_inv / matrix_pow, finfields.py:872-976) on K9 and K1c.  det: a field element for one matrix, a limb-backed array
    of shape a.shape[:-2] for a stack; solve / inv / matrix_power: a limb-backed (n, m) array.  Operands must be arrays of
    class cls, limb-backed or of at least min_size elements (both are packed once one qualifies, as for @).  _MISS, so that
    the reference raises its own errors, for: non-square or ndim < 2 operands, n == 0 or empty stacks, stacked solve / inv /
    matrix_power, a b that is not a 2-D array of cls with n rows, an exponent that is not a Python int, binary fields and
    unknown arguments."""
    name = func.__name__
    names = _LINALG_PARAMS[name]
    bound = _bind(names, args, kwargs)
    if bound is None or not _linalg_backend() or len(bound) != len(names):
        return _MISS
    ctx = _ctx_of(cls)
    A, B = bound[names[0]], bound.get('B')
    if ctx is None or ctx.binary or type(A) is not cls:
        return _MISS
    shape = getattr(raw_value(A), 'shape', None)
    if shape is None or len(shape) < 2 or shape[-1] != shape[-2] or shape[-1] == 0 or (name != 'det' and len(shape) != 2):
        return _MISS
    n = shape[-1]
    batch = layout._prod(shape[:-2])
    if batch == 0:
        return _MISS
    operands = [A]
    if name == 'solve':
        sb = getattr(raw_value(B), 'shape', None) if type(B) is cls else None
        if sb is None or len(sb) != 2 or sb[0] != n or sb[1] == 0:
            return _MISS
        operands.append(B)
    elif name == 'matrix_power' and (type(bound['n']) is not int or not hasattr(backend, 'matrix_power')):
        return _MISS
    limbish = any(as_limb_value(raw_value(x)) is not None for x in operands)
    if not limbish and np.size(raw_value(A)) < min_size:
        return _MISS
    ops = [_operand(ctx, cls, x, any_size=True) for x in operands]
    if any(o is None for o in ops):
        return _MISS
    a = ops[0][0]
    if name == 'det':
        out = backend.det(ctx, a, batch, n)
        return _element(cls, ctx, out) if len(shape) == 2 else _wrap(cls, ctx, out, shape[:-2])
    if name == 'solve':
        nrhs = ops[1][1][1]
        return _wrap(cls, ctx, backend.solve(ctx, a, n, ops[1][0], nrhs), (n, nrhs))
    if name == 'inv':
        return _wrap(cls, ctx, backend.solve(ctx, a, n, None, n), (n, n))
    return _wrap(cls, ctx, backend.matrix_power(ctx, a, n, bound['n']), (n, n))


def _public_ints(x):
    """The entries of a public 1-D integer operand of np.convolve as a list of Python ints: a list, tuple or range of
    ints, an integer-dtype ndarray or an object ndarray of Python ints.  None for anything else (floats, bools, field
    elements, other dimensions)."""
    if isinstance(x, range):
        return list(x)
    if isinstance(x, (list, tuple)):
        return list(x) if all(type(e) is int for e in x) else None
    if isinstance(x, np.ndarray) and x.ndim == 1:
        if x.dtype.kind in 'iu':
            return [int(e) for e in x.tolist()]
        if x.dtype == object and all(type(e) is int for e in x):
            return x.tolist()
    return None


_CONVOLVE_MODES = ('full', 'same', 'valid')


def convolve(cls, args, kwargs):
    """np.convolve(a, v, mode) of prime-field vectors (FiniteFieldArray.__array_function__, finfields.py:766-819; the local
    step of Runtime.np_convolve and of np_roll's secret shift) on K10: a limb-backed array of cls holding the window of
    the full result that mode selects.  One operand is a 1-D array of cls; the other is one too, or a public integer
    sequence (_public_ints), whose entries are reduced mod p and packed -- exact, as convolution is bilinear and the
    reference's cls(result) reduces.  Both are packed once one operand is limb-backed or m * n >= min_size, as for
    np.outer.  _MISS, so that the reference keeps its own results and errors, for: binary or uncovered fields, operands
    that are 0-d, field elements, empty or not 1-D, other dtypes, arrays of another field, modes other than the three
    strings, operands passed by keyword, unknown arguments and a backend without convolve."""
    if not 2 <= len(args) <= 3 or not set(kwargs) <= ({'mode'} if len(args) == 2 else set()) or not hasattr(backend, 'convolve'):
        return _MISS                      # operands by keyword: the reference recurses (it unpacks positional ones only)
    mode = args[2] if len(args) == 3 else kwargs.get('mode', 'full')
    if type(mode) is not str or mode not in _CONVOLVE_MODES:
        return _MISS
    ctx = _ctx_of(cls)
    if ctx is None or ctx.binary:
        return _MISS
    operands = list(args[:2])
    if not any(type(x) is cls for x in operands):
        return _MISS
    sizes, public, limbish = [], [None, None], False
    for k, x in enumerate(operands):
        if type(x) is cls:
            shape = getattr(raw_value(x), 'shape', None)
            limbish = limbish or as_limb_value(raw_value(x)) is not None
        else:
            public[k] = _public_ints(x)
            shape = None if public[k] is None else (len(public[k]),)
        if shape is None or len(shape) != 1 or shape[0] == 0:
            return _MISS
        sizes.append(shape[0])
    m, n = sizes
    if not limbish and m * n < min_size:
        return _MISS
    stores = [None, None]
    for k, x in enumerate(operands):
        if public[k] is None:
            op = _operand(ctx, cls, x, any_size=True)
            if op is None:
                return _MISS
            stores[k] = op[0]
    for k, ints in enumerate(public):
        if ints is not None:
            calls['packed'] += 1
            stores[k] = codec.ints_to_limbs([e % ctx.modulus for e in ints], ctx)
    s, g = min(m, n), max(m, n)
    lo, count = {'full': (0, m + n - 1), 'same': ((s - 1) // 2, g), 'valid': (s - 1, g - s + 1)}[mode]
    return _wrap(cls, ctx, backend.convolve(ctx, stores[0], m, stores[1], n, lo, count), (count,))


# ---- K11: division, powers, square roots and np.where of field arrays ------------------------------------------------

def _divsel_backend():
    """K11's hooks run only when the backend has divide and select.  CudaBackend always does; a substituted backend without
    them (a test stand-in) leaves division and selection to the reference's code, as before K11 existed."""
    return hasattr(backend, 'divide') and hasattr(backend, 'select')


def _public_scalar(cls, x):
    """x as a Python int when it is an int (not a bool) or an element of cls.field -- what the reference's _coerce passes
    on for a scalar; None otherwise."""
    if isinstance(x, cls.field):
        x = x.value
    return x if isinstance(x, int) and not isinstance(x, bool) else None


def _zero(cls):
    z = np.empty(1, dtype=object)
    z[0] = 0
    return z


def _reference_error(fn):
    """Raise what the reference raises for a zero where an inverse is needed: fn runs the reference's own code on a single
    zero (its message depends on whether gmpy2 is installed).  Falls back to ZeroDivisionError if it does not raise."""
    fn()
    raise ZeroDivisionError('invert() no inverse exists')


def divide(self, other, reflected=False):
    """self / other (reflected: other / self) for a limb-backed or large prime-field array (FiniteFieldArray.__truediv__ /
    __rtruediv__, finfields.py:1199-1215): by a same-shape array of the class in one ff_div pass; by an int or field element
    as a product with its inverse, computed on the host; an int or field element divided by the array as ff_inv and a
    scalar product.  A zero divisor raises the reference's exception.  Returns a limb-backed array, or _MISS (broadcasting,
    other operand types, binary fields, backends without K11)."""
    cls = type(self)
    ctx = _ctx_of(cls)
    if ctx is None or ctx.binary or not _divsel_backend():
        return _MISS
    k = _public_scalar(cls, other)
    if k is None and not reflected and type(other) is cls:
        mine, theirs = raw_value(self), raw_value(other)
        if not _qualifies(mine) and as_limb_value(theirs) is None:
            return _MISS
        if np.shape(mine) != np.shape(theirs) or not layout._prod(np.shape(mine)):
            return _MISS
        a, b = _operand(ctx, cls, self), _operand(ctx, cls, other)
        if a is None or b is None:
            return _MISS
        try:
            out = backend.divide(ctx, a[0], b[0])
        except ZeroDivisionError:
            _reference_error(lambda: cls._reciprocal(_zero(cls)))
        return _wrap(cls, ctx, out, a[1])
    if k is None:
        return _MISS
    op = _array_operand(self, _divsel_backend(), nonempty=True)
    if op is None:
        return _MISS
    _, _, store, shape = op
    p = ctx.modulus
    if not reflected:
        if k % p == 0:
            _reference_error(lambda: cls._reciprocal(0))
        return _wrap(cls, ctx, backend.binop_scalar(ctx, _cabi.OP_MUL, store, pow(k, -1, p)), shape)
    try:
        inv = backend.inverse(ctx, store)
    except ZeroDivisionError:
        _reference_error(lambda: cls._reciprocal(_zero(cls)))
    calls['limb_ops'] += 1
    return _wrap(cls, ctx, backend.binop_scalar(ctx, _cabi.OP_MUL, inv, k % p), shape)


def reciprocal(self):
    """self.reciprocal() (finfields.py:1278-1281) on ff_inv: a limb-backed array, or _MISS as for divide."""
    op = _array_operand(self, _divsel_backend(), nonempty=True)
    if op is None:
        return _MISS
    cls, ctx, store, shape = op
    try:
        out = backend.inverse(ctx, store)
    except ZeroDivisionError:
        _reference_error(lambda: cls._reciprocal(_zero(cls)))
    return _wrap(cls, ctx, out, shape)


def power(self, e):
    """self ** e for a Python int e (finfields.py:1159-1167,1408-1414; powmod semantics: a negative e inverts first, e == 0
    gives ones, 0 ** 0 included).  A zero with e < 0 raises the reference's exception.  An integer ndarray e of the array's
    shape runs on K12 (`power_exp`).  _MISS for other exponents (NumPy or bool ones) and as for divide."""
    if isinstance(e, np.ndarray):
        return power_exp(self, e)
    if type(e) is not int:
        return _MISS
    op = _array_operand(self, _divsel_backend(), nonempty=True)
    if op is None:
        return _MISS
    cls, ctx, store, shape = op
    if e == 0:
        return _wrap(cls, ctx, backend.axpb(ctx, store, 0, 1), shape)
    try:
        out = backend.power(ctx, store, e)
    except ZeroDivisionError:
        _reference_error(lambda: cls._pow(_zero(cls), e))
    return _wrap(cls, ctx, out, shape)


# ---- K12: per-element exponents ---------------------------------------------------------------------------------------

def _powexp_backend():
    """K12's hooks run only when the backend has pow_exp (CudaBackend does; a stand-in without it leaves these calls to the
    reference's code)."""
    return hasattr(backend, 'pow_exp')


def _exponents(e, n):
    """codec.exponents_to_limbs(e) for n exponents, or None (not covered, or another count)."""
    r = codec.exponents_to_limbs(e)
    return r if r is not None and r[0].shape[0] == n else None


def power_exp(self, e):
    """self ** e for an int64 / uint64 / object ndarray e of Python ints of exactly self's shape (finfields.py:1159-1167 with
    PrimeFieldArray._pow, finfields.py:1409-1414), on k_powexp_elem.  _MISS -- the reference computes -- for broadcasting,
    other dtypes, exponents wider than 256 bits, negative exponents, binary fields and backends without K12."""
    if not _powexp_backend():
        return _MISS
    op = _array_operand(self, _divsel_backend(), nonempty=True)
    if op is None or e.shape != op[3]:
        return _MISS
    cls, ctx, store, shape = op
    ex = _exponents(e, layout._prod(shape))
    if ex is None or ex[1] is not None:
        return _MISS
    calls['pow_exp'] += 1
    return _wrap(cls, ctx, backend.pow_exp(ctx, store, ex[0], None, ex[2]), shape)


def powmod_exp_list(base, exp_lst, mod):
    """gmpy.powmod_exp_list(base, exp_lst, mod) (mpyc/gmpy.py:288-290) on k_powexp_fixed: a list of Python ints base^y mod
    mod for y in exp_lst.  Covered: mod the modulus of a prime field the engine already holds a context for, an int base,
    and at least min_size exponents given as Python ints in a list / tuple or a 1-D object ndarray.  _MISS for everything
    else -- NumPy integer exponents included: the reference's three-argument pow rejects them with a TypeError, which stays
    its own -- and for a base = 0 (mod mod) with a negative exponent, so that the error is the reference's."""
    if not _powexp_backend() or type(base) is not int or type(mod) is not int:
        return _MISS
    from mpyc_b200 import field
    ctx = field._contexts.get((mod, False))
    listed = isinstance(exp_lst, (list, tuple)) or (isinstance(exp_lst, np.ndarray) and exp_lst.dtype == object
                                                     and exp_lst.ndim == 1)
    if ctx is None or not listed or len(exp_lst) < max(min_size, 1):
        return _MISS
    ex = codec.exponents_to_limbs(exp_lst)
    if ex is None:
        return _MISS
    limbs, signs, bits = ex
    b = base % mod
    if b == 0 and signs is not None:
        return _MISS
    calls['pow_exp'] += 1
    out = backend.pow_exp(ctx, b, limbs, signs, bits)
    return codec.limbs_to_ints(backend.to_host(ctx, out), ctx).tolist()


def sqrt(self, INV=False):
    """self.sqrt(INV) for Blum primes (PrimeFieldArray._sqrt, finfields.py:1424-1438) on K1b; INV with a zero raises the
    reference's ZeroDivisionError('no inverse sqrt of 0').  _MISS for other primes and as for divide."""
    op = _array_operand(self, _divsel_backend(), nonempty=True)
    if op is None or not isinstance(INV, bool):
        return _MISS
    cls, ctx, store, shape = op
    if ctx.modulus & 3 != 3:
        return _MISS
    try:
        out = backend.sqrt(ctx, store, INV)
    except ZeroDivisionError:
        _reference_error(lambda: cls._sqrt(_zero(cls), INV=True))
    return _wrap(cls, ctx, out, shape)


def is_sqr(self):
    """self.is_sqr() (finfields.py:1298-1300, 1463-1470) on K1b: a host bool ndarray of the array's shape (0 counts as a
    square).  _MISS for 0-d arrays and as for divide."""
    op = _array_operand(self, _divsel_backend(), nonempty=True)
    if op is None or not op[3]:
        return _MISS
    cls, ctx, store, shape = op
    calls['limb_ops'] += 1
    return np.asarray(backend.is_sqr(ctx, store), dtype=bool).reshape(shape)


def where(cls, args, kwargs):
    """np.where(cond, x, y) with field arrays (FiniteFieldArray.__array_function__, finfields.py:766-819) on k_select: cond a
    bool or integer ndarray of the result's shape, x and y arrays of cls of that shape, ints or field elements of cls, at
    least one an array.  A limb-backed array of cls, or _MISS -- so that the reference keeps its own results and errors --
    for binary fields, broadcasting, the one-argument form, keywords, other operand types and backends without K11."""
    ctx = _ctx_of(cls)
    if len(args) != 3 or kwargs or ctx is None or ctx.binary:
        return _MISS
    cond, x, y = args
    if type(cond) is not np.ndarray:
        return _MISS
    if not any(type(v) is cls and _qualifies(raw_value(v)) for v in (x, y)):
        return _MISS
    r = _where(ctx, cls, cond, x, y)
    return _MISS if r is None else r


def conv2d(x, W, b):
    """The local step of np_cnnmnist's convolvetensor (demos/np_cnnmnist.py:69-82) as one kernel call: x (k, r, m, n),
    W (v, r, s, s), b (v) -- field arrays of one covered prime field, as `mpc.gather` returns them -- to the field array
    Y (k, v, m, n) with Y[i, j] = b[j] + sum_l correlate2d(x[i, l], W[j, l], 'same'), limb-backed, ready for
    `mpc._reshare(Y)`.  The demo is caller code that install() cannot reach; INTEGRATION.md section 5 shows the edit."""
    cls = type(x)
    ctx = _ctx_of(cls)
    if ctx is None or ctx.binary or type(W) is not cls or type(b) is not cls:
        raise _cabi.UnsupportedFieldError('conv2d: operands must be arrays of one covered prime field')
    sx, sw, sb = (getattr(raw_value(a), 'shape', None) for a in (x, W, b))
    if len(sx) != 4 or len(sw) != 4 or len(sb) != 1 or sx[1] != sw[1] or sw[2] != sw[3] or sb[0] != sw[0]:
        raise ValueError(f'conv2d: shapes {sx}, {sw}, {sb} do not fit (k,r,m,n), (v,r,s,s), (v,)')
    ops = [_operand(ctx, cls, a, any_size=True) for a in (x, W, b)]
    if any(o is None for o in ops):
        raise _cabi.UnsupportedFieldError('conv2d: operands must be limb-backed or object arrays of the field')
    k, r, m, n = sx
    v, s = sw[0], sw[2]
    out = backend.conv2d(ctx, ops[0][0], ops[1][0], ops[2][0], k, r, m, n, v, s)
    return _wrap(cls, ctx, out, (k, v, m, n))
