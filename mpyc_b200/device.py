"""Device-resident field arrays: limb tensors that stay in HBM between operations.

torch is used for what it is good at here -- device memory, streams, (later) torch.distributed --
while every computation goes through the C ABI (mpyc_b200._cabi) on the tensor's data pointer and
torch's current CUDA stream.  A DeviceArray mirrors the operator surface of the reference's
PrimeFieldArray / BinaryFieldArray (mpyc/finfields.py:1056-1281,1371-1470) for 1-D arrays.
"""
import ctypes

import numpy as np
import torch

from mpyc_b200 import _cabi, codec
from mpyc_b200._cabi import lib, check
from mpyc_b200.field import FieldContext


def _stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError('mpyc_b200: no CUDA device available (there is no CPU fallback)')


def _alloc(ctx, rows, n, device):
    """Uninitialised limb storage: int64 (rows, n, L) or uint8 (rows, n); row stride padded to 32 bytes
    so that every row start allows the 32-byte vector path."""
    _require_cuda()
    if ctx.binary:
        stride = (n + 31) // 32 * 32
        return torch.empty((rows, stride), dtype=torch.uint8, device=device)[:, :n]
    L = ctx.nlimbs
    q = {1: 4, 2: 2, 3: 4, 4: 1}[L]
    stride = (n + q - 1) // q * q
    return torch.empty((rows, stride, L), dtype=torch.int64, device=device)[:, :n]


class DeviceArray:
    """n elements of one field in device memory (1-D)."""

    __slots__ = ('ctx', 't')

    def __init__(self, ctx: FieldContext, tensor):
        self.ctx = ctx
        self.t = tensor   # int64 (n, L) contiguous, or uint8 (n,)

    # ---- construction / extraction ---------------------------------------------------------------
    @classmethod
    def empty(cls, ctx, n, device='cuda'):
        return cls(ctx, _alloc(ctx, 1, n, device)[0])

    @classmethod
    def from_limbs(cls, ctx, limbs, device='cuda'):
        _require_cuda()
        a = np.ascontiguousarray(limbs)
        src = torch.from_numpy(a if ctx.binary else a.view(np.int64))
        out = cls.empty(ctx, a.shape[0], device)
        out.t.copy_(src)
        return out

    @classmethod
    def from_ints(cls, ctx, values, device='cuda', reduce=True):
        return cls.from_limbs(ctx, codec.ints_to_limbs(values, ctx, reduce=reduce), device)

    @classmethod
    def random(cls, ctx, n, seed, stream_id=0, device='cuda'):
        """Deterministic synthetic residues (same recipe as oracle.synth_elements)."""
        out = cls.empty(ctx, n, device)
        check(lib.mpyc_b200_fill_random(ctx.handle, out.ptr, n, seed & (2**64 - 1), stream_id, _stream_ptr()))
        return out

    def to_limbs(self):
        a = self.t.contiguous().cpu().numpy()
        return a if self.ctx.binary else a.view(np.uint64)

    def to_ints(self):
        return codec.limbs_to_ints(self.to_limbs(), self.ctx)

    @property
    def ptr(self):
        return ctypes.c_void_p(self.t.data_ptr())

    def __len__(self):
        return self.t.shape[0]

    @property
    def n(self):
        return self.t.shape[0]

    def _like(self):
        return DeviceArray.empty(self.ctx, self.n, self.t.device)

    def _check_contiguous(self):
        if not self.t.is_contiguous():
            self.t = self.t.contiguous()

    # ---- arithmetic (finfields.py:1056-1124,1189-1281) ---------------------------------------------
    def _binop(self, other, op):
        self._check_contiguous()
        out = self._like()
        if isinstance(other, DeviceArray):
            if other.ctx is not self.ctx or other.n != self.n:
                raise ValueError('operands must share field and length')
            other._check_contiguous()
            check(lib.mpyc_b200_ff_binop(self.ctx.handle, op, self.ptr, other.ptr, out.ptr, self.n, _stream_ptr()))
        elif isinstance(other, (int, np.integer)):
            check(lib.mpyc_b200_ff_binop_scalar(self.ctx.handle, op, self.ptr, self.ctx.scalar_limbs(other), out.ptr,
                                                self.n, _stream_ptr()))
        else:
            return NotImplemented
        return out

    def __add__(self, other):
        return self._binop(other, _cabi.OP_ADD)

    __radd__ = __add__

    def __sub__(self, other):
        return self._binop(other, _cabi.OP_SUB)

    def __rsub__(self, other):
        return (-self)._binop(other, _cabi.OP_ADD)

    def __mul__(self, other):
        return self._binop(other, _cabi.OP_MUL)

    __rmul__ = __mul__

    def __neg__(self):
        self._check_contiguous()
        out = self._like()
        check(lib.mpyc_b200_ff_neg(self.ctx.handle, self.ptr, out.ptr, self.n, _stream_ptr()))
        return out

    def __pow__(self, e):
        """a ** e for one public integer exponent (negative allowed: powmod semantics, finfields.py:1408-1414)."""
        if not isinstance(e, (int, np.integer)):
            return NotImplemented
        e = int(e)
        base = self
        if e < 0:
            base, e = self.reciprocal(), -e
        base._check_contiguous()
        q1 = self.ctx.order - 1
        if e > q1:   # a^(q-1) = 1 for a != 0, and 0^e = 0 for e > 0: keep the exponent in 1..q-1
            e = e % q1 or q1
        out = base._like()
        nl = max(1, (e.bit_length() + 63) // 64)
        check(lib.mpyc_b200_ff_pow(self.ctx.handle, base.ptr, _cabi.u64_array(_cabi.int_to_limbs(e, nl)), nl, out.ptr,
                                   self.n, _stream_ptr()))
        return out

    def reciprocal(self):
        """Elementwise inverse; ZeroDivisionError if any element is 0 (gmpy2.invert, finfields.py:1416-1422)."""
        self._check_contiguous()
        out = self._like()
        check(lib.mpyc_b200_ff_inv(self.ctx.handle, self.ptr, out.ptr, self.n, _stream_ptr()))
        return out

    def __truediv__(self, other):
        if isinstance(other, DeviceArray):
            return self * other.reciprocal()
        if isinstance(other, (int, np.integer)) and not self.ctx.binary:
            return self * pow(int(other), -1, self.ctx.order)
        return NotImplemented

    def __lshift__(self, k):
        if self.ctx.binary:
            return NotImplemented   # polynomial shifts of GF(2^8) arrays are not part of the batched surface
        return self * pow(2, int(k), self.ctx.order)

    def __rshift__(self, k):
        """'>> k' multiplies by (2^k)^-1 mod p (finfields.py:1250-1259) -- not a bit shift."""
        if self.ctx.binary:
            return NotImplemented
        return self * pow(pow(2, int(k), self.ctx.order), -1, self.ctx.order)

    def sqrt(self, INV=False):
        self._check_contiguous()
        out = self._like()
        check(lib.mpyc_b200_ff_sqrt(self.ctx.handle, self.ptr, 1 if INV else 0, out.ptr, self.n, _stream_ptr()))
        return out

    def is_sqr(self):
        self._check_contiguous()
        out = torch.empty(self.n, dtype=torch.uint8, device=self.t.device)
        check(lib.mpyc_b200_ff_is_sqr(self.ctx.handle, self.ptr, ctypes.c_void_p(out.data_ptr()), self.n, _stream_ptr()))
        return out.bool()

    def signed_(self):
        """Host-side signed representatives (finfields.py:1395-1398)."""
        p = self.ctx.modulus
        v = self.to_ints()
        return np.where(v > p >> 1, v - p, v)

    def count_mismatch(self, other):
        cnt = torch.zeros(1, dtype=torch.int64, device=self.t.device)
        self._check_contiguous()
        other._check_contiguous()
        check(lib.mpyc_b200_count_mismatch(self.ctx.handle, self.ptr, other.ptr, self.n,
                                           ctypes.c_void_p(cnt.data_ptr()), _stream_ptr()))
        return int(cnt.item())


class DeviceMatrix:
    """rows x n elements (row-major, row stride in elements) -- share or coefficient matrices."""

    __slots__ = ('ctx', 't')

    def __init__(self, ctx, tensor):
        self.ctx = ctx
        self.t = tensor   # int64 (rows, n, L) with stride(0) = row stride * L, or uint8 (rows, n)

    @classmethod
    def empty(cls, ctx, rows, n, device='cuda'):
        return cls(ctx, _alloc(ctx, rows, n, device))

    @classmethod
    def from_ints(cls, ctx, rows_of_values, device='cuda'):
        rows = [codec.ints_to_limbs(r, ctx) for r in rows_of_values]
        out = cls.empty(ctx, len(rows), rows[0].shape[0] if rows else 0, device)
        for i, r in enumerate(rows):
            out.t[i].copy_(torch.from_numpy(r if ctx.binary else r.view(np.int64)))
        return out

    @property
    def rows(self):
        return self.t.shape[0]

    @property
    def n(self):
        return self.t.shape[1]

    @property
    def stride(self):
        """row stride in elements"""
        if self.t.shape[0] <= 1:
            return max(self.n, 1)
        return self.t.stride(0) // (1 if self.ctx.binary else self.ctx.nlimbs)

    @property
    def ptr(self):
        return ctypes.c_void_p(self.t.data_ptr())

    def row(self, i):
        return DeviceArray(self.ctx, self.t[i])

    def to_ints(self):
        return [self.row(i).to_ints() for i in range(self.rows)]


def shamir_split(ctx, secrets: DeviceArray, coeffs, t, m, out=None):
    """Device-resident np_random_split with explicit coefficients (mpyc/thresha.py:47-64).

    coeffs: DeviceMatrix with t rows (row j-1 = coefficient of X^j), or None when t == 0."""
    n = secrets.n
    secrets._check_contiguous()
    if out is None:
        out = DeviceMatrix.empty(ctx, m, n, secrets.t.device)
    cptr, cstride = (coeffs.ptr, coeffs.stride) if (t > 0 and coeffs is not None) else (ctypes.c_void_p(0), n)
    check(lib.mpyc_b200_shamir_split(ctx.handle, secrets.ptr, cptr, cstride, out.ptr, out.stride, n, t, m, _stream_ptr()))
    return out


def shamir_recombine(ctx, xs, rows, x_rs=0, out=None):
    """Device-resident np_recombine (mpyc/thresha.py:119-132). rows: list of DeviceArray (one per x in xs)."""
    single = not isinstance(x_rs, (list, tuple))
    pts = [x_rs] if single else list(x_rs)
    n = rows[0].n
    for r in rows:
        r._check_contiguous()
    if out is None:
        out = DeviceMatrix.empty(ctx, len(pts), n, rows[0].t.device)
    check(lib.mpyc_b200_shamir_recombine(ctx.handle, _cabi.ptr_array([r.t.data_ptr() for r in rows]),
                                         _cabi.i64_array([int(x) for x in xs]), len(rows),
                                         _cabi.i64_array([int(x) for x in pts]), len(pts), out.ptr, out.stride, n,
                                         _stream_ptr()))
    return out.row(0) if single else out


def shamir_split_generate(ctx, secrets: DeviceArray, t, m, key=None, nonce=0, out=None):
    """Share generation with coefficients drawn INSIDE the kernel from a ChaCha20 keystream (never written
    to memory).  key: 32 bytes of fresh CSPRNG output (default: os.urandom(32)); nonce: 63-bit call counter.
    The role of secrets.randbelow in mpyc/thresha.py:58-60; not bit-reproducible against anything unless the
    key is fixed (tests do that)."""
    import os
    key = os.urandom(32) if key is None else bytes(key)
    if len(key) != 32:
        raise ValueError('key must be 32 bytes')
    n = secrets.n
    secrets._check_contiguous()
    if out is None:
        out = DeviceMatrix.empty(ctx, m, n, secrets.t.device)
    kbuf = (ctypes.c_uint8 * 32).from_buffer_copy(key)
    check(lib.mpyc_b200_shamir_split_generate(ctx.handle, secrets.ptr, out.ptr, out.stride, n, t, m, kbuf,
                                              int(nonce) & (2**63 - 1), _stream_ptr()))
    return out


def shamir_split_generate_rows(ctx, secrets: DeviceArray, t, m, row_ptrs, key=None, nonce=0):
    """As shamir_split_generate, every share row written to its own destination: row_ptrs = m device addresses
    (ints), each with room for n elements, 32-byte aligned for the vector path.  A row may live on another GPU
    (memory mapped through CUDA IPC with peer access enabled): the kernel then stores it there over NVLink."""
    import os
    key = os.urandom(32) if key is None else bytes(key)
    if len(key) != 32 or len(row_ptrs) != m:
        raise ValueError('key must be 32 bytes and row_ptrs must hold m addresses')
    secrets._check_contiguous()
    kbuf = (ctypes.c_uint8 * 32).from_buffer_copy(key)
    check(lib.mpyc_b200_shamir_split_generate_rows(ctx.handle, secrets.ptr, _cabi.ptr_array([int(a) for a in row_ptrs]),
                                                   secrets.n, t, m, kbuf, int(nonce) & (2**63 - 1), _stream_ptr()))


def matmul(ctx, A, B, r, k, c):
    """C = A @ B mod p for row-major DeviceArrays A (r*k elements) and B (k*c elements): DeviceArray of r*c
    elements (FiniteFieldArray.__matmul__, mpyc/finfields.py:1126-1146)."""
    if A.n != r * k or B.n != k * c:
        raise ValueError('matmul: shapes do not match the buffers')
    A._check_contiguous()
    B._check_contiguous()
    out = DeviceArray.empty(ctx, r * c, A.t.device)
    check(lib.mpyc_b200_ff_matmul(ctx.handle, A.ptr, B.ptr, out.ptr, r, k, c, _stream_ptr()))
    return out


def matmul_int(ctx, X, w, r, k, c, w_left=False):
    """C = X @ W mod p, or W @ X with w_left, on the K14 kernels: X a row-major DeviceArray of r*k (w_left: k*c) field
    elements, w a NumPy integer array of k*c (w_left: r*k) entries (FiniteFieldArray @ an integer ndarray,
    mpyc/finfields.py:1126-1146).  The entries go to the device as 64-bit integers, never as Python ints: int8 ... int64 and
    uint8 ... uint32 as int64, uint64 as itself with the kernel's unsigned flag.  Returns a DeviceArray of r*c elements."""
    w = np.asarray(w)
    if w.dtype.kind not in 'iu':
        raise TypeError(f'matmul_int: integer entries expected, not {w.dtype}')
    unsigned = w.dtype == np.uint64
    buf = np.ascontiguousarray(w).view(np.int64) if unsigned else np.ascontiguousarray(w, dtype=np.int64)
    if X.n != (k * c if w_left else r * k) or buf.size != (r * k if w_left else k * c):
        raise ValueError('matmul_int: shapes do not match the buffers')
    X._check_contiguous()
    if not buf.flags.writeable:           # torch.from_numpy warns about read-only arrays
        buf = buf.copy()
    W = torch.from_numpy(buf.reshape(-1)).to(X.t.device)
    out = DeviceArray.empty(ctx, r * c, X.t.device)
    check(lib.mpyc_b200_ff_matmul_int(ctx.handle, X.ptr, ctypes.c_void_p(W.data_ptr()), 1 if unsigned else 0,
                                      1 if w_left else 0, out.ptr, r, k, c, _stream_ptr()))
    return out


# ---- protocol-local algebra on raw share values (SURVEY 8f N3 / N4; csrc/local.cuh) -----------------------------

def fma(a: DeviceArray, b, c: DeviceArray):
    """a*b + c, or a*a + c when b is None -- np_random_bits' `_r.value**2 + z.value` (mpyc/runtime.py:4252)."""
    if c.ctx is not a.ctx or c.n != a.n or (b is not None and (b.ctx is not a.ctx or b.n != a.n)):
        raise ValueError('operands must share field and length')
    for x in (a, b, c):
        if x is not None:
            x._check_contiguous()
    out = a._like()
    check(lib.mpyc_b200_ff_fma(a.ctx.handle, a.ptr, b.ptr if b is not None else ctypes.c_void_p(0), c.ptr, out.ptr, a.n,
                               _stream_ptr()))
    return out


def axpb(a: DeviceArray, s, t):
    """a*s + t for public integers s, t (reduced here) -- the affine steps on raw values: `bits += 1; bits *= (p+1)>>1;
    bits <<= f` (mpyc/runtime.py:4267-4271), `(r_bits << 1) - 1` (:3646), `x + (1 << l)` (:3656)."""
    a._check_contiguous()
    q = a.ctx.order
    out = a._like()
    check(lib.mpyc_b200_ff_axpb(a.ctx.handle, a.ptr, a.ctx.scalar_limbs(int(s) % q), a.ctx.scalar_limbs(int(t) % q), out.ptr,
                                a.n, _stream_ptr()))
    return out


def low_bits(a: DeviceArray, nbits):
    """a & (2^nbits - 1) on canonical residues -- `c.value & ((1<<f) - 1)` (mpyc/runtime.py:870, 3657)."""
    a._check_contiguous()
    out = a._like()
    check(lib.mpyc_b200_ff_low_bits(a.ctx.handle, a.ptr, int(nbits), out.ptr, a.n, _stream_ptr()))
    return out


def nonzero(a: DeviceArray, want_mask=True):
    """(bool tensor a != 0 or None, number of non-zero elements) -- `_r2.value != 0` (mpyc/runtime.py:4254-4255)."""
    a._check_contiguous()
    mask = torch.empty(a.n, dtype=torch.uint8, device=a.t.device) if want_mask else None
    cnt = torch.zeros(1, dtype=torch.int64, device=a.t.device)
    check(lib.mpyc_b200_ff_nonzero(a.ctx.handle, a.ptr, ctypes.c_void_p(mask.data_ptr() if want_mask else 0),
                                   ctypes.c_void_p(cnt.data_ptr()), a.n, _stream_ptr()))
    return (mask.bool() if want_mask else None), int(cnt.item())


def bits_compose(bits: DeviceArray, n, f, descending=False):
    """out[i] = sum_j bits[i*f + j] << e(j) mod p, e(j) = j or f-1-j: `np.sum(r_bits.reshape((n, f)) << shifts, axis=1)`
    (mpyc/runtime.py:860, 3650-3651, 4415).  bits: n*f residues, row-major."""
    if bits.n != n * f:
        raise ValueError('bits_compose: buffer does not hold n*f elements')
    bits._check_contiguous()
    out = DeviceArray.empty(bits.ctx, n, bits.t.device)
    if n and f:
        check(lib.mpyc_b200_ff_bits_compose(bits.ctx.handle, bits.ptr, n, f, 1 if descending else 0, out.ptr, _stream_ptr()))
    elif n:
        out.t.zero_()
    return out


def bits_decompose(c: DeviceArray, l, descending=False):
    """DeviceMatrix (l, n): row j = bit e(j) of every c[i] as a field element: `np.right_shift.outer(c, shifts).T & 1`
    (mpyc/runtime.py:3659-3660, 4422-4423)."""
    c._check_contiguous()
    out = DeviceMatrix.empty(c.ctx, l, c.n, c.t.device)
    if l and c.n:
        check(lib.mpyc_b200_ff_bits_decompose(c.ctx.handle, c.ptr, c.n, l, 1 if descending else 0, out.ptr, out.stride,
                                              _stream_ptr()))
    return out


def conv2d(X: DeviceArray, W: DeviceArray, B: DeviceArray, k, r, m, n, v, s):
    """np_cnnmnist's convolvetensor body (demos/np_cnnmnist.py:69-81) mod p: X (k,r,m,n), W (v,r,s,s), B (v) row-major
    -> Y (k,v,m,n)."""
    if X.n != k * r * m * n or W.n != v * r * s * s or B.n != v:
        raise ValueError('conv2d: shapes do not match the buffers')
    for x in (X, W, B):
        x._check_contiguous()
    out = DeviceArray.empty(X.ctx, k * v * m * n, X.t.device)
    check(lib.mpyc_b200_ff_conv2d(X.ctx.handle, X.ptr, W.ptr, B.ptr, out.ptr, k, r, m, n, v, s, _stream_ptr()))
    return out


def bits_decompose_flat(c: DeviceArray, l, descending=False):
    """As bits_decompose, into ONE contiguous buffer of l*n elements (row-major (l, n), no row padding)."""
    c._check_contiguous()
    out = DeviceArray.empty(c.ctx, l * c.n, c.t.device)
    if l and c.n:
        check(lib.mpyc_b200_ff_bits_decompose(c.ctx.handle, c.ptr, c.n, l, 1 if descending else 0, out.ptr, c.n, _stream_ptr()))
    return out


def transpose(a: DeviceArray, rows, cols):
    """(rows, cols) row-major -> (cols, rows): `r_bits.T` (mpyc/runtime.py:3661)."""
    if a.n != rows * cols:
        raise ValueError('transpose: buffer does not hold rows*cols elements')
    a._check_contiguous()
    out = a._like()
    check(lib.mpyc_b200_ff_transpose(a.ctx.handle, a.ptr, rows, cols, out.ptr, _stream_ptr()))
    return out


def cumsum_rows(a: DeviceArray, rows, cols):
    """Running sums down the rows of a (rows, cols) matrix: `np.cumsum(x, axis=0)` mod p (mpyc/runtime.py:3667)."""
    if a.n != rows * cols:
        raise ValueError('cumsum_rows: buffer does not hold rows*cols elements')
    a._check_contiguous()
    out = a._like()
    check(lib.mpyc_b200_ff_cumsum_rows(a.ctx.handle, a.ptr, rows, cols, out.ptr, _stream_ptr()))
    return out


def _check_elements(a: DeviceArray, shape, what):
    n = 1
    for s in shape:
        n *= int(s)
    if a.n != n:
        raise ValueError(f'{what}: buffer does not hold the {n} elements of shape {tuple(shape)}')
    a._check_contiguous()


def sum_axis(a: DeviceArray, shape, axis=None, keepdims=False, initial=0):
    """np.sum(a.reshape(shape), axis=axis, keepdims=keepdims, initial=initial) mod p on the K7 kernels (Runtime.np_sum,
    mpyc/runtime.py:3476-3506; FiniteFieldArray.sum, mpyc/finfields.py:1332-1337).  axis: None, an int or a tuple, negative
    axes allowed.  Returns (DeviceArray of the result's elements, result shape); a 0-d result is one element."""
    from mpyc_b200 import axes
    _check_elements(a, shape, 'sum_axis')
    passes, out_shape = axes.sum_plan(shape, axis, keepdims)
    init = a.ctx.scalar_limbs(int(initial) % a.ctx.order)
    cur = a
    for j, (O, R, I) in enumerate(passes):
        out = DeviceArray.empty(a.ctx, O * I, a.t.device)
        last = j == len(passes) - 1
        check(lib.mpyc_b200_ff_sum_axis(a.ctx.handle, cur.ptr, O, R, I, init if last else None, out.ptr, _stream_ptr()))
        cur = out
    return cur, out_shape


def cumsum_axis(a: DeviceArray, shape, axis=None, include_initial=False):
    """np.cumsum(a.reshape(shape), axis) (axis=None: flattened) and, with include_initial, np.cumulative_sum(...,
    include_initial=True) mod p on the K7 kernels (mpyc/runtime.py:3510-3549).  Returns (DeviceArray, result shape)."""
    from mpyc_b200 import axes
    _check_elements(a, shape, 'cumsum_axis')
    (O, R, I), out_shape = axes.scan_plan(shape, axis, include_initial)
    out = DeviceArray.empty(a.ctx, O * (R + (1 if include_initial else 0)) * I, a.t.device)
    check(lib.mpyc_b200_ff_cumsum_axis(a.ctx.handle, a.ptr, O, R, I, 1 if include_initial else 0, out.ptr, _stream_ptr()))
    return out, out_shape


def prod_axis(a: DeviceArray, shape, axis=None, keepdims=False, initial=1):
    """np.prod(a.reshape(shape), axis=axis, keepdims=keepdims, initial=initial) mod p on the K13 kernels
    (FiniteFieldArray.prod, mpyc/finfields.py:1339-1349).  axis: None, an int or a tuple, negative axes allowed; a tuple of
    axes that are not adjacent is reduced one run of adjacent axes at a time, as sum_axis does.  Returns (DeviceArray of
    the result's elements, result shape); a 0-d result is one element."""
    from mpyc_b200 import axes
    _check_elements(a, shape, 'prod_axis')
    passes, out_shape = axes.sum_plan(shape, axis, keepdims)
    init = a.ctx.scalar_limbs(int(initial) % a.ctx.order)
    cur = a
    for j, (O, R, I) in enumerate(passes):
        out = DeviceArray.empty(a.ctx, O * I, a.t.device)
        last = j == len(passes) - 1
        check(lib.mpyc_b200_ff_prod_axis(a.ctx.handle, cur.ptr, O, R, I, init if last else None, out.ptr, _stream_ptr()))
        cur = out
    return cur, out_shape


def cumprod_axis(a: DeviceArray, shape, axis=None, include_initial=False):
    """np.cumprod(a.reshape(shape), axis) (axis=None: flattened) and, with include_initial, np.cumulative_prod(...,
    include_initial=True) mod p on the K13 kernels.  Returns (DeviceArray, result shape)."""
    from mpyc_b200 import axes
    _check_elements(a, shape, 'cumprod_axis')
    (O, R, I), out_shape = axes.scan_plan(shape, axis, include_initial)
    out = DeviceArray.empty(a.ctx, O * (R + (1 if include_initial else 0)) * I, a.t.device)
    check(lib.mpyc_b200_ff_cumprod_axis(a.ctx.handle, a.ptr, O, R, I, 1 if include_initial else 0, out.ptr, _stream_ptr()))
    return out, out_shape


def all_any_axis(a: DeviceArray, shape, axis=None, keepdims=False, any=False):
    """np.all (any=False) / np.any (any=True) of a.reshape(shape) along axis, as field elements 0 / 1 (the reference's
    `cls(bool_array)`, mpyc/finfields.py:766-819) on the K13 kernels.  Returns (DeviceArray, result shape).  A reduction to
    one bool needs no kernel of its own: nonzero's count answers it."""
    from mpyc_b200 import axes
    _check_elements(a, shape, 'all_any_axis')
    passes, out_shape = axes.sum_plan(shape, axis, keepdims)
    cur = a
    for O, R, I in passes:
        out = DeviceArray.empty(a.ctx, O * I, a.t.device)
        check(lib.mpyc_b200_ff_all_any_axis(a.ctx.handle, cur.ptr, O, R, I, 1 if any else 0, out.ptr, _stream_ptr()))
        cur = out
    return cur, out_shape


def _view(v, index_keep):
    """mpyc_b200.layout.View -> the C struct (its index table stays alive in index_keep)."""
    c = _cabi.View()
    c.offset, c.rank, c.index_axis = v.offset, len(v.shape), v.index_axis
    if c.rank > _cabi.VIEW_RANK:
        raise ValueError(f'view of rank {c.rank} > {_cabi.VIEW_RANK}: collapse it first (mpyc_b200.layout.collapse)')
    for k, (e, s) in enumerate(zip(v.shape, v.strides)):
        c.extent[k], c.stride[k] = e, s
    if v.index_axis >= 0:
        idx = np.ascontiguousarray(v.index, dtype=np.int64)
        index_keep.append(idx)
        c.index = idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    return c


def _elem_bytes(ctx):
    return 1 if ctx.binary else 8 * ctx.nlimbs


def copy_view(src: DeviceArray, src_view, dst: DeviceArray, dst_view):
    """dst[dst_view] <- src[src_view] on the K8 kernels, for views (mpyc_b200.layout.View) of equal extents; any field.
    Index tables are uploaded from the views' NumPy arrays."""
    if src.ctx is not dst.ctx:
        raise ValueError('copy_view: arrays of different fields')
    keep = []
    sv, dv = _view(src_view, keep), _view(dst_view, keep)
    check(lib.mpyc_b200_copy_view(_elem_bytes(src.ctx), src.ptr, src.n, ctypes.byref(sv), dst.ptr, dst.n, ctypes.byref(dv),
                                  _stream_ptr()))


def binop_view(a: DeviceArray, a_view, b: DeviceArray, b_view, op):
    """a[a_view] (op) b[b_view] into a new contiguous array (C order of the views' extents) on the K8 kernel; op
    _cabi.OP_ADD / OP_SUB / OP_MUL, prime fields."""
    if a.ctx is not b.ctx:
        raise ValueError('binop_view: arrays of different fields')
    keep = []
    av, bv = _view(a_view, keep), _view(b_view, keep)
    out = DeviceArray.empty(a.ctx, a_view.size, a.t.device)
    check(lib.mpyc_b200_ff_binop_view(a.ctx.handle, op, a.ptr, a.n, ctypes.byref(av), b.ptr, b.n, ctypes.byref(bv), out.ptr,
                                      _stream_ptr()))
    return out


# ---- K15: GF(2^8) bit composition, broadcast arithmetic and stacked products (csrc/gf_local.cuh) ----------------------

def gf_bits_compose(bits: DeviceArray, n, l):
    """out[i] = sum_j bits[i l + j] X^j mod poly over GF(2^8), bits (n, l) row-major: np.sum(v << np.arange(l), axis=-1) of
    BinaryPolynomial values reduced by field.array (mpyc/runtime.py:4415, 4483).  A DeviceArray of n elements."""
    if bits.n != n * l:
        raise ValueError('gf_bits_compose: shape does not match the buffer')
    bits._check_contiguous()
    out = DeviceArray.empty(bits.ctx, n, bits.t.device)
    check(lib.mpyc_b200_gf_bits_compose(bits.ctx.handle, bits.ptr, n, l, out.ptr, _stream_ptr()))
    return out


def gf_binop_view(a: DeviceArray, a_view, b: DeviceArray, b_view, op):
    """a[a_view] (op) b[b_view] over GF(2^8) into a new contiguous array (C order of the views' extents); op _cabi.OP_ADD /
    OP_SUB (both XOR) / OP_MUL."""
    if a.ctx is not b.ctx:
        raise ValueError('gf_binop_view: arrays of different fields')
    keep = []
    av, bv = _view(a_view, keep), _view(b_view, keep)
    out = DeviceArray.empty(a.ctx, a_view.size, a.t.device)
    check(lib.mpyc_b200_gf_binop_view(a.ctx.handle, op, a.ptr, a.n, ctypes.byref(av), b.ptr, b.n, ctypes.byref(bv), out.ptr,
                                      _stream_ptr()))
    return out


def gf_matmul_batched(A: DeviceArray, a_stacked, B: DeviceArray, b_stacked, batch, r, k, c):
    """C[b] = A[b] @ B[b] over GF(2^8) for b < batch: A holds batch (a_stacked) or one r x k matrix, B batch (b_stacked) or
    one k x c matrix, all row-major.  A DeviceArray of batch * r * c elements."""
    if A.ctx is not B.ctx:
        raise ValueError('gf_matmul_batched: arrays of different fields')
    if A.n != (batch if a_stacked else 1) * r * k or B.n != (batch if b_stacked else 1) * k * c:
        raise ValueError('gf_matmul_batched: shapes do not match the buffers')
    A._check_contiguous()
    B._check_contiguous()
    out = DeviceArray.empty(A.ctx, batch * r * c, A.t.device)
    check(lib.mpyc_b200_gf_matmul_batched(A.ctx.handle, A.ptr, r * k if a_stacked else 0, B.ptr, k * c if b_stacked else 0,
                                          out.ptr, batch, r, k, c, _stream_ptr()))
    return out


# ---- K9: determinants, solves, inverses and powers of matrices (csrc/linalg.cuh) ------------------------------------

def det(a: DeviceArray, batch, n):
    """det of each n x n matrix of a (batch x n x n, row-major) as FiniteFieldArray.gauss_det computes it: row swaps do not
    change the sign (mpyc/finfields.py:916-955).  A DeviceArray of batch elements."""
    _check_elements(a, (batch, n, n), 'det')
    out = DeviceArray.empty(a.ctx, batch, a.t.device)
    check(lib.mpyc_b200_ff_det(a.ctx.handle, a.ptr, batch, n, out.ptr, _stream_ptr()))
    return out


def solve(a: DeviceArray, b, n, nrhs):
    """X (n x nrhs) with a X = b for a (n x n) and b (n x nrhs); b None: the inverse of a (nrhs = n).  ZeroDivisionError('no
    inverse exists') for a singular a (gauss_solve / gauss_inv, mpyc/finfields.py:872-914)."""
    _check_elements(a, (n, n), 'solve')
    if b is not None:
        if b.ctx is not a.ctx:
            raise ValueError('solve: arrays of different fields')
        _check_elements(b, (n, nrhs), 'solve')
    elif nrhs != n:
        raise ValueError('solve: the identity right-hand side has n columns')
    out = DeviceArray.empty(a.ctx, n * nrhs, a.t.device)
    check(lib.mpyc_b200_ff_solve(a.ctx.handle, a.ptr, n, b.ptr if b is not None else ctypes.c_void_p(0), nrhs, out.ptr,
                                 _stream_ptr()))
    return out


def inv(a: DeviceArray, n):
    return solve(a, None, n, n)


def identity(ctx, n, device='cuda'):
    e = DeviceArray(ctx, torch.zeros((n * n, ctx.nlimbs), dtype=torch.int64, device=device))
    e.t[::n + 1, 0] = 1
    return e


def matrix_power(a: DeviceArray, n, e):
    """a^e for an n x n matrix a and a Python int e: square and multiply on K1c (matrix_pow, mpyc/finfields.py:957-976);
    the inverse first for e < 0 (ZeroDivisionError for a singular a), the identity for e == 0."""
    _check_elements(a, (n, n), 'matrix_power')
    if e < 0:
        a, e = inv(a, n), -e
    c = None
    while e:
        if e & 1:
            c = a if c is None else matmul(a.ctx, c, a, n, n, n)
        e >>= 1
        if e:
            a = matmul(a.ctx, a, a, n, n, n)
    return identity(a.ctx, n, a.t.device) if c is None else c


# ---- K10: 1-D convolution (csrc/conv.cuh) ------------------------------------------------------------------------

def convolve(ctx, a: DeviceArray, m, b: DeviceArray, n, lo, count):
    """c[j] = sum_{i + l = lo + j} a[i] b[l] mod p for j < count: the window [lo, lo + count) of np.convolve(a, b)
    (m + n - 1 elements), computed alone (np.convolve of field arrays, mpyc/finfields.py:766-819).  A DeviceArray of
    count elements."""
    if a.ctx is not ctx or b.ctx is not ctx:
        raise ValueError('convolve: arrays of different fields')
    _check_elements(a, (m,), 'convolve')
    _check_elements(b, (n,), 'convolve')
    out = DeviceArray.empty(ctx, count, a.t.device)
    check(lib.mpyc_b200_ff_convolve(ctx.handle, a.ptr, m, b.ptr, n, lo, count, out.ptr, _stream_ptr()))
    return out


# ---- K11: division and selection (k_inv_batch with a numerator, csrc/select.cuh) ------------------------------------

def divide(num: DeviceArray, den: DeviceArray):
    """num[h] * den[h]^-1 in one Montgomery-trick pass (FiniteFieldArray.__truediv__, mpyc/finfields.py:1199-1206);
    ZeroDivisionError if any den[h] == 0."""
    if num.ctx is not den.ctx or num.n != den.n:
        raise ValueError('divide: operands must share field and length')
    num._check_contiguous()
    den._check_contiguous()
    out = num._like()
    check(lib.mpyc_b200_ff_div(num.ctx.handle, num.ptr, den.ptr, out.ptr, num.n, _stream_ptr()))
    return out


def _mask_tensor(mask, n, where):
    """A device uint8 tensor of n bytes from a device tensor (any dtype, nonzero = true) or a host bool / integer array."""
    if isinstance(mask, torch.Tensor):
        if mask.dtype not in (torch.uint8, torch.bool):
            mask = mask != 0
        mask = mask.reshape(-1).to(device=where, dtype=torch.uint8).contiguous()
    else:
        a = np.asarray(mask)
        if a.dtype.kind not in 'biu':
            raise TypeError('select: the mask must be a bool or integer array')
        mask = torch.from_numpy(np.ascontiguousarray(a.reshape(-1) != 0).view(np.uint8)).to(where)
    if mask.numel() != n:
        raise ValueError(f'select: the mask holds {mask.numel()} entries, not {n}')
    return mask


def select(mask, x, x_map, y, y_map, n=None, invert=False):
    """out[h] = mask[h] ? x[h] * sx + tx : y[h] * sy + ty (with invert: the other side), the np.where of field arrays and
    raw share values (mpyc/runtime.py:1819, 3614-3615).  x, y: DeviceArrays, or None for the constant tx / ty;
    x_map = (sx, tx), y_map = (sy, ty): public integers, reduced here.  mask: a device tensor or a host bool / integer
    array (uploaded).  n: the element count (needed when both sides are constants)."""
    arrays = [a for a in (x, y) if a is not None]
    if not arrays:
        raise ValueError('select: at least one side must be an array')
    ctx = arrays[0].ctx
    if n is None:
        n = arrays[0].n
    for a in arrays:
        if a.ctx is not ctx or a.n != n:
            raise ValueError('select: arrays must share field and length')
        a._check_contiguous()
    where = arrays[0].t.device
    m = _mask_tensor(mask, n, where)
    q, L = ctx.order, ctx.nlimbs

    def st(sm):
        s, t = sm
        return _cabi.u64_array(_cabi.int_to_limbs(int(s) % q, L) + _cabi.int_to_limbs(int(t) % q, L))
    out = DeviceArray.empty(ctx, n, where)
    null = ctypes.c_void_p(0)
    check(lib.mpyc_b200_ff_select(ctx.handle, ctypes.c_void_p(m.data_ptr()), 1 if invert else 0, x.ptr if x is not None else null,
                                  st(x_map), y.ptr if y is not None else null, st(y_map), out.ptr, n, _stream_ptr()))
    return out


def nonzero_mask(a: DeviceArray):
    """a != 0 as a device uint8 tensor (k_nonzero), without reading the count back to the host."""
    a._check_contiguous()
    mask = torch.empty(a.n, dtype=torch.uint8, device=a.t.device)
    cnt = torch.zeros(1, dtype=torch.int64, device=a.t.device)
    check(lib.mpyc_b200_ff_nonzero(a.ctx.handle, a.ptr, ctypes.c_void_p(mask.data_ptr()), ctypes.c_void_p(cnt.data_ptr()), a.n,
                                   _stream_ptr()))
    return mask


# ---- K12: per-element exponents (csrc/powexp.cuh) --------------------------------------------------------------------

def pow_exp(ctx, base, exps, signs, bits, device=None):
    """out[h] = base(h)^e[h] mod p (PrimeFieldArray._pow with an exponent array, mpyc/finfields.py:1409-1414;
    gmpy.powmod_exp_list, mpyc/gmpy.py:288-290).  base: a DeviceArray (one base per element) or a Python int (one public
    base, reduced here).  exps, signs, bits: codec.exponents_to_limbs's (limbs (n, EL), signs or None, B), uploaded here;
    signs only with an int base.  ZeroDivisionError for a zero base with signs.  A DeviceArray of n elements."""
    import torch
    exps = np.ascontiguousarray(exps, dtype=np.uint64)
    n, el = exps.shape
    if isinstance(base, DeviceArray):
        if base.ctx is not ctx or base.n != n:
            raise ValueError('pow_exp: bases and exponents must share field and length')
        base._check_contiguous()
        where = base.t.device
    else:
        _require_cuda()
        where = torch.device('cuda', torch.cuda.current_device()) if device is None else device
    e = torch.from_numpy(exps.view(np.int64)).to(where)
    s = torch.from_numpy(np.ascontiguousarray(signs, dtype=np.uint8)).to(where) if signs is not None else None
    out = DeviceArray.empty(ctx, n, where)
    null = ctypes.c_void_p(0)
    if isinstance(base, DeviceArray):
        d_base, h_base = base.ptr, null
    else:
        d_base, h_base = null, ctx.scalar_limbs(base)
    check(lib.mpyc_b200_ff_pow_exp(ctx.handle, d_base, h_base, ctypes.c_void_p(e.data_ptr()), el, int(bits),
                                   ctypes.c_void_p(s.data_ptr()) if s is not None else null, n, out.ptr, _stream_ptr(where)))
    return out


def binop_rows(a: DeviceArray, b: DeviceArray, op, rows, cols, reflected=False):
    """a (rows, cols) (op) b (cols) broadcast over the rows; reflected: b (op) a (mpyc/runtime.py:3670)."""
    if a.n != rows * cols or b.n != cols or a.ctx is not b.ctx:
        raise ValueError('binop_rows: shapes do not match the buffers')
    a._check_contiguous()
    b._check_contiguous()
    out = a._like()
    check(lib.mpyc_b200_ff_binop_rows(a.ctx.handle, op, 1 if reflected else 0, a.ptr, b.ptr, out.ptr, rows, cols, _stream_ptr()))
    return out
