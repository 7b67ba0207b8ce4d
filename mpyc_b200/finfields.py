"""Batched replacements for the per-element hot spots of the reference's prime-field arrays.

In mpyc/finfields.py the array type does inverse, power, square root and the quadratic-residue test by
mapping a Python function over the object array (np.vectorize around gmpy2.invert / powmod / legendre,
finfields.py:1408-1470) -- 5 us per element with the pure-Python stubs.  The functions below have the
signatures of those classmethods (value arrays in, value arrays out) and run one kernel over the whole
array; mpyc_b200.install.install(finfields=...) assigns them over PrimeFieldArray's methods.

Per-element exponents (a ** b with an integer array b of a's shape, non-negative) run on K12 through the resident
backend's pow_exp.  Other exponent arrays and non-Blum square roots are not batched here: those calls are handed back to
the reference implementation that was in place before install().
"""
import numpy as np

from mpyc_b200 import codec
from mpyc_b200.device import DeviceArray
from mpyc_b200.field import context_for


def _to_device(cls, a):
    ctx = context_for(cls.field.modulus)
    a = np.asarray(a, dtype=object)
    return ctx, a.shape, DeviceArray.from_ints(ctx, a.reshape(-1))


def _back(arr, shape):
    out = arr.to_ints()
    return out.reshape(shape)


def reciprocal(cls, a):
    """PrimeFieldArray._reciprocal (finfields.py:1416-1422); ZeroDivisionError if any element is 0."""
    ctx, shape, A = _to_device(cls, a)
    return _back(A.reciprocal(), shape)


def _power_exp(cls, a, b):
    """a ** b elementwise on K12 for an exponent ndarray b of a's shape (codec.exponents_to_limbs covers it, no entry
    negative), through resident.backend.pow_exp; None when not covered or the backend has no pow_exp."""
    from mpyc_b200 import resident
    a = np.asarray(a, dtype=object)
    if not resident._powexp_backend() or b.shape != a.shape or not a.size:
        return None
    ex = codec.exponents_to_limbs(b)
    if ex is None or ex[1] is not None:
        return None
    ctx = context_for(cls.field.modulus)
    resident.calls['pow_exp'] += 1
    out = resident.backend.pow_exp(ctx, codec.ints_to_limbs(a.reshape(-1), ctx), ex[0], None, ex[2])
    return codec.limbs_to_ints(resident.backend.to_host(ctx, out), ctx).reshape(a.shape)


def power(cls, a, b, _fallback=None):
    """PrimeFieldArray._pow (finfields.py:1408-1414) for one integer exponent (negative allowed), or per element for an
    integer exponent array of a's shape (K12)."""
    if isinstance(b, (int, np.integer)):
        ctx, shape, A = _to_device(cls, a)
        return _back(A ** int(b), shape)
    if isinstance(b, np.ndarray):
        r = _power_exp(cls, a, b)
        if r is not None:
            return r
    if _fallback is None:
        raise TypeError('per-element exponents are not batched by mpyc_b200')
    return _fallback(a, b)


def sqrt(cls, a, INV=False, _fallback=None):
    """PrimeFieldArray._sqrt (finfields.py:1424-1461) for Blum primes; ZeroDivisionError for INV on a 0."""
    p = cls.field.modulus
    if p & 3 != 3:
        if _fallback is None:
            raise TypeError('only Blum primes (p % 4 == 3) are batched by mpyc_b200')
        return _fallback(a, INV=INV)
    ctx, shape, A = _to_device(cls, a)
    return _back(A.sqrt(INV=INV), shape)


def is_sqr(cls, a):
    """PrimeFieldArray._is_sqr (finfields.py:1463-1470): boolean array, 0 counts as a square."""
    ctx, shape, A = _to_device(cls, a)
    return A.is_sqr().cpu().numpy().reshape(shape)


def matmul(cls, a, b):
    """(a @ b) % p for 2-D (or 1-D) value arrays (finfields.py:1126-1135)."""
    from mpyc_b200.device import matmul as dev_matmul
    ctx = context_for(cls.field.modulus)
    a, b = np.asarray(a, dtype=object), np.asarray(b, dtype=object)
    a2 = a.reshape(1, -1) if a.ndim == 1 else a
    b2 = b.reshape(-1, 1) if b.ndim == 1 else b
    r, k = a2.shape
    k2, c = b2.shape
    if k != k2:
        raise ValueError(f'matmul: shapes {a.shape} and {b.shape} do not align')
    out = dev_matmul(ctx, DeviceArray.from_ints(ctx, a2.reshape(-1)), DeviceArray.from_ints(ctx, b2.reshape(-1)), r, k, c)
    res = out.to_ints().reshape(r, c)
    if a.ndim == 1 and b.ndim == 1:
        return res[0, 0]
    if a.ndim == 1:
        return res[0]
    if b.ndim == 1:
        return res[:, 0]
    return res
