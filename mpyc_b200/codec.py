"""Conversions between the reference's data representation and limb buffers.

MPyC field arrays hold NumPy dtype=object arrays of Python ints (mpyc/finfields.py:703-725); the
kernels work on little-endian 64-bit limbs, `nlimbs` per element (one byte per element for GF(2^8)).
The fixed-width little-endian byte string of FiniteFieldElement.to_bytes/from_bytes
(mpyc/finfields.py:91-102) is the same layout when byte_length == 8*nlimbs; `wire_to_limbs` /
`limbs_to_wire` handle the general byte_length.
"""
import numpy as np

from mpyc_b200 import _pycodec   # C extension built in-tree by mpyc_b200._build (csrc/pycodec.c)


def ints_to_limbs(values, ctx, reduce=True):
    """values: iterable / object ndarray of Python ints (any sign/size if reduce) -> uint64 (n, nlimbs),
    or uint8 (n,) for GF(2^8) (values may be ints or gfpx polynomials: int() gives the encoding)."""
    if ctx.binary:
        flat = [int(v) for v in np.asarray(values, dtype=object).reshape(-1)]
        if any(v < 0 or v > 255 for v in flat):
            raise ValueError('GF(2^8) values must be reduced polynomials (0..255)')
        return np.array(flat, dtype=np.uint8)
    L, p = ctx.nlimbs, ctx.modulus
    if isinstance(values, np.ndarray):
        values = values.reshape(-1).tolist()     # ~10-20 ns per element; PySequence_Fast needs a list/tuple
    buf = _pycodec.pack(values, 8 * L, p)        # reduces out-of-range values mod p
    return np.frombuffer(buf, dtype='<u8').reshape(-1, L)


def limbs_to_ints(limbs, ctx):
    """uint64 (n, nlimbs) (or uint8 (n,)) -> object ndarray (n,) of Python ints."""
    if ctx.binary:
        out = np.empty(limbs.shape[0], dtype=object)
        out[:] = [int(v) for v in limbs.tolist()]
        return out
    limbs = np.ascontiguousarray(limbs, dtype=np.uint64)
    n, L = limbs.shape
    out = np.empty(n, dtype=object)          # freshly allocated, C-contiguous, n object slots (all None)
    if n:
        _pycodec.unpack_into(limbs, 8 * L, out.ctypes.data)
    return out


def wire_to_limbs(data, ctx):
    """Fixed-width little-endian wire bytes (field.to_bytes, finfields.py:91-95) -> limb array."""
    r = ctx.byte_length
    raw = np.frombuffer(data, dtype=np.uint8)
    if ctx.binary:
        return raw.copy()
    n = raw.shape[0] // r
    out = np.zeros((n, 8 * ctx.nlimbs), dtype=np.uint8)
    out[:, :r] = raw.reshape(n, r)
    return out.view('<u8').reshape(n, ctx.nlimbs)


def limbs_to_wire(limbs, ctx):
    """Limb array -> fixed-width little-endian wire bytes (field.from_bytes inverse)."""
    if ctx.binary:
        return np.ascontiguousarray(limbs, dtype=np.uint8).tobytes()
    r = ctx.byte_length
    n = limbs.shape[0]
    raw = np.ascontiguousarray(limbs, dtype='<u8').view(np.uint8).reshape(n, 8 * ctx.nlimbs)
    return np.ascontiguousarray(raw[:, :r]).tobytes()


MAX_EXP_LIMBS = 4     # K12 takes exponents of up to 256 bits


def exponents_to_limbs(e):
    """Exponents for K12 (mpyc_b200_ff_pow_exp): an int64 / uint64 ndarray, an object ndarray of Python ints, or a list /
    tuple of Python ints -> (limbs uint64 (n, EL), signs uint8 (n,) or None when no entry is negative, B), with EL =
    max(1, ceil(B / 64)) limbs of each magnitude and B the largest bit length.  None when not covered: other dtypes (bool,
    float, smaller integers), entries that are not ints, or exponents wider than 256 bits."""
    if isinstance(e, np.ndarray) and e.dtype.kind in 'iu':
        if e.dtype.itemsize != 8:
            return None
        u = np.ascontiguousarray(e.reshape(-1)).view(np.uint64)
        signs = None
        if e.dtype.kind == 'i' and (neg := u >> np.uint64(63)).any():
            signs = neg.astype(np.uint8)
            u = np.where(signs != 0, ~u + np.uint64(1), u)      # |e|, also for -2^63
        top = int(u.max()) if u.size else 0
        return u.reshape(-1, 1), signs, top.bit_length()
    if isinstance(e, np.ndarray):
        if e.dtype != object:
            return None
        e = e.reshape(-1).tolist()
    elif not isinstance(e, (list, tuple)):
        return None
    r = _pycodec.pack_exponents(e, MAX_EXP_LIMBS)
    if r is None:
        return None
    limbs, signs, bits, el = r
    signs = None if signs is None else np.frombuffer(signs, dtype=np.uint8)
    return np.frombuffer(limbs, dtype='<u8').reshape(-1, el), signs, bits
