"""Drop-in replacements for the reference's secret-sharing module, backed by the sm_90a engine.

Same names, argument meaning, return types and error behaviour as mpyc/thresha.py:
    random_split :23, np_random_split :47, _recombination_vector :67, recombine :88,
    np_recombine :119, _f_S_i :135, pseudorandom_share :144, np_pseudorandom_share :163,
    pseudorandom_share_zero :176, np_pseudorandom_share_0 :201, PRF :220
so that mpyc/runtime.py (which looks these up as module attributes at call time,
runtime.py:478-485,565-572,647-656,4057,4099) runs unchanged after mpyc_b200.install().

`field` is an MPyC field class (finfields.GF(...)) or anything with .modulus/.order/.array.
Data arrive as the reference hands them over -- Python ints in lists or NumPy object arrays -- are
packed into limb buffers (mpyc_b200.codec), pushed through the C ABI's host-buffer entry points
(H2D copy, kernel, D2H copy pipelined inside the library) and unpacked again.  The arithmetic runs
on the GPU only; there is no CPU fallback.

Randomness.  The reference draws coefficients with secrets.randbelow per element
(thresha.py:37,58-60).  `coefficient_source`, when set to a callable (order, count) -> ints, is
used instead -- the parity tests inject deterministic streams this way, in the reference's own
consumption order (np: (t, n) row-major; list: element-major, Horner order).  When None (default)
the coefficients are generated inside the kernel from a ChaCha20 stream keyed with 32 fresh bytes of
OS randomness per call (mpyc_b200_shamir_split_generate_host; t <= 4), or drawn from os.urandom in bulk
(64 bits wider than the modulus, then reduced) for GF(2^8) and t > 4.
"""
import ctypes
import os
from hashlib import shake_128
from math import prod

import numpy as np

from mpyc_b200 import _cabi, codec
from mpyc_b200._cabi import lib, check
from mpyc_b200.field import context_of_field
from mpyc_b200.wire import ShareRow, ShareRows
from mpyc_b200 import resident as _res

__all__ = ['random_split', 'recombine', 'pseudorandom_share', 'pseudorandom_share_zero',
           'np_random_split', 'np_recombine', 'np_pseudorandom_share', 'np_pseudorandom_share_0', 'PRF']

coefficient_source = None     # callable(order, count) -> sequence of ints, or None (CSPRNG)
device = 0                    # CUDA device ordinal used by the host-buffer entry points
prss_threads = 0              # host threads for the SHAKE128 sponges of one PRSS call (0 = all hardware threads)
limb_wire = False             # True: np_random_split returns limb-backed ShareRows (mpyc_b200.wire) that
                              # pickle as fixed-width bytes and feed np_recombine without becoming ints


def _ptr(a):
    return ctypes.c_void_p(a.__array_interface__['data'][0])


def _values_of(field, s):
    """Plain values of s: list/array of ints or field elements, or a field array."""
    arr_t = getattr(field, 'array', None)
    if arr_t is not None and isinstance(s, arr_t):
        s = s.value
    if isinstance(s, np.ndarray):
        return s.reshape(-1)
    if isinstance(s, (ShareRow, _res.LimbValue)):
        return s.__array__().reshape(-1)
    s = list(s)
    if s and isinstance(s[0], field):
        s = [a.value for a in s]
    return s


def _wrap_poly(field, ctx, ints):
    """GF(2^8): hand values back as the reference's polynomial objects (gfpx.BinaryPolynomial)."""
    if not ctx.binary:
        return ints
    tp = type(field.modulus)
    out = np.empty(len(ints), dtype=object)
    out[:] = [tp(int(v)) for v in ints]
    return out


def _draw(ctx, order, count):
    """count uniform residues as a limb array (count, L) / uint8 (count,)."""
    if coefficient_source is not None:
        return codec.ints_to_limbs(list(coefficient_source(order, count)), ctx)
    if ctx.binary:
        return np.frombuffer(os.urandom(count), dtype=np.uint8).copy()
    # 64 extra bits make the bias of the modular reduction < 2^-64
    nb = (ctx.bits + 64 + 7) // 8
    raw = os.urandom(count * nb)
    vals = [int.from_bytes(raw[i:i + nb], 'little') % order for i in range(0, count * nb, nb)]
    return codec.ints_to_limbs(vals, ctx, reduce=False)


def _split_limbs(ctx, sec, C, t, m):
    """sec: limbs (n, L); C: limbs (t, n, L) -> shares limbs (m, n, L) via the host-buffer ABI."""
    n = sec.shape[0]
    shape = (m, n) if ctx.binary else (m, n, ctx.nlimbs)
    shares = np.empty(shape, dtype=np.uint8 if ctx.binary else np.uint64)
    sec = np.ascontiguousarray(sec)
    C = np.ascontiguousarray(C)
    check(lib.mpyc_b200_shamir_split_host(ctx.handle, _ptr(sec), _ptr(C) if t else None, n, _ptr(shares), n, n, t, m,
                                          device))
    return shares


_nonce = [int.from_bytes(os.urandom(7), 'little')]


def _split_generate(ctx, sec, t, m):
    """Default (CSPRNG) path for prime fields: secrets go to the GPU, the coefficients are generated INSIDE
    the kernel from a ChaCha20 stream keyed with 32 fresh bytes of OS randomness per call
    (mpyc_b200_shamir_split_generate_host: H2D copy, kernel and D2H copy pipelined chunk by chunk) and never
    exist in memory; shares come back as a limb array (m, n, L)."""
    n = sec.shape[0]
    sec = np.ascontiguousarray(sec)
    shares = np.empty((m, n, ctx.nlimbs), dtype=np.uint64)
    _nonce[0] = (_nonce[0] + (1 << 20)) & (2**63 - 1)        # the library uses nonce + chunk index (< 2^20 chunks per call)
    key = (ctypes.c_uint8 * 32).from_buffer_copy(os.urandom(32))
    check(lib.mpyc_b200_shamir_split_generate_host(ctx.handle, _ptr(sec), _ptr(shares), n, n, t, m, key, _nonce[0], device))
    return shares


def _use_generate(ctx, t, n):
    return coefficient_source is None and not ctx.binary and 1 <= t <= 4 and n > 0


def _limb_secrets(field, s):
    """(store, n) when the secrets arrive limb-backed (a resident field array, its .value, or a ShareRow)."""
    arr_t = getattr(field, 'array', None)
    if arr_t is not None and isinstance(s, arr_t):
        s = _res.raw_value(s)
    lv = _res.as_limb_value(s)
    if lv is None or lv.ctx is not context_of_field(field):
        return None
    return lv.store, lv.size


def np_random_split(field, s, t, m):
    """Split each secret in s into m Shamir shares of degree t (0 <= t < m): object ndarray (m, n)."""
    ctx = context_of_field(field)
    limb = _limb_secrets(field, s)
    if limb is not None:
        # resident secrets (mpyc_b200.resident): no Python ints on the way in
        store, n = limb
        C = None
        if coefficient_source is not None or ctx.binary or not 1 <= t <= 4:
            C = _draw(ctx, field.order, t * n).reshape((t, n) if ctx.binary else (t, n, ctx.nlimbs))
        shares = _split_store(ctx, store, C, t, m) if n else np.zeros((m, 0) if ctx.binary else (m, 0, ctx.nlimbs),
                                                                  dtype=np.uint8 if ctx.binary else np.uint64)
    else:
        s = _values_of(field, s)
        n = len(s)
        sec = codec.ints_to_limbs(s, ctx)
        if _use_generate(ctx, t, n):
            shares = _split_generate(ctx, sec, t, m)
        else:
            C = _draw(ctx, field.order, t * n)
            C = C.reshape((t, n) if ctx.binary else (t, n, ctx.nlimbs))
            shares = _split_limbs(ctx, sec, C, t, m)
    if limb_wire:
        return ShareRows(ctx, shares, type(field.modulus) if ctx.binary else None)
    if not ctx.binary:
        return codec.limbs_to_ints(shares.reshape(m * n, ctx.nlimbs), ctx).reshape(m, n)   # one pass over all m rows
    out = np.empty((m, n), dtype=object)
    for i in range(m):
        out[i] = _wrap_poly(field, ctx, codec.limbs_to_ints(shares[i], ctx))
    return out


def _split_store(ctx, store, C, t, m):
    """Device round trip of a split whose secrets are already limbs (possibly in HBM): host limb rows (m, n, L)."""
    if isinstance(store, np.ndarray):      # host limbs (they came over the wire): the pipelined host-buffer entry points
        return _split_generate(ctx, store, t, m) if C is None else _split_limbs(ctx, store, C, t, m)
    return _res.backend.split(ctx, store, t, m, C)


def random_split(field, s, t, m):
    """List form: m lists of n ints.  A draw stream is consumed element by element, and the Horner
    evaluation of thresha.py:39-43 makes the FIRST value drawn for a secret the coefficient of X^t."""
    ctx = context_of_field(field)
    s = _values_of(field, s)
    n = len(s)
    sec = codec.ints_to_limbs(s, ctx)
    if _use_generate(ctx, t, n):
        shares = _split_generate(ctx, sec, t, m)
    else:
        c = _draw(ctx, field.order, t * n)
        c = c.reshape((n, t) if ctx.binary else (n, t, ctx.nlimbs))
        # element-major draws, first draw = highest power  ->  row j-1 = coefficient of X^j
        C = np.ascontiguousarray(np.swapaxes(c, 0, 1)[::-1])
        shares = _split_limbs(ctx, sec, C, t, m)
    return [list(_wrap_poly(field, ctx, codec.limbs_to_ints(shares[i], ctx))) for i in range(m)]


def _recombination_vector(field, xs, x_r):
    """Lagrange coefficients for x-coordinates xs at x_r (canonical values)."""
    ctx = context_of_field(field)
    lam = ctx.recombination_vector(xs, [x_r])[0]
    return list(_wrap_poly(field, ctx, lam)) if ctx.binary else lam


def _check_rows(ctx, rows):
    """Every share row must hold the same number of elements in the field's limb layout: rows come from peers
    (unpickled arrays or ShareRows whose length the sender chose), and the C ABI copies n elements from each
    (the reference raises from field.array(shares) on ragged input, thresha.py:128)."""
    if len(rows) > _cabi.MAX_POINTS:
        raise _cabi.UnsupportedFieldError(f'recombination of more than {_cabi.MAX_POINTS} shares is not covered by mpyc_b200')
    n = len(rows[0])
    want = (n,) if ctx.binary else (n, ctx.nlimbs)
    dt = np.uint8 if ctx.binary else np.uint64
    for r in rows:
        if isinstance(r, np.ndarray):
            ok = r.shape == want and r.dtype == dt
        else:                                     # a store in HBM (mpyc_b200.device.DeviceArray of this field)
            ok = len(r) == n and getattr(r, 'ctx', None) is ctx
        if not ok:
            raise ValueError(f'recombine: share rows must all have {n} elements of this field '
                             f'(got lengths {[len(x) for x in rows]})')
    return n


def _recombine_limbs(ctx, xs, rows, pts):
    n = _check_rows(ctx, rows)
    width = len(pts)
    shape = (width, n) if ctx.binary else (width, n, ctx.nlimbs)
    out = np.empty(shape, dtype=np.uint8 if ctx.binary else np.uint64)
    rows = [np.ascontiguousarray(r) for r in rows]
    check(lib.mpyc_b200_shamir_recombine_host(ctx.handle, _cabi.ptr_array([r.ctypes.data for r in rows]),
                                              _cabi.i64_array([int(x) for x in xs]), len(rows),
                                              _cabi.i64_array([int(x) for x in pts]), width, _ptr(out), n, n, device))
    return out


def _row_limbs(field, ctx, sh):
    """One share row as limbs: ShareRow / resident values as they are, anything else through the codec."""
    if isinstance(sh, ShareRow) and sh.ctx is ctx and sh._ints is None:
        return sh.limbs
    arr_t = getattr(field, 'array', None)
    lv = _res.as_limb_value(_res.raw_value(sh) if arr_t is not None and isinstance(sh, arr_t) else sh)
    if lv is not None and lv.ctx is ctx:
        return lv.store
    return codec.ints_to_limbs(_values_of(field, sh), ctx)


def np_recombine(field, points, x_rs=0):
    """Recombine shares given by points [(x_i, share_i), ...] at x_rs: field.array (n,) or (width, n)."""
    ctx = context_of_field(field)
    xs, shares = zip(*points)
    single = not isinstance(x_rs, list)
    pts = [x_rs] if single else x_rs
    rows = [_row_limbs(field, ctx, sh) for sh in shares]
    n = _check_rows(ctx, rows)
    if _res.resident and single and n:
        # the result stays limb-backed (in HBM): the next local operation / split consumes it without Python ints
        store = _recombine_store(ctx, xs, rows, pts)
        return field.array(_res.LimbValue(ctx, store, (n,), type(field.modulus) if ctx.binary else None), check=False)
    rows = [_res.backend.to_host(ctx, r) for r in rows]
    out = _recombine_limbs(ctx, xs, rows, pts)
    vals = np.empty((len(pts), n), dtype=object)
    for r in range(len(pts)):
        vals[r] = _wrap_poly(field, ctx, codec.limbs_to_ints(out[r], ctx))
    return field.array(vals[0] if single else vals, check=False)


def _recombine_store(ctx, xs, rows, pts):
    """Device round trip of a resident recombination: one store (DeviceArray) for the single point pts[0]."""
    return _res.backend.recombine(ctx, xs, rows, pts)[0]


def recombine(field, points, x_rs=0):
    """List form.  Returns reduced values (the reference leaves plain-int sums unreduced,
    thresha.py:109, and every caller reduces them: runtime.py:588,682); field elements in,
    field elements out (thresha.py:110-113)."""
    ctx = context_of_field(field)
    xs, shares = zip(*points)
    single = not isinstance(x_rs, list)
    pts = [x_rs] if single else x_rs
    is_elt = len(shares[0]) > 0 and isinstance(shares[0][0], field)
    rows = [codec.ints_to_limbs(_values_of(field, sh), ctx) for sh in shares]
    _check_rows(ctx, rows)
    out = _recombine_limbs(ctx, xs, rows, pts)
    sums = []
    for r in range(len(pts)):
        vals = list(_wrap_poly(field, ctx, codec.limbs_to_ints(out[r], ctx)))
        sums.append([field(v) for v in vals] if is_elt else vals)
    return sums[0] if single else sums


# ---------------------------------------------------------------------------------------------
# PRF and pseudorandom secret sharing
# ---------------------------------------------------------------------------------------------

class PRF:
    """Pseudorandom function: SHAKE128(key + input) cut into fixed-width little-endian chunks,
    each reduced modulo `bound` (same construction and attributes as mpyc/thresha.py:220-266)."""

    def __init__(self, key, bound):
        self.key = key
        self.max = bound
        width = ((bound - 1).bit_length() + 7) // 8
        if bound & (bound - 1):
            width += len(key)   # extra key-length bytes make the reduction bias negligible
        self.byte_length = width

    def stream(self, s, count):
        """Raw XOF output for `count` values."""
        return shake_128(self.key + s).digest(count * self.byte_length) if self.byte_length and count else b''

    def __call__(self, s, n=None):
        shape = n if isinstance(n, tuple) else None
        count = 1 if n is None else (prod(shape) if shape is not None else n)
        w = self.byte_length
        if count == 0:
            vals = []
        elif w == 0:
            vals = [0] * count
        else:
            raw, bound = self.stream(s, count), self.max
            vals = [int.from_bytes(raw[k:k + w], 'little') % bound for k in range(0, count * w, w)]
        if shape is not None:
            arr = np.empty(count, dtype=object)
            arr[:] = vals
            return arr.reshape(shape)
        return vals[0] if n is None else vals


def _f_S_i(field, m, i, S):
    """f_S(i+1) for the degree-t polynomial with f_S(0) = 1 and f_S(j+1) = 0 for j outside S."""
    ctx = context_of_field(field)
    xs = [0] + [x + 1 for x in range(m) if x not in S]
    lam = ctx.recombination_vector(xs, [i + 1])[0]
    return _wrap_poly(field, ctx, lam[:1])[0] if ctx.binary else lam[0]


def _prss(field, m, i, prfs, uci, n, d, weights):
    """Shared engine call: sum_S f_S(i) * sum_j PRF_S[h*d + j] * weights[j]  as a limb array (n, L)."""
    ctx = context_of_field(field)
    subsets = list(prfs.items())
    bound = subsets[0][1].max
    width = subsets[0][1].byte_length
    if any(f.max != bound for _, f in subsets):
        raise ValueError('all PRFs of one call must share their bound')
    # Which form of the bound the engine sees (thresha.py:257-261 computes chunk % bound for ANY bound):
    #   the field order, or 2^b <= order  -> folded into the combine kernel (bound_bits)
    #   anything else up to 2^256         -> reduced by its own kernel first (mpyc_b200_prss_host_bound):
    #       runtime._convert's (1 << (k+l)) // comb(m,t) + 1 and a source field's order used on a smaller
    #       target field (runtime.py:735-739,758-760)
    general = None
    if bound == field.order or bound == 1:      # bound 1: width 0, all values 0 (handled below)
        bound_bits = 0
    elif bound >= 2 and bound & (bound - 1) == 0 and bound <= field.order:
        bound_bits = bound.bit_length() - 1
    elif 2 <= bound <= 1 << 256:
        bound_bits, general = 0, bound
    else:
        raise _cabi.UnsupportedFieldError('PRF bounds above 2^256 are not covered by mpyc_b200')
    nl = max(ctx.nlimbs, 1)
    if n == 0:
        return np.zeros((0,) if ctx.binary else (0, nl), dtype=np.uint8 if ctx.binary else np.uint64)
    if width == 0:   # bound == 1: all PRF values are 0
        return np.zeros((n,) if ctx.binary else (n, nl), dtype=np.uint8 if ctx.binary else np.uint64)
    # The XOF runs inside the library: one SHAKE128 sponge per key subset on its own host thread, squeezed chunk
    # by chunk into pinned buffers while the previous chunk is copied and combined on the GPU
    # (mpyc_b200_prss_host) -- hashlib.shake_128().digest() holds the GIL and would serialise the subsets.
    keys = [f.key for _, f in subsets]
    klen = len(keys[0])
    if any(len(k) != klen for k in keys):
        raise ValueError('all PRF keys of one call must have the same length')
    coef = []
    for S, f in subsets:
        coef.extend(_cabi.int_to_limbs(int(_f_S_i(field, m, i, S)), nl))
    wl = []
    for w in weights:
        wl.extend(_cabi.int_to_limbs(int(w), nl))
    return _prss_device(ctx, keys, bytes(uci), d, width, bound_bits, coef, wl, n, general)


def _prss_device(ctx, keys, uci, d, width, bound_bits, coef, weights, n, general=None):
    """The device round trip of a PRSS call (mpyc_b200_prss_host[_bound]): keys / uci / constants in, limb array
    (n, L) out.  general: the PRF bound as an int when it is neither the field order nor 2^bound_bits <= order."""
    nl = max(ctx.nlimbs, 1)
    out = np.empty((n,) if ctx.binary else (n, nl), dtype=np.uint8 if ctx.binary else np.uint64)
    if general is None:
        check(lib.mpyc_b200_prss_host(ctx.handle, b''.join(keys), len(keys[0]), uci, len(uci), len(keys), d, width, bound_bits,
                                      _cabi.u64_array(coef), _cabi.u64_array(weights), _ptr(out), n, device, prss_threads))
    else:
        bl = _cabi.int_to_limbs(general, 5)
        check(lib.mpyc_b200_prss_host_bound(ctx.handle, b''.join(keys), len(keys[0]), uci, len(uci), len(keys), d, width,
                                            _cabi.u64_array(bl), 5, _cabi.u64_array(coef), _cabi.u64_array(weights), _ptr(out),
                                            n, device, prss_threads))
    return out


def _array_from_limbs(field, ctx, limbs):
    """field.array over a host limb array: limb-backed in resident mode, else unpacked to Python ints."""
    if _res.resident and len(limbs):
        return field.array(_res.LimbValue(ctx, limbs, (len(limbs),), type(field.modulus) if ctx.binary else None), check=False)
    return field.array(_wrap_poly(field, ctx, codec.limbs_to_ints(limbs, ctx)), check=False)


def np_pseudorandom_share(field, m, i, prfs, uci, n):
    """Pseudorandom Shamir shares of n random values for party i: field.array (n,)."""
    ctx = context_of_field(field)
    limbs = _prss(field, m, i, prfs, uci, n, 1, [1])
    return _array_from_limbs(field, ctx, limbs)


def pseudorandom_share(field, m, i, prfs, uci, n):
    """List form: n field elements."""
    ctx = context_of_field(field)
    limbs = _prss(field, m, i, prfs, uci, n, 1, [1])
    return [field(v) for v in _wrap_poly(field, ctx, codec.limbs_to_ints(limbs, ctx))]


def _powers(field, ctx, i, d, horner):
    """Weights for the d PRF values of one zero-share: np order (i+1)^(j+1), list (Horner) order (i+1)^(d-j)."""
    if ctx.binary:
        poly = ctx.modulus

        def mul(a, b):
            r = 0
            for _ in range(8):
                if b & 1:
                    r ^= a
                b >>= 1
                a <<= 1
                if a & 0x100:
                    a ^= poly
            return r
        pw, cur = [], 1
        for _ in range(d):
            cur = mul(cur, i + 1)
            pw.append(cur)
    else:
        pw = [pow(i + 1, j, ctx.modulus) for j in range(1, d + 1)]
    return pw[::-1] if horner else pw


def np_pseudorandom_share_0(field, m, i, prfs, uci, n):
    """Pseudorandom degree-2t... sharings of 0 (NumPy order: PRF value (h, j) multiplies (i+1)^(j+1))."""
    ctx = context_of_field(field)
    d = m - len(next(iter(prfs.keys())))
    limbs = _prss(field, m, i, prfs, uci, n, d, _powers(field, ctx, i, d, horner=False)) if d else None
    if limbs is None:
        return field.array(np.zeros(n, dtype=object), check=False)
    return _array_from_limbs(field, ctx, limbs)


def pseudorandom_share_zero(field, m, i, prfs, uci, n):
    """List form (Horner order: PRF value h*d+j multiplies (i+1)^(d-j), thresha.py:191-195)."""
    ctx = context_of_field(field)
    subsets = list(prfs.keys())
    d = m - len(subsets[0]) if subsets else 0
    if d == 0 or n == 0:
        zero = 0 if not ctx.binary else type(field.modulus)(0)
        return [field(zero) for _ in range(n)]
    limbs = _prss(field, m, i, prfs, uci, n, d, _powers(field, ctx, i, d, horner=True))
    return [field(v) for v in _wrap_poly(field, ctx, codec.limbs_to_ints(limbs, ctx))]
