"""TEST INFRASTRUCTURE: K11's device calls (resident.CudaBackend.divide / select / inverse / power / is_sqr and the count-only
nonzero) answered on host limb arrays with Python ints, straight from their definitions, for the CPU stand-in backend of
tests/oracle_device.py.  Never imported by the package."""
import numpy as np

from mpyc_b200 import codec
from oracle import shamir_oracle as orc


def divide(self, ctx, num, den):
    p = ctx.modulus
    x, y = self._ints(ctx, num), self._ints(ctx, den)
    if any(v % p == 0 for v in y):
        raise ZeroDivisionError('inverse of zero')
    return codec.ints_to_limbs([a * pow(b, -1, p) % p for a, b in zip(x, y)], ctx)


def inverse(self, ctx, a):
    return divide(self, ctx, codec.ints_to_limbs([1] * len(a), ctx), a)


def power(self, ctx, a, e):
    p = ctx.modulus
    x = self._ints(ctx, a)
    if e < 0 and any(v == 0 for v in x):
        raise ZeroDivisionError('inverse of zero')
    return codec.ints_to_limbs([pow(v, e, p) for v in x], ctx)


def is_sqr(self, ctx, a):
    return np.array(orc.ff_is_sqr(ctx.modulus, self._ints(ctx, a)), dtype=bool)


def nonzero(self, ctx, a, want_mask=True):
    mask = np.array(orc.local_nonzero(self._ints(ctx, a)), dtype=bool)
    return (mask if want_mask else None), int(mask.sum())


def select(self, ctx, mask, x, x_map, y, y_map, n):
    """mask: host bool array, or a store whose nonzero elements select x"""
    p = ctx.modulus
    m = mask if isinstance(mask, np.ndarray) and mask.dtype == bool else np.array([v != 0 for v in self._ints(ctx, mask)])
    assert m.shape == (n,)

    def side(st, sm):
        s, t = sm
        vals = self._ints(ctx, st) if st is not None else [0] * n
        return [(v * s + t) % p if st is not None else t % p for v in vals]
    xs, ys = side(x, x_map), side(y, y_map)
    return codec.ints_to_limbs([a if c else b for c, a, b in zip(m, xs, ys)], ctx)


METHODS = {'divide': divide, 'inverse': inverse, 'power': power, 'is_sqr': is_sqr, 'nonzero': nonzero, 'select': select}


def extend(backend_class):
    """Give the stand-in backend class the K11 methods."""
    for name, fn in METHODS.items():
        setattr(backend_class, name, fn)


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7 to K11 (undone with the monkeypatch fixture)."""
    import oracle_conv
    oracle_conv.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    for name, fn in METHODS.items():
        monkeypatch.setattr(resident.backend, name, fn.__get__(resident.backend), raising=False)
