"""TEST INFRASTRUCTURE: K13's device calls (resident.CudaBackend.prod_axis / cumprod_axis / all_any_axis) answered by NumPy
object arithmetic mod p, for the CPU stand-in backend of tests/oracle_device.py.  Without these methods the stand-in
leaves np.prod / np.cumprod / np.cumulative_prod / np.all / np.any to the reference's code; with them the hooks of
mpyc_b200.resident run as they do on the GPU.  Never imported by the package."""
import numpy as np

from mpyc_b200 import codec


def _mulmod(p):
    return np.frompyfunc(lambda a, b: a * b % p, 2, 1)


def prod_axis(self, ctx, a, shape, axis, keepdims, initial):
    x = np.array(self._ints(ctx, a), dtype=object).reshape(shape)
    r = np.prod(x, axis=axis, keepdims=keepdims, initial=initial)                 # exact products, then mod p
    return codec.ints_to_limbs(np.reshape(np.array(r, dtype=object) % ctx.modulus, -1), ctx)


def cumprod_axis(self, ctx, a, shape, axis, include_initial):
    x = np.array(self._ints(ctx, a), dtype=object).reshape(shape)
    if axis is None:
        x, axis = x.reshape(-1), 0
    r = _mulmod(ctx.modulus).accumulate(x, axis=axis, dtype=object) if x.shape[axis] else x.copy()
    if include_initial:
        ones = np.ones(x.shape[:axis % x.ndim] + (1,) + x.shape[axis % x.ndim + 1:], dtype=object)
        r = np.concatenate([ones, r], axis=axis)
    return codec.ints_to_limbs(np.reshape(r, -1), ctx)


def all_any_axis(self, ctx, a, shape, axis, keepdims, any):
    x = np.array(self._ints(ctx, a), dtype=object).reshape(shape) != 0
    r = (np.any if any else np.all)(x, axis=axis, keepdims=keepdims)
    return codec.ints_to_limbs([int(v) for v in np.reshape(r, -1)], ctx)


METHODS = {'prod_axis': prod_axis, 'cumprod_axis': cumprod_axis, 'all_any_axis': all_any_axis}


def extend(backend_class):
    """Give the stand-in backend class the K13 methods."""
    for name, fn in METHODS.items():
        setattr(backend_class, name, fn)


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7 to K13 (undone with the monkeypatch fixture)."""
    import oracle_powexp
    oracle_powexp.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    for name, fn in METHODS.items():
        monkeypatch.setattr(resident.backend, name, fn.__get__(resident.backend), raising=False)
