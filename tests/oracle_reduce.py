"""TEST INFRASTRUCTURE: K7's device calls (resident.CudaBackend.sum_axis / cumsum_axis) answered by NumPy object
arithmetic mod p, for the CPU stand-in backend of tests/oracle_device.py.  Without these two methods the stand-in leaves
np.sum / np.cumsum / np.cumulative_sum to the reference's code; with them the hooks of mpyc_b200.resident run as they do
on the GPU.  Never imported by the package."""
import numpy as np

from mpyc_b200 import codec


def sum_axis(self, ctx, a, shape, axis, keepdims, initial):
    x = np.array(self._ints(ctx, a), dtype=object).reshape(shape)
    r = np.sum(x, axis=axis, keepdims=keepdims, initial=initial)
    return codec.ints_to_limbs(np.reshape(np.array(r, dtype=object) % ctx.modulus, -1), ctx)


def cumsum_axis(self, ctx, a, shape, axis, include_initial):
    x = np.array(self._ints(ctx, a), dtype=object).reshape(shape)
    if axis is None:
        x, axis = x.reshape(-1), 0
    r = np.cumulative_sum(x, axis=axis, include_initial=include_initial) % ctx.modulus
    return codec.ints_to_limbs(np.reshape(r, -1), ctx)


def extend(backend_class):
    """Give the stand-in backend class the two K7 methods."""
    backend_class.sum_axis = sum_axis
    backend_class.cumsum_axis = cumsum_axis


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7 (undone with the monkeypatch fixture)."""
    import oracle_device
    oracle_device.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    monkeypatch.setattr(resident.backend, 'sum_axis', sum_axis.__get__(resident.backend), raising=False)
    monkeypatch.setattr(resident.backend, 'cumsum_axis', cumsum_axis.__get__(resident.backend), raising=False)
