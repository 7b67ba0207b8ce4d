"""TEST INFRASTRUCTURE: K8's device calls (resident.CudaBackend.copy_view / binop_view) answered with NumPy on host limb
arrays, for the CPU stand-in backend of tests/oracle_device.py: copies by fancy indexing, arithmetic by NumPy object
arithmetic mod p.  Without these two methods the stand-in leaves views, joins and broadcasts to the reference's code;
with them the hooks of mpyc_b200.resident run as they do on the GPU.  Never imported by the package."""
import numpy as np

from mpyc_b200 import _cabi, codec


def positions(view):
    """Element numbers of a mpyc_b200.layout.View, shaped like the view (the NumPy interpreter of a descriptor)."""
    pos = np.full(view.shape, view.offset, dtype=np.int64)
    for k, (e, st) in enumerate(zip(view.shape, view.strides)):
        c = np.asarray(view.index, dtype=np.int64) if k == view.index_axis else np.arange(e, dtype=np.int64)
        pos = pos + (c * st).reshape((1,) * k + (e,) + (1,) * (len(view.shape) - k - 1))
    return pos


def copy_view(self, ctx, n, base, items):
    if base is not None:
        out = np.array(base, copy=True)
    else:
        out = np.zeros((n,) if ctx.binary else (n, ctx.nlimbs), dtype=np.uint8 if ctx.binary else np.uint64)
    for st, sv, dv in items:
        out[positions(dv).reshape(-1)] = np.asarray(st)[positions(sv).reshape(-1)]
    return out


def binop_view(self, ctx, op, a, a_view, b, b_view):
    x = np.array(self._ints(ctx, np.asarray(a)[positions(a_view).reshape(-1)]), dtype=object)
    y = np.array(self._ints(ctx, np.asarray(b)[positions(b_view).reshape(-1)]), dtype=object)
    r = (x + y) if op == _cabi.OP_ADD else ((x - y) if op == _cabi.OP_SUB else (x * y))
    return codec.ints_to_limbs(r % ctx.modulus, ctx)


def extend(backend_class):
    """Give the stand-in backend class the two K8 methods."""
    backend_class.copy_view = copy_view
    backend_class.binop_view = binop_view


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7 and K8 (undone with the monkeypatch fixture)."""
    import oracle_reduce
    oracle_reduce.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    monkeypatch.setattr(resident.backend, 'copy_view', copy_view.__get__(resident.backend), raising=False)
    monkeypatch.setattr(resident.backend, 'binop_view', binop_view.__get__(resident.backend), raising=False)
