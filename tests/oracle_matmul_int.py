"""TEST INFRASTRUCTURE: K14's device call (resident.CudaBackend.matmul_int) answered by NumPy object arithmetic mod p, for
the CPU stand-in backend of tests/oracle_device.py.  Without this method the stand-in leaves @ and np.matmul with integer
ndarrays to the reference's code; with it the hooks of mpyc_b200.resident run as they do on the GPU.  The integer operand
takes the device path's 64-bit form first (int64, or uint64 as is).  Never imported by the package."""
import numpy as np

from mpyc_b200 import codec


def matmul_int(self, ctx, x, w, r, k, c, w_left):
    w = np.asarray(w)
    w64 = np.ascontiguousarray(w) if w.dtype == np.uint64 else np.ascontiguousarray(w, dtype=np.int64)
    W = np.array([int(v) for v in w64.reshape(-1)], dtype=object)
    X = np.array(self._ints(ctx, x), dtype=object)
    if w_left:
        C = W.reshape(r, k) @ X.reshape(k, c) if k else np.zeros((r, c), dtype=object)
    else:
        C = X.reshape(r, k) @ W.reshape(k, c) if k else np.zeros((r, c), dtype=object)
    return codec.ints_to_limbs(np.reshape(C, -1) % ctx.modulus, ctx)


METHODS = {'matmul_int': matmul_int}


def extend(backend_class):
    """Give the stand-in backend class the K14 method."""
    for name, fn in METHODS.items():
        setattr(backend_class, name, fn)


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7 to K14 (undone with the monkeypatch fixture)."""
    import oracle_prod
    oracle_prod.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    for name, fn in METHODS.items():
        monkeypatch.setattr(resident.backend, name, fn.__get__(resident.backend), raising=False)
