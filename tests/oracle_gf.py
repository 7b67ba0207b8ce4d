"""TEST INFRASTRUCTURE: K15's device calls (resident.CudaBackend.gf_bits_compose / gf_binop_view / gf_matmul_batched)
answered on host byte arrays with a GF(2^8) product table built by the oracle's field arithmetic, for the CPU stand-in backend
of tests/oracle_device.py.  Without these methods the stand-in leaves GF(2^8) broadcasts, stacked products, bit compositions
and binary object-array operands to the reference's code; with them the hooks of mpyc_b200.resident run as they do on the
GPU.  Never imported by the package."""
import functools

import numpy as np

from oracle import shamir_oracle as orc
from mpyc_b200 import _cabi


@functools.lru_cache(maxsize=None)
def mul_table(poly):
    F = orc.field_of(poly, binary=True)
    return np.array([[F.red(F.mul(a, b)) for b in range(256)] for a in range(256)], dtype=np.uint8)


def gf_bits_compose(self, ctx, bits, n, l):
    T = mul_table(ctx.modulus)
    xj = [1]
    for _ in range(1, l):
        xj.append(int(T[xj[-1], 2]))
    x = np.asarray(bits, dtype=np.uint8).reshape(n, l)
    out = np.zeros(n, dtype=np.uint8)
    for j in range(l):
        out ^= T[x[:, j], xj[j]]
    return out


def gf_binop_view(self, ctx, op, a, a_view, b, b_view):
    from oracle_layout import positions
    x = np.asarray(a, dtype=np.uint8)[positions(a_view).reshape(-1)]
    y = np.asarray(b, dtype=np.uint8)[positions(b_view).reshape(-1)]
    return mul_table(ctx.modulus)[x, y] if op == _cabi.OP_MUL else x ^ y


def gf_matmul_batched(self, ctx, a, a_stacked, b, b_stacked, batch, r, k, c):
    T = mul_table(ctx.modulus)
    A = np.asarray(a, dtype=np.uint8).reshape(-1, r, k)
    B = np.asarray(b, dtype=np.uint8).reshape(-1, k, c)
    out = np.zeros((batch, r, c), dtype=np.uint8)
    for i in range(batch):
        Ai, Bi = A[i if a_stacked else 0], B[i if b_stacked else 0]
        for l in range(k):
            out[i] ^= T[Ai[:, l][:, None], Bi[l][None, :]]
    return out.reshape(-1)


METHODS = {'gf_bits_compose': gf_bits_compose, 'gf_binop_view': gf_binop_view, 'gf_matmul_batched': gf_matmul_batched}


def extend(backend_class):
    """Give the stand-in backend class the K15 methods."""
    for name, fn in METHODS.items():
        setattr(backend_class, name, fn)


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7 to K15 (undone with the monkeypatch fixture)."""
    import oracle_matmul_int
    oracle_matmul_int.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    for name, fn in METHODS.items():
        monkeypatch.setattr(resident.backend, name, fn.__get__(resident.backend), raising=False)
