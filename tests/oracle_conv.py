"""TEST INFRASTRUCTURE: K10's device call (resident.CudaBackend.convolve) answered on host limb arrays with Python ints,
straight from the definition full[k] = sum_{i + l = k} a[i] b[l] mod p, for the CPU stand-in backend of
tests/oracle_device.py.  Only the window [lo, lo + count) is formed, as the kernel does.  Never imported by the package."""
from mpyc_b200 import codec


def convolve_ints(a, b, lo, count, p):
    m, n = len(a), len(b)
    out = []
    for k in range(lo, lo + count):
        out.append(sum(a[i] * b[k - i] for i in range(max(0, k - n + 1), min(m - 1, k) + 1)) % p)
    return out


def convolve(self, ctx, a, m, b, n, lo, count):
    x, y = self._ints(ctx, a), self._ints(ctx, b)
    assert len(x) == m and len(y) == n and lo + count <= m + n - 1
    return codec.ints_to_limbs(convolve_ints(x, y, lo, count, ctx.modulus), ctx)


def extend(backend_class):
    """Give the stand-in backend class the K10 method."""
    backend_class.convolve = convolve


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7, K8, K9 and K10 (undone with the monkeypatch fixture)."""
    import oracle_linalg
    oracle_linalg.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    monkeypatch.setattr(resident.backend, 'convolve', convolve.__get__(resident.backend), raising=False)
