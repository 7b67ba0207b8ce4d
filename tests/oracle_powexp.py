"""TEST INFRASTRUCTURE: K12's device call (resident.CudaBackend.pow_exp) answered on host limb arrays with Python's pow,
straight from the definition out[h] = base(h)^e[h] mod p, for the CPU stand-in backend of tests/oracle_device.py.
Never imported by the package."""
import numpy as np

from mpyc_b200 import codec


def exponents(exps, signs, bits):
    """The Python ints that codec.exponents_to_limbs packed, checked against its bit length."""
    e = [sum(int(w) << (64 * i) for i, w in enumerate(row)) for row in np.asarray(exps, dtype=np.uint64)]
    assert all(v.bit_length() <= bits for v in e) and (not e or max(v.bit_length() for v in e) == bits)
    if signs is not None:
        e = [-v if s else v for v, s in zip(e, signs)]
    return e


def pow_exp(self, ctx, base, exps, signs, bits):
    p = ctx.modulus
    e = exponents(exps, signs, bits)
    if isinstance(base, int):
        assert 0 <= base < p
        if base == 0 and signs is not None:
            raise ZeroDivisionError('inverse of zero')
        return codec.ints_to_limbs([pow(base, v, p) for v in e], ctx)
    assert signs is None
    x = self._ints(ctx, base)
    assert len(x) == len(e)
    return codec.ints_to_limbs([pow(a, v, p) for a, v in zip(x, e)], ctx)


def extend(backend_class):
    """Give the stand-in backend class the K12 method."""
    backend_class.pow_exp = pow_exp


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7 to K12 (undone with the monkeypatch fixture)."""
    import oracle_divsel
    oracle_divsel.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    monkeypatch.setattr(resident.backend, 'pow_exp', pow_exp.__get__(resident.backend), raising=False)
