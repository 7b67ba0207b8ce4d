"""TEST INFRASTRUCTURE: K9's device calls (resident.CudaBackend.det / solve / matrix_power) answered on host limb arrays
by a Python restatement of csrc/linalg.cuh's algorithm, for the CPU stand-in backend of tests/oracle_device.py: the
division-free elimination with the reference's pivot rule, the determinant P_{n-1} / (P_0 ... P_{n-2}) and the Gauss-Jordan
solve with row scales P_{i-1} / P_{n-1}.  Compared with the uninstalled reference, it checks the algorithm as well as the
hooks.  Never imported by the package."""
import numpy as np

from mpyc_b200 import codec


def eliminate(M, n, W, p, jordan):
    """Division-free elimination of the n x W list-of-rows M in place: the pivots p_0 .. p_{n-1}, or None when a column
    has no pivot (singular)."""
    piv = []
    for k in range(n):
        x = next((i for i in range(k, n) if M[i][k]), None)
        if x is None:
            return None
        M[k], M[x] = M[x], M[k]
        pk = M[k][k]
        for i in (range(n) if jordan else range(k + 1, n)):
            if i == k:
                continue
            aik = M[i][k]
            M[i] = M[i][:k + 1] + [(pk * M[i][j] - aik * M[k][j]) % p for j in range(k + 1, W)]
        piv.append(pk)
    return piv


def det_ints(vals, n, p):
    M = [list(vals[i * n:(i + 1) * n]) for i in range(n)]
    piv = eliminate(M, n, n, p, False)
    if piv is None:
        return 0
    P, Q = 1, 1
    for k, pk in enumerate(piv):
        P = P * pk % p
        if k < n - 1:
            Q = Q * P % p
    return P * pow(Q, -1, p) % p


def solve_ints(vals, n, rhs, nrhs, p):
    """X (n * nrhs values) = A^-1 B; rhs None: the identity.  ZeroDivisionError for a singular A."""
    W = n + nrhs
    M = [list(vals[i * n:(i + 1) * n]) + ([int(j == i) for j in range(n)] if rhs is None else list(rhs[i * nrhs:(i + 1) * nrhs]))
         for i in range(n)]
    piv = eliminate(M, n, W, p, True)
    if piv is None:
        raise ZeroDivisionError('no inverse exists')
    scale, P = [], 1
    for pk in piv:
        scale.append(P)
        P = P * pk % p
    inv = pow(P, -1, p)
    return [M[i][n + j] * scale[i] * inv % p for i in range(n) for j in range(nrhs)]


def det(self, ctx, a, batch, n):
    v = self._ints(ctx, a)
    return codec.ints_to_limbs([det_ints(v[b * n * n:(b + 1) * n * n], n, ctx.modulus) for b in range(batch)], ctx)


def solve(self, ctx, a, n, b, nrhs):
    return codec.ints_to_limbs(solve_ints(self._ints(ctx, a), n, None if b is None else self._ints(ctx, b), nrhs, ctx.modulus), ctx)


def matrix_power(self, ctx, a, n, e):
    p = ctx.modulus
    A = np.array(self._ints(ctx, a), dtype=object).reshape(n, n)
    if e < 0:
        A, e = np.array(solve_ints(A.reshape(-1).tolist(), n, None, n, p), dtype=object).reshape(n, n), -e
    C = np.eye(n, dtype=object)
    while e:
        if e & 1:
            C = (C @ A) % p
        A = (A @ A) % p
        e >>= 1
    return codec.ints_to_limbs(C.reshape(-1), ctx)


def extend(backend_class):
    """Give the stand-in backend class the K9 methods."""
    backend_class.det = det
    backend_class.solve = solve
    backend_class.matrix_power = matrix_power


def patch_resident(monkeypatch):
    """resident.backend = the oracle stand-in with K7, K8 and K9 (undone with the monkeypatch fixture)."""
    import oracle_layout
    oracle_layout.patch_resident(monkeypatch)
    from mpyc_b200 import resident
    for name, fn in (('det', det), ('solve', solve), ('matrix_power', matrix_power)):
        monkeypatch.setattr(resident.backend, name, fn.__get__(resident.backend), raising=False)
