"""K9 (csrc/linalg.cuh) through the C ABI: the reference's determinants, solutions, inverses and matrix powers
(tests/golden/linalg.json) replayed on the device, both forms on both sides of the shared-memory tile limit, batched
determinants of (10^5, 4, 4) and (10^4, 16, 16) stacks, and algebraic properties at n = 1024 and 2048 checked through K1c."""
import hashlib
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import codec, device as dev         # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
import oracle_linalg                               # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden_linalg', os.path.join(HERE, 'golden', 'make_golden_linalg.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
P64, P128, P256 = 2**64 - 189, 2**128 - 173, 2**256 - 189

with open(os.path.join(HERE, 'golden', 'linalg.json')) as _fh:
    CASES = json.load(_fh)


def upload(ctx, rows):
    return DeviceArray.from_ints(ctx, [v for r in rows for v in r])


def ints(a):
    return [int(v) for v in a.to_ints()]


@pytest.mark.parametrize('i', range(len(CASES)))
def test_golden_replay(i):
    c = CASES[i]
    p, n = int(c['p'], 16), c['n']
    ctx = mpyc_b200.context_for(p)
    mats = [gold.matrix(p, n, k, c['seed'] + 100 * j) for j, k in enumerate(c['kinds'])]
    A = upload(ctx, [r for m in mats for r in m])
    try:
        if c['op'] == 'det':
            got = [str(v) for v in ints(dev.det(A, len(mats), n))]
        elif c['op'] == 'inv':
            got = gold.digest(ints(dev.inv(A, n)))
        elif c['op'] == 'solve':
            B = upload(ctx, gold.rhs(p, n, c['nrhs'], c['seed']))
            got = gold.digest(ints(dev.solve(A, B, n, c['nrhs'])))
        else:
            got = gold.digest(ints(dev.matrix_power(A, n, c['e'])))
    except ZeroDivisionError as e:
        assert str(e) == 'no inverse exists'
        got = 'ZeroDivisionError'
    assert got == c['result'], c


def tile_limit(L, inverse):
    """largest n whose det (n x n) or inverse (n x 2n and n + 1 row scales) tile fits the device's shared memory beside
    k_lin_tile's 32 bytes of static shared memory (inst_linalg.cu: tile_bytes, smem_limit)"""
    smem = torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 32

    def tile(n):
        return (n * 2 * n + n + 1 if inverse else n * n) * 8 * L
    n = 1
    while tile(n + 1) <= smem:
        n += 1
    return n


@pytest.mark.parametrize('p', [P64, P128, 2**255 - 19, P256])
def test_both_forms_at_the_tile_limit(p):
    ctx = mpyc_b200.context_for(p)
    for solve in (False, True):
        m = tile_limit(ctx.nlimbs, solve)
        for n in (m, m + 1):
            A = gold.matrix(p, n, 'perm' if n % 2 else 'rand', 21)
            flat = [v for r in A for v in r]
            d = upload(ctx, A)
            if solve:
                assert ints(dev.inv(d, n)) == oracle_linalg.solve_ints(flat, n, None, n, p), (p, n)
            else:
                assert ints(dev.det(d, 1, n)) == [oracle_linalg.det_ints(flat, n, p)], (p, n)


@pytest.mark.parametrize('p', [P64, 9409569905028393239, P256])
@pytest.mark.parametrize('batch, n', [(10**5, 4), (10**4, 16)])
def test_batched_det(p, batch, n):
    ctx = mpyc_b200.context_for(p)
    rng = np.random.default_rng(batch + n)
    A = DeviceArray.random(ctx, batch * n * n, seed=n)
    # every 7th matrix gets a zero first column, every 5th a zero top-left entry: singular ones and swaps in the stack
    t = A.t.view(batch, n, n, ctx.nlimbs)
    t[::7, :, 0] = 0
    t[1::5, 0, 0] = 0
    got = dev.det(A, batch, n).to_ints()
    host = A.to_ints()
    for b in sorted(set(rng.integers(0, batch, size=150).tolist()) | {0, 1, 6, batch - 1}):
        v = [int(x) for x in host[b * n * n:(b + 1) * n * n]]
        assert int(got[b]) == oracle_linalg.det_ints(v, n, p), b
    assert all(int(got[b]) == 0 for b in range(0, batch, 7))


def matmul(ctx, a, b, n):
    return dev.matmul(ctx, a, b, n, n, n)


@pytest.mark.parametrize('p, n', [(P64, 1024), (P256, 1024), (P128, 2048)])
def test_properties_at_scale(p, n):
    ctx = mpyc_b200.context_for(p)
    A = DeviceArray.random(ctx, n * n, seed=n + 1)
    B = DeviceArray.random(ctx, n * 3, seed=n + 2)
    X = dev.solve(A, B, n, 3)
    assert dev.matmul(ctx, A, X, n, n, 3).count_mismatch(B) == 0             # A @ solve(A, B) == B
    Ai = dev.inv(A, n)
    assert matmul(ctx, Ai, A, n).count_mismatch(dev.identity(ctx, n)) == 0  # inv(A) @ A == I
    C = DeviceArray.random(ctx, n * n, seed=n + 3)                         # random: no zero pivot, so no swap
    dA, dC, dAC = (int(dev.det(M, 1, n).to_ints()[0]) for M in (A, C, matmul(ctx, A, C, n)))
    assert dAC == dA * dC % p
    U = DeviceArray(ctx, torch.triu(A.t.view(n, n, ctx.nlimbs).permute(2, 0, 1)).permute(1, 2, 0).reshape(n * n, ctx.nlimbs)
                    .contiguous())
    diag = [int(v) for v in U.to_ints()[::n + 1]]
    want = 1
    for v in diag:
        want = want * v % p
    assert int(dev.det(U, 1, n).to_ints()[0]) == want                      # triangular: product of the diagonal
    L = DeviceArray(ctx, torch.tril(A.t.view(n, n, ctx.nlimbs).permute(2, 0, 1)).permute(1, 2, 0).reshape(n * n, ctx.nlimbs)
                    .contiguous())
    assert int(dev.det(L, 1, n).to_ints()[0]) == want


def test_singular_solve_raises_and_inputs_are_untouched():
    ctx = mpyc_b200.context_for(P128)
    for n in (5, 40, 300):
        A = gold.matrix(P128, n, 'dep', 3)
        d = upload(ctx, A)
        before = d.to_limbs().copy()
        with pytest.raises(ZeroDivisionError, match='no inverse exists'):
            dev.inv(d, n)
        assert int(dev.det(d, 1, n).to_ints()[0]) == 0
        assert np.array_equal(d.to_limbs(), before)
        torch.cuda.synchronize()


def test_digest_helper_is_the_fixtures():
    assert gold.digest([1, 2]) == hashlib.sha256(b'1,2').hexdigest()
