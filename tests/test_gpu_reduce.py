"""K7 (csrc/reduce.cuh) through the C ABI against NumPy object arithmetic mod p: sums and running sums along the middle
axis of (O, R, I) arrays for every column / rows form, tile edge, split-R and three-phase shape, inputs that start on an
odd 8-byte boundary, and size-independent properties at 10^8 elements.  Bit-exact."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import device as dev                # noqa: E402
from mpyc_b200._cabi import lib, check             # noqa: E402
from mpyc_b200.device import DeviceArray, _stream_ptr   # noqa: E402

P61, P64, P64G, P128, P256 = 2**61 - 1, 2**64 - 189, 9409569905028393239, 2**128 - 173, 2**256 - 189
P160 = 0x80000004f1bbcdcbfa53e0af9ce60302e76e423f
PRIMES = [P61, P64, P64G, P128, P160, P256]


def ints(x):
    return [int(v) for v in x.to_ints()]


def shapes():
    """(O, R, I): both forms, R around the step of each form (8 rows per column; 8 steps of floor(32/I) rows per warp),
    R large enough to be split (columns: >= 128 rows; rows form: >= 2048 elements), O = 1 and 5"""
    out = []
    for I in (1, 2, 3, 7, 17, 31, 32, 33, 1000):
        tile = 8 if I >= 32 else 8 * (32 // I)
        split = 300 if I >= 32 else -(-5000 // I)
        for R in sorted({0, 1, 2, tile - 1, tile, tile + 1, split}):
            for O in (1, 5):
                if O * R * I <= 400_000:
                    out.append((O, R, I))
    return out


def offset_copy(a, odd):
    """a's elements in a buffer that starts one element (8 L bytes) into an allocation when odd"""
    if not odd:
        return a
    buf = DeviceArray.empty(a.ctx, a.n + 1)
    buf.t[1:].copy_(a.t)
    return DeviceArray(a.ctx, buf.t[1:])


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}_{p % 1000}')
def test_sum_and_cumsum_against_object_arithmetic(p):
    ctx = mpyc_b200.context_for(p)
    for j, (O, R, I) in enumerate(shapes()):
        n = O * R * I
        a = offset_copy(DeviceArray.random(ctx, n, seed=1000 * p.bit_length() + j), j % 2 == 1)
        x = np.array(ints(a), dtype=object).reshape(O, R, I)
        init = (p - 1 - j) % p
        out = DeviceArray.empty(ctx, O * I)
        check(lib.mpyc_b200_ff_sum_axis(ctx.handle, a.ptr, O, R, I, ctx.scalar_limbs(init), out.ptr, _stream_ptr()))
        assert ints(out) == ((x.sum(axis=1) + init) % p).reshape(-1).tolist(), (O, R, I)
        for inc in (0, 1):
            cs = DeviceArray.empty(ctx, O * (R + inc) * I)
            check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, a.ptr, O, R, I, inc, cs.ptr, _stream_ptr()))
            want = np.cumulative_sum(x, axis=1, include_initial=bool(inc)) % p
            assert ints(cs) == want.reshape(-1).tolist(), (O, R, I, inc)


def test_device_api_axes_and_multi_axis_plans():
    p = P128
    ctx = mpyc_b200.context_for(p)
    shape = (3, 5, 4, 7)
    a = DeviceArray.random(ctx, 3 * 5 * 4 * 7, seed=5)
    x = np.array(ints(a), dtype=object).reshape(shape)
    for axis in (None, 0, -1, (1, 2), (0, 2), (0, 1, 3), (), (3, 0)):
        for keepdims in (False, True):
            got, gshape = dev.sum_axis(a, shape, axis, keepdims, initial=-7)
            want = np.sum(x, axis=axis, keepdims=keepdims, initial=-7) % p
            assert gshape == np.shape(want) and ints(got) == np.reshape(want, -1).tolist(), (axis, keepdims)
    for axis in (None, 0, 1, -1):
        got, gshape = dev.cumsum_axis(a, shape, axis)
        want = np.cumsum(x, axis=axis) % p
        assert gshape == want.shape and ints(got) == want.reshape(-1).tolist()
    got, gshape = dev.cumsum_axis(a, shape, 2, include_initial=True)
    assert ints(got) == (np.cumulative_sum(x, axis=2, include_initial=True) % p).reshape(-1).tolist()


def fill(ctx, n, v):
    """n copies of the residue v"""
    a = DeviceArray.empty(ctx, n)
    for j in range(ctx.nlimbs):
        w = (v >> (64 * j)) & (2**64 - 1)
        a.t[:, j].fill_(w - 2**64 if w >= 2**63 else w)
    return a


def sum_dev(a, O, R, I, init=None):
    out = DeviceArray.empty(a.ctx, O * I)
    check(lib.mpyc_b200_ff_sum_axis(a.ctx.handle, a.ptr, O, R, I, init, out.ptr, _stream_ptr()))
    return out


def scan_dev(a, O, R, I, inc=0):
    out = DeviceArray.empty(a.ctx, O * (R + inc) * I)
    check(lib.mpyc_b200_ff_cumsum_axis(a.ctx.handle, a.ptr, O, R, I, inc, out.ptr, _stream_ptr()))
    return out


@pytest.mark.parametrize('p', [P64, P128, P256], ids=lambda p: f'p{p.bit_length()}')
def test_properties_at_1e8(p):
    ctx = mpyc_b200.context_for(p)
    n = 10**8 if p.bit_length() <= 128 else 4 * 10**7
    top = fill(ctx, n, p - 1)                                 # lazy accumulators at their bound
    for O, R, I in ((1, n, 1), (10, n // 10, 1), (1, n // 100, 100), (n // 100, 100, 1), (n // 3, 3, 1), (4, n // 40, 10)):
        assert set(ints(sum_dev(top, O, R, I))) == {(-R) % p}, (O, R, I)
    a, b = DeviceArray.random(ctx, n, seed=1), DeviceArray.random(ctx, n, seed=2)
    for O, R, I in ((1, n, 1), (100, n // 10000, 100)):
        assert ints(sum_dev(a + b, O, R, I)) == ints(sum_dev(a, O, R, I) + sum_dev(b, O, R, I))
    cs = scan_dev(a, 1, n, 1)
    assert ints(DeviceArray(ctx, cs.t[n - 1:])) == ints(sum_dev(a, 1, n, 1))
    assert (DeviceArray(ctx, cs.t[1:]) - DeviceArray(ctx, cs.t[:-1])).count_mismatch(DeviceArray(ctx, a.t[1:])) == 0
    del cs
    for O, R, I in ((10, n // 10, 1), (1, n // 1000, 1000), (1000, n // 1000, 1)):
        cs = scan_dev(a, O, R, I, inc=1)
        lastrows = cs.t.reshape(O, R + 1, I, ctx.nlimbs)[:, R].contiguous().reshape(O * I, ctx.nlimbs)
        assert ints(DeviceArray(ctx, lastrows)) == ints(sum_dev(a, O, R, I)), (O, R, I)
        rows = cs.t.reshape(O, R + 1, I, ctx.nlimbs)
        diff = DeviceArray(ctx, rows[:, 1:].reshape(-1, ctx.nlimbs).contiguous()) - \
            DeviceArray(ctx, rows[:, :-1].reshape(-1, ctx.nlimbs).contiguous())
        assert diff.count_mismatch(a) == 0, (O, R, I)
        del cs, rows, diff


def test_more_than_2_31_terms_at_one_limb():
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * 2**30:
        pytest.skip('needs 24 GiB of free device memory')
    p = P64
    ctx = mpyc_b200.context_for(p)
    R = 2**31 + 7
    top = fill(ctx, R, p - 1)
    assert ints(sum_dev(top, 1, R, 1, ctx.scalar_limbs(5))) == [(5 - R) % p]
    assert ints(sum_dev(top, 1, R // 7, 7)) == [(-(R // 7)) % p] * 7


def test_matmul_split_k_through_k7():
    """split-k matmul (few output tiles, long k): its slice sum is K7's columns form"""
    p = P128
    ctx = mpyc_b200.context_for(p)
    r, k, c = 1, 3136, 1024
    A, B = DeviceArray.random(ctx, r * k, seed=3), DeviceArray.random(ctx, k * c, seed=4)
    got = ints(dev.matmul(ctx, A, B, r, k, c))
    a = np.array(ints(A), dtype=object).reshape(r, k)
    bm = np.array(ints(B), dtype=object).reshape(k, c)
    assert got == ((a @ bm) % p).reshape(-1).tolist()
