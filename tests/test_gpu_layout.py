"""K8 (csrc/layout.cuh) through the C ABI: copies between strided views against NumPy indexing of the same host limb
arrays (exact: K8 only moves bytes) for every element size, form, tile edge, index table, odd 8-byte offsets, empty views
and offsets above 2^31; broadcast arithmetic against K1 on the materialised operands and against object arithmetic mod p;
transpose and flip applied twice at 10^8 elements."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import _cabi, device as dev, layout  # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from oracle_layout import positions                # noqa: E402

P61, P64, P64G, P128, P256 = 2**61 - 1, 2**64 - 189, 9409569905028393239, 2**128 - 173, 2**256 - 189
P160 = 0x80000004f1bbcdcbfa53e0af9ce60302e76e423f
PRIMES = [P61, P64, P64G, P128, P160, P256]
CTX = {1: lambda: mpyc_b200.context_for(283, binary=True), 8: lambda: mpyc_b200.context_for(P64),
       16: lambda: mpyc_b200.context_for(P128), 24: lambda: mpyc_b200.context_for(P160), 32: lambda: mpyc_b200.context_for(P256)}


def host_elements(ctx, n, seed):
    rng = np.random.default_rng(seed)
    if ctx.binary:
        return rng.integers(0, 256, size=n, dtype=np.uint8)
    return rng.integers(0, 2**63, size=(n, ctx.nlimbs), dtype=np.uint64)


def placed(ctx, host, odd):
    """host elements on the device, starting one element into an allocation when odd"""
    a = DeviceArray.from_limbs(ctx, host)
    if not odd:
        return a
    buf = DeviceArray.empty(ctx, a.n + 1)
    buf.t[1:].copy_(a.t)
    return DeviceArray(ctx, buf.t[1:])


def run_copy(ctx, shape, src_view, odd_src=False, odd_dst=False, seed=0):
    """copy_view(src_view -> C order) on the device vs NumPy, after collapsing like the hooks do"""
    n = int(np.prod(shape))
    host = host_elements(ctx, n, seed)
    src = placed(ctx, host, odd_src)
    m = src_view.size
    dst = placed(ctx, np.zeros((m,) + host.shape[1:], dtype=host.dtype), odd_dst)
    s, d = layout.collapse(src_view, layout.View.full(src_view.shape))
    dev.copy_view(src, s, dst, d)
    got = dst.to_limbs()
    want = host[positions(src_view).reshape(-1)]
    assert got.shape == want.shape and np.array_equal(got, want), (shape, src_view)


def key_views(shape):
    out = []
    nd = len(shape)
    keys = [(slice(None, None, 2),), (Ellipsis, slice(None, None, -1)), (Ellipsis, slice(1, None, 3)),
            (Ellipsis, [0, shape[-1] - 1, 1]), ([shape[0] - 1, 0],), (slice(1, None),) + (slice(None),) * (nd - 1)]
    for key in keys:
        plan = layout.getitem_plan(shape, key)
        if plan is not None:
            out.append(plan[0])
    if nd >= 2:
        out.append(layout.permuted(shape, tuple(reversed(range(nd)))))
        out.append(layout.permuted(shape, layout.swapaxes_axes(nd, 0, -1)))
    out.append(layout.flip_view(shape))
    return out


@pytest.mark.parametrize('E', [1, 8, 16, 24, 32])
def test_copy_forms_at_tile_edges(E):
    ctx = CTX[E]()
    shapes = [(31, 33), (32, 32), (33, 31), (3, 8192 // E - 1), (2, 8192 // E + 1), (5, 64, 33), (1, 1), (7,)]
    for shape in shapes:
        for view in key_views(shape):
            for odd in ((False, False), (True, False), (False, True), (True, True)) if E >= 8 else ((False, False),):
                run_copy(ctx, shape, view, *odd, seed=E)


@pytest.mark.parametrize('E', [1, 8, 16, 24, 32])
def test_copy_ranks_strides_and_tables(E):
    ctx = CTX[E]()
    rng = np.random.default_rng(E)
    for nd in range(1, 7):
        shape = tuple(int(v) for v in rng.integers(2, 6, size=nd))
        perm = tuple(int(v) for v in rng.permutation(nd))
        run_copy(ctx, shape, layout.permuted(shape, perm))
        run_copy(ctx, shape, layout.flip_view(shape, tuple(range(0, nd, 2))))
        for k in range(nd):                                  # an index table on every axis, the innermost included
            key = (slice(None),) * k + (list(rng.integers(0, shape[k], size=3)),)
            view = layout.getitem_plan(shape, key)[0]
            run_copy(ctx, shape, view)
        # zero strides (a broadcast source), as setitem writes a value into a selection
        _, vv, _ = layout.broadcast_views((shape[-1],), shape)
        run_copy(ctx, (shape[-1],), vv)


def test_copy_into_index_view_and_empty_views():
    ctx = CTX[16]()
    host = host_elements(ctx, 24, 1)
    src = DeviceArray.from_limbs(ctx, host[:8])
    base = DeviceArray.from_limbs(ctx, host)
    dview = layout.getitem_plan((4, 6), (slice(None), [5, 0]))[0]             # a write through (..., I)
    s, d = layout.collapse(layout.View.full((4, 2)), dview)
    dev.copy_view(src, s, base, d)
    want = host.copy()
    want[positions(dview).reshape(-1)] = host[:8]
    assert np.array_equal(base.to_limbs(), want)
    empty = layout.getitem_plan((4, 6), (slice(2, 2),))[0]
    dev.copy_view(src, empty, base, layout.View.full(empty.shape))
    assert np.array_equal(base.to_limbs(), want)


def test_copy_offsets_above_2_31():
    ctx = CTX[1]()
    n = 2**31 + 4096
    big = DeviceArray.empty(ctx, n)
    big.t[-4096:].copy_(torch.arange(4096, device='cuda', dtype=torch.int32).to(torch.uint8))
    out = DeviceArray.empty(ctx, 100)
    dev.copy_view(big, layout.View(n - 4000, (100,), (3,)), out, layout.View.full((100,)))
    tail = np.arange(4096).astype(np.uint8)
    assert np.array_equal(out.to_limbs(), tail[96 + 3 * np.arange(100)])
    dev.copy_view(big, layout.View(n - 1, (100,), (-1,)), out, layout.View.full((100,)))
    assert np.array_equal(out.to_limbs(), tail[4095 - np.arange(100)])


def test_copy_of_more_than_2_31_elements():
    """2^31 + 64 one-byte elements: the flip is the gather form with 64-bit item numbers, the plain copy the runs form"""
    ctx = CTX[1]()
    n = 2**31 + 64
    a = DeviceArray.empty(ctx, n)
    a.t.copy_(torch.arange(n, device='cuda', dtype=torch.int64).remainder_(251).to(torch.uint8))
    out = DeviceArray.empty(ctx, n)
    dev.copy_view(a, layout.flip_view((n,)), out, layout.View.full((n,)))
    assert torch.equal(out.t, torch.flip(a.t, (0,)))
    del out
    back = DeviceArray.empty(ctx, n)
    dev.copy_view(a, layout.View.full((n,)), back, layout.View.full((n,)))
    assert torch.equal(back.t, a.t)


def test_abi_rejects_bad_views_before_any_cuda_call():
    ctx = CTX[8]()
    a = DeviceArray.from_limbs(ctx, host_elements(ctx, 16, 0))
    b = DeviceArray.empty(ctx, 16)
    with pytest.raises(ValueError):                                            # outside the buffer
        dev.copy_view(a, layout.View(1, (16,), (1,)), b, layout.View.full((16,)))
    with pytest.raises(ValueError):                                            # overlap
        dev.copy_view(a, layout.View.full((8,)), DeviceArray(ctx, a.t[4:12]), layout.View.full((8,)))


def broadcast_cases():
    return [((64, 1), (64, 37)), ((5, 1, 1), (3, 5, 7, 9)), ((40, 33), (33,)), ((33,), (40, 33)), ((1,), (1000,)),
            ((3, 5, 7, 9), (5, 1, 1))]


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}_{p % 1000}')
def test_binop_view_matches_k1_and_object_arithmetic(p):
    ctx = mpyc_b200.context_for(p)
    rng = np.random.default_rng(p % 1000)
    for sa, sb in broadcast_cases():
        for op in (_cabi.OP_ADD, _cabi.OP_SUB, _cabi.OP_MUL):
            na, nb = int(np.prod(sa)), int(np.prod(sb))
            xa = [p - 1] + [(int(v) << 70 | int(v)) % p for v in rng.integers(0, 2**62, size=na - 1)]
            xb = [(int(v) * 7919 + p // 3) % p for v in rng.integers(0, 2**62, size=nb)]
            A, B = DeviceArray.from_ints(ctx, xa), DeviceArray.from_ints(ctx, xb)
            shape, va, vb = layout.broadcast_views(sa, sb)
            ca, cb = layout.collapse(va, vb)
            got = dev.binop_view(A, ca, B, cb, op)
            # K1 on the materialised operands
            n = int(np.prod(shape))
            Am, Bm = DeviceArray.empty(ctx, n), DeviceArray.empty(ctx, n)
            dev.copy_view(A, ca, Am, layout.View.full(ca.shape))
            dev.copy_view(B, cb, Bm, layout.View.full(cb.shape))
            assert got.to_ints().tolist() == Am._binop(Bm, op).to_ints().tolist()
            X = np.array(xa, dtype=object).reshape(sa)
            Y = np.array(xb, dtype=object).reshape(sb)
            want = {0: X + Y, 1: X - Y, 2: X * Y}[op] % p
            assert [int(v) for v in got.to_ints()] == [int(v) for v in want.reshape(-1)]


def test_transpose_and_flip_twice_are_the_identity_at_1e8():
    ctx = CTX[16]()
    R, C = 10_000, 10_000
    a = DeviceArray.random(ctx, R * C, seed=7)
    t = DeviceArray.empty(ctx, R * C)
    dev.copy_view(a, layout.permuted((R, C), (1, 0)), t, layout.View.full((C, R)))
    back = DeviceArray.empty(ctx, R * C)
    dev.copy_view(t, layout.permuted((C, R), (1, 0)), back, layout.View.full((R, C)))
    assert torch.equal(back.t, a.t)
    dev.copy_view(a, layout.flip_view((R * C,)), t, layout.View.full((R * C,)))
    dev.copy_view(t, layout.flip_view((R * C,)), back, layout.View.full((R * C,)))
    assert torch.equal(back.t, a.t) and torch.equal(t.t[:1], a.t[-1:])
