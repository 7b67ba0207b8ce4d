"""Views, writes, axis permutations, joins, flips, rolls and broadcast arithmetic behind install(operators=True) on the
reference's own finfields (K8 through mpyc_b200.resident, answered here by the CPU stand-in of tests/oracle_layout.py):
every result equals the uninstalled reference's in kind, shape and value, limb-backed inputs are never turned into Python
ints, uncovered calls reach the reference, and a backend without K8 leaves everything to the reference.  Also the argument
errors of the two K8 C-ABI entry points, which need no GPU."""
import ctypes
import sys

import numpy as np
import pytest

from oracle import reference
from test_reduce_hooks import call, outcome

REF = reference.path()
PRIMES = [2**64 - 189, 2**128 - 173, 0x80000004f1bbcdcbfa53e0af9ce60302e76e423f, 2**256 - 189]


@pytest.fixture(scope='module')
def mpyc_mods():
    if REF is None:
        pytest.skip('reference not present ($MPYC_REFERENCE, or the copy build() makes in oracle/_ref)')
    sys.dont_write_bytecode = True
    sys.path.insert(0, REF)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import thresha, finfields, gfpx
    finally:
        sys.argv = argv
    yield thresha, finfields, gfpx
    sys.path.remove(REF)


def cases(binary):
    """(name, covered, shape(s), fn(*arrays)) -- covered: the hooks must take the call"""
    I = np.array([2, 0, 3])
    out = [
        ('step', True, [(4, 5)], lambda a: a[:, ::2]), ('neg_step', True, [(4, 5)], lambda a: a[::-1]),
        ('none', True, [(4, 5)], lambda a: a[None, 1:3, None]), ('index_last', True, [(4, 5)], lambda a: a[..., I]),
        ('index_first', True, [(4, 5)], lambda a: a[[3, 1]]), ('index_mixed', True, [(2, 4, 5)], lambda a: a[1, :, [0, 4]]),
        ('element', True, [(4, 5)], lambda a: a[2, -1]), ('element_1d', True, [(5,)], lambda a: a[3]),
        ('zero_d_array', True, [(4, 5)], lambda a: a[2, 3, ...]), ('empty', True, [(4, 5)], lambda a: a[2:2]),
        ('rows', True, [(4, 5)], lambda a: a[1:3]), ('slice_col', True, [(4, 5)], lambda a: a[:, 1:2]),
        ('T', True, [(4, 5)], lambda a: a.T), ('transpose', True, [(2, 3, 4)], lambda a: a.transpose(2, 0, 1)),
        ('transpose_t', True, [(2, 3, 4)], lambda a: a.transpose((1, 0, 2))), ('swapaxes', True, [(2, 3, 4)], lambda a: a.swapaxes(0, 2)),
        ('np_transpose', True, [(2, 3, 4)], lambda a: np.transpose(a, axes=(1, 2, 0))),
        ('np_swapaxes', True, [(2, 3, 4)], lambda a: np.swapaxes(a, 1, -1)), ('moveaxis', True, [(2, 3, 4)], lambda a: np.moveaxis(a, 0, -1)),
        ('concat1', True, [(2, 3), (2, 4)], lambda a, b: np.concatenate((a, b), axis=1)),
        ('concat_neg', True, [(2, 3), (2, 1)], lambda a, b: np.concatenate([a, b], axis=-1)),
        ('concat_none', True, [(2, 3), (4,)], lambda a, b: np.concatenate((a, b), axis=None)),
        ('concat0', True, [(2, 3), (1, 3)], lambda a, b: np.concatenate((a, b))),
        ('stack1', True, [(2, 3), (2, 3)], lambda a, b: np.stack((a, b), axis=1)),
        ('vstack', True, [(3,), (2, 3)], lambda a, b: np.vstack((a, b))), ('hstack', True, [(2, 3), (2, 2)], lambda a, b: np.hstack((a, b))),
        ('flip', True, [(3, 4)], lambda a: np.flip(a)), ('flip1', True, [(3, 4)], lambda a: np.flip(a, 1)),
        ('roll', True, [(3, 4)], lambda a: np.roll(a, 1, axis=1)), ('roll_none', True, [(3, 4)], lambda a: np.roll(a, -5)),
        ('expand', True, [(3, 4)], lambda a: np.expand_dims(a, 1)), ('squeeze', True, [(3, 1, 4)], lambda a: np.squeeze(a)),
        # left to the reference
        ('mask', False, [(4, 5)], lambda a: a[np.ones((4, 5), dtype=bool)]), ('two_arrays', False, [(4, 5)], lambda a: a[[0, 1], [1, 2]]),
        ('bad_index', False, [(4, 5)], lambda a: a[9]), ('bad_axes', False, [(2, 3)], lambda a: a.transpose(0, 0)),
        ('roll_tuple', False, [(3, 4)], lambda a: np.roll(a, (1, 2), axis=(0, 1))),
        ('concat_bad', False, [(2, 3), (3, 4)], lambda a, b: np.concatenate((a, b), axis=1)),
        ('stack_pub', False, [(2, 3)], lambda a: np.stack((a, np.ones((2, 3), dtype=object)))),
    ]
    if not binary:
        out += [('bc_col', True, [(4, 1), (4, 5)], lambda a, b: a * b), ('bc_4d', True, [(3, 1, 1), (2, 3, 4, 5)], lambda a, b: a + b),
                ('bc_rows', True, [(4, 5), (5,)], lambda a, b: a - b), ('bc_rows_r', True, [(5,), (4, 5)], lambda a, b: a - b),
                ('bc_one', True, [(1,), (6,)], lambda a, b: a * b), ('bc_bad', False, [(4, 5), (4,)], lambda a, b: a + b)]
    return out


def run_cases(F, ctx, binary):
    from mpyc_b200 import resident, codec
    p = F.field.modulus

    def values(shape, salt):
        n = int(np.prod(shape, dtype=object))
        if binary:
            return [(37 * i + salt) % 256 for i in range(n)]
        return [(7 * i * i + 3 * i + salt + (p - 1 if i % 3 == 0 else 0)) % p for i in range(n)]

    def plain(shape, salt):
        return F(np.array(values(shape, salt), dtype=object).reshape(shape))

    def limb(shape, salt):
        return F(resident.LimbValue(ctx, codec.ints_to_limbs(values(shape, salt), ctx), shape,
                                    type(F.field.modulus) if binary else None), check=False)

    table = cases(binary)
    want = [outcome(call(lambda: fn(*[plain(s, 5 * j) for j, s in enumerate(shapes)]))) for _, _, shapes, fn in table]
    return table, want, plain, limb


@pytest.mark.parametrize('field', ['p64', 'p128', 'p160', 'p256', 'gf256'])
def test_layout_hooks_equal_the_reference(mpyc_mods, monkeypatch, field):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_layout
    oracle_device.patch(monkeypatch)
    oracle_layout.patch_resident(monkeypatch)
    binary = field == 'gf256'
    if binary:
        G = finfields.GF(gfpx.GFpX(2)(283))
        ctx = mpyc_b200.context_for(283, binary=True)
    else:
        P = PRIMES[['p64', 'p128', 'p160', 'p256'].index(field)]
        G = finfields.GF(P)
        ctx = mpyc_b200.context_for(P)
    F = G.array
    table, want, plain, limb = run_cases(F, ctx, binary)
    assert sum(w[0] == 'raises' for w in want) >= 3
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for (name, covered, shapes, fn), w in zip(table, want):
            args = [limb(s, 5 * j) for j, s in enumerate(shapes)]
            mat, ops = resident.calls['materialised'], resident.calls['limb_ops']
            r = call(lambda: fn(*args))
            if covered:                      # on the limbs: a K8 call, or a result sharing the input's store
                assert resident.calls['materialised'] == mat, name
                shared = isinstance(r, F) and resident.as_limb_value(resident.raw_value(r)) is not None
                assert resident.calls['limb_ops'] > ops or (shared and name in ('rows', 'slice_col', 'none', 'zero_d_array', 'empty', 'expand', 'squeeze')), name
            else:                            # the reference's code: it reads .value, which settles the limb-backed input
                assert resident.calls['limb_ops'] == ops and resident.calls['materialised'] > mat, name
            assert outcome(r) == w, (name, outcome(r), w)
            # plain arrays alone
            assert outcome(call(lambda: fn(*[plain(s, 5 * j) for j, s in enumerate(shapes)]))) == w, name
            if len(shapes) == 2 and covered and not binary and name.startswith(('concat', 'stack', 'vstack', 'hstack')):
                # a join of a limb-backed and a plain piece: the plain one is packed
                packed, ops = resident.calls['packed'], resident.calls['limb_ops']
                r = call(lambda: fn(limb(shapes[0], 0), plain(shapes[1], 5)))
                assert resident.calls['packed'] == packed + 1 and resident.calls['limb_ops'] > ops, name
                assert outcome(r) == w, name
    finally:
        inst.uninstall()


@pytest.mark.parametrize('field', ['p128', 'gf256'])
def test_setitem_equals_the_reference(mpyc_mods, monkeypatch, field):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_layout
    oracle_device.patch(monkeypatch)
    oracle_layout.patch_resident(monkeypatch)
    binary = field == 'gf256'
    G = finfields.GF(gfpx.GFpX(2)(283)) if binary else finfields.GF(2**128 - 173)
    ctx = mpyc_b200.context_for(283, binary=True) if binary else mpyc_b200.context_for(2**128 - 173)
    F = G.array
    p = 256 if binary else G.modulus
    vals = [(11 * i + 3) % p for i in range(20)]
    poly = type(G.modulus) if binary else None

    def limb(v, shape):
        return F(resident.LimbValue(ctx, codec.ints_to_limbs(v, ctx), shape, poly), check=False)

    def plain(v, shape):
        return F(np.array(v, dtype=object).reshape(shape))
    writes = [((slice(None), 1), lambda mk: mk([7, 8, 9, 10], (4,)), True), ((slice(1, 3),), lambda mk: mk([1, 2, 3, 4, 5], (5,)), True),
              ((Ellipsis, [4, 0]), lambda mk: mk([5, 6], (2,)), True), ((slice(None, None, 2), [1, 3]), lambda mk: 3, True),
              ((2, slice(None, None, -1)), lambda mk: G(5), not binary), ((Ellipsis, [1, 1]), lambda mk: mk([5, 6], (2,)), False),
              ((slice(None), 1), lambda mk: mk([1, 2, 3], (3,)), False), ((np.ones((4, 5), dtype=bool),), lambda mk: 1, False)]
    want = []
    for key, val, _ in writes:
        a = plain(vals, (4, 5))
        b = a.copy()
        r = call(lambda: a.__setitem__(key, val(plain)))
        want.append((outcome(r) if isinstance(r, tuple) else None, outcome(a), outcome(b)))
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for (key, val, covered), w in zip(writes, want):
            a = limb(vals, (4, 5))
            shared = a[:]                                              # shares a's store: must not change
            v = val(limb)
            mat, ops = resident.calls['materialised'], resident.calls['limb_ops']
            r = call(lambda: a.__setitem__(key, v))
            if covered:
                assert resident.calls['materialised'] == mat and resident.calls['limb_ops'] > ops, key
            assert (outcome(r) if isinstance(r, tuple) else None, outcome(a), outcome(shared)) == w, key
    finally:
        inst.uninstall()


def test_a_backend_without_k8_leaves_layout_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_reduce
    oracle_device.patch(monkeypatch)
    oracle_reduce.patch_resident(monkeypatch)                           # K7 but no K8
    P = 2**128 - 173
    F = finfields.GF(P).array
    ctx = mpyc_b200.context_for(P)
    vals = [(3 * i + 1) % P for i in range(12)]
    calls = [lambda a: a[:, ::2], lambda a: a.T, lambda a: np.flip(a), lambda a: np.concatenate((a, a), axis=1),
             lambda a: a * F(np.array(vals[:3], dtype=object).reshape(3, 1)), lambda a: a[1, 2]]
    want = [outcome(call(lambda: fn(F(np.array(vals, dtype=object).reshape(3, 4))))) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for fn, w in zip(calls, want):
            a = F(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), (3, 4)), check=False)
            ops = resident.calls['limb_ops']
            r = call(lambda: fn(a))
            assert resident.calls['limb_ops'] == ops
            assert outcome(r) == w
    finally:
        inst.uninstall()


def test_k8_abi_argument_errors():
    """Bad views are rejected before any CUDA call; valid ones without a device fail with a CUDA error."""
    import mpyc_b200
    from mpyc_b200 import _cabi
    from mpyc_b200._cabi import lib, check
    torch = pytest.importorskip('torch')
    ctx = mpyc_b200.context_for(2**64 - 189)

    def view(offset, shape, strides, index=None, axis=-1):
        v = _cabi.View()
        v.offset, v.rank, v.index_axis = offset, len(shape), axis
        for k, (e, s) in enumerate(zip(shape, strides)):
            v.extent[k], v.stride[k] = e, s
        if index is not None:
            v.index = index.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
        return v
    a, b = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 30)           # never dereferenced: every call below fails first
    ok = view(0, (4, 4), (4, 1))

    def copy(src, dst, n=16, E=8, pa=a, pb=b):
        return lib.mpyc_b200_copy_view(E, pa, n, ctypes.byref(src), pb, n, ctypes.byref(dst), None)
    seven = view(0, (1,) * 6, (1,) * 6)
    seven.rank = 7
    idx = np.array([0, 5], dtype=np.int64)
    for bad in [lambda: copy(seven, seven), lambda: copy(view(0, (4, -1), (4, 1)), view(0, (4, -1), (4, 1))),
                lambda: copy(view(1, (4, 4), (4, 1)), ok), lambda: copy(view(3, (4,), (-1,)), view(0, (4,), (1,)), n=3),
                lambda: copy(view(0, (2, 2), (4, 1), idx, 0), view(0, (2, 2), (2, 1))),
                lambda: copy(ok, ok, pb=ctypes.c_void_p((1 << 20) + 64)), lambda: copy(ok, view(0, (2, 8), (8, 1))),
                lambda: copy(ok, ok, E=12)]:
        with pytest.raises(ValueError):
            check(bad())
    check(copy(view(0, (0, 4), (4, 1)), view(0, (0, 4), (4, 1))))                   # empty: nothing to do
    v3 = view(0, (4,), (0,))
    with pytest.raises(ValueError):                                                  # index tables are not taken here
        check(lib.mpyc_b200_ff_binop_view(ctx.handle, 0, a, 16, ctypes.byref(view(0, (2,), (1,), idx, 0)), b, 16,
                                          ctypes.byref(v3), b, None))
    with pytest.raises(ValueError):                                                  # out overlaps b
        check(lib.mpyc_b200_ff_binop_view(ctx.handle, 0, a, 16, ctypes.byref(v3), b, 16, ctypes.byref(v3), b, None))
    with pytest.raises(ValueError):
        check(lib.mpyc_b200_ff_binop_view(ctx.handle, 3, a, 16, ctypes.byref(v3), b, 16, ctypes.byref(v3), b, None))
    g = mpyc_b200.context_for(283, binary=True)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(lib.mpyc_b200_ff_binop_view(g.handle, 0, a, 16, ctypes.byref(v3), b, 16, ctypes.byref(v3), None, None))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(copy(ok, view(0, (4, 4), (1, 4))))
