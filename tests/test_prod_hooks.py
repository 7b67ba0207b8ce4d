"""Products, running products and all / any behind install() on the reference's own finfields (K13 through
mpyc_b200.resident, answered here by the CPU stand-in of tests/oracle_prod.py): np.prod, FiniteFieldArray.prod, np.cumprod,
np.cumulative_prod, np.all and np.any reproduce tests/golden/prod.json -- the unmodified reference's values and result
types, and its exception type and message where it raises -- without turning limb-backed inputs into Python ints or
modifying them.  The calls left to the reference reach it with its own result or error; uninstall() restores prod; the
C-ABI entry points reject bad arguments without a GPU."""
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import pytest

from oracle import reference

REF = reference.path()
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden_prod', os.path.join(HERE, 'golden', 'make_golden_prod.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'prod.json')) as _fh:
    FIXTURES = json.load(_fh)


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


def encoded(fn):
    try:
        r = fn()
    except Exception as e:   # noqa: BLE001
        return {'error': [type(e).__name__, str(e)]}
    return gold.encode(r)


def want_of(c):
    return {k: v for k, v in c.items() if k not in ('p', 'case')}


def limb(F, ctx, vals, shape):
    from mpyc_b200 import resident, codec
    return F(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), shape), check=False)


def installed(monkeypatch, thresha, finfields, min_size=1):
    from mpyc_b200 import install as inst
    import oracle_device
    import oracle_prod
    oracle_device.patch(monkeypatch)
    oracle_prod.patch_resident(monkeypatch)
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=min_size)
    return inst


def test_fixture_inventory():
    assert len(FIXTURES) == 6 * len(gold.CASES) == 582
    assert sum('error' in c for c in FIXTURES) == 6 * 9
    kinds = {c.get('kind') for c in FIXTURES}
    assert kinds == {'array', 'element', 'bool', None}     # np.True_ / np.False_ report their type as 'bool' in NumPy 2


def test_hooks_reproduce_the_golden_fixtures(mpyc_mods, monkeypatch):
    """Limb-backed operands: every case without an error runs on K13 (one call), settles nothing, returns the reference's
    type and values and leaves its input's store intact; the errors are the reference's own."""
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for c in FIXTURES:
            p = int(c['p'], 16)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            d, fn = gold.CASES[c['case']]
            vals = gold.values(p, d)
            x = limb(F, ctx, vals, gold.SHAPES[d])
            keep = resident.raw_value(x)
            mat, k13 = resident.calls['materialised'], resident.calls['prod']
            try:
                r = fn(F, x)
            except Exception as e:   # noqa: BLE001
                r = e
            if 'error' in c:
                assert resident.calls['prod'] == k13, c['case']
                assert isinstance(r, Exception) and [type(r).__name__, str(r)] == c['error'], c['case']
                continue
            assert resident.calls['materialised'] == mat, c['case']
            assert resident.calls['prod'] == k13 + 1, c['case']
            if c['kind'] == 'bool':
                assert r is (np.True_ if c['bool'] else np.False_), c['case']
            elif c['kind'] == 'element':
                assert type(r) is F.field, c['case']
            else:
                assert type(r) is F and type(resident.raw_value(r)) is resident.LimbValue, c['case']
            assert gold.encode(r) == want_of(c), c['case']
            assert [int(v) for v in np.reshape(keep._materialise(), -1)] == vals, c['case']   # the input's store is intact
    finally:
        inst.uninstall()


def test_plain_object_arrays_match_the_fixtures(mpyc_mods, monkeypatch):
    """Object arrays of at least operators_min_size elements take the same hooks (the rule of np.sum)."""
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import resident
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for c in FIXTURES:
            if c['p'] not in (hex(gold.P64G), hex(gold.P256)):
                continue
            F = finfields.GF(int(c['p'], 16)).array
            d, fn = gold.CASES[c['case']]
            k13 = resident.calls['prod']
            assert encoded(lambda: fn(F, gold.operand(F, d))) == want_of(c), c['case']
            size = int(np.prod(gold.SHAPES[d]))
            assert resident.calls['prod'] == k13 + ('error' not in c and size >= 1), c['case']   # empty: below min_size
    finally:
        inst.uninstall()


def outcome(fn):
    try:
        r = fn()
    except Exception as e:   # noqa: BLE001
        return ('raises', type(e).__name__, str(e))
    if r is np.True_ or r is np.False_ or isinstance(r, (bool, np.ndarray)):
        return ('plain', type(r).__name__, np.asarray(r).tolist())
    v = r.value
    return (type(r).__name__, np.shape(v), [str(e) for e in np.reshape(np.asarray(v, dtype=object), -1)])


def test_calls_left_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    P = 2**127 - 1
    F = finfields.GF(P).array
    G = finfields.GF(gfpx.GFpX(2)(283)).array
    ctx = mpyc_b200.context_for(P)
    vals = [2, 3, 0, 5, 7, 1]
    table = [
        ('dtype', F, lambda x: np.prod(x, dtype=object)),
        ('out', F, lambda x: np.prod(x, axis=0, out=np.empty(2, dtype=object))),
        ('where', F, lambda x: np.prod(x, where=np.array([[True, False, True]] * 2))),
        ('all_where', F, lambda x: np.all(x, axis=0, where=np.array([[True, False, True]] * 2))),
        ('any_out', F, lambda x: np.any(x, axis=1, out=np.empty(2, dtype=bool))),
        ('cumprod_dtype', F, lambda x: np.cumprod(x, axis=0, dtype=object)),
        ('init_float', F, lambda x: np.prod(x, axis=0, initial=2.0)),
        ('init_bool', F, lambda x: np.prod(x, axis=0, initial=True)),
        ('init_np_int', F, lambda x: np.prod(x, axis=1, initial=np.int64(3))),
        ('init_element', F, lambda x: np.prod(x, initial=F.field(3))),
        ('meth_init_float', F, lambda x: x.prod(initial=2.5)),
        ('meth_init_other_field', F, lambda x: x.prod(axis=0, initial=finfields.GF(2**61 - 1)(3))),
        ('meth_init_positional', F, lambda x: x.prod(None, None, None, False, 3)),
        ('meth_where', F, lambda x: x.prod(where=np.array([[True, False, True]] * 2))),
        ('meth_dup', F, lambda x: x.prod(0, axis=1)),
        ('keepdims_int', F, lambda x: np.prod(x, axis=0, keepdims=1)),
        ('binary_prod', G, lambda x: np.prod(x, axis=0)),
        ('binary_all', G, lambda x: np.all(x)),
        ('binary_cumprod', G, lambda x: np.cumprod(x)),
        ('binary_meth', G, lambda x: x.prod(axis=1)),
    ]

    def make(cls, limbed):
        if limbed and cls is F:
            return limb(F, ctx, vals, (2, 3))
        return cls(np.array(vals, dtype=object).reshape(2, 3))
    want = [outcome(lambda: fn(make(cls, False))) for _, cls, fn in table]
    assert sum(w[0] == 'raises' for w in want) >= 3
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for (name, cls, fn), w in zip(table, want):
            k13 = resident.calls['prod']
            assert outcome(lambda: fn(make(cls, True))) == w, name
            assert resident.calls['prod'] == k13, name
    finally:
        inst.uninstall()


def test_min_size_and_a_backend_without_k13(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    P = 2**64 - 189
    F = finfields.GF(P).array
    ctx = mpyc_b200.context_for(P)
    inst = installed(monkeypatch, thresha, finfields, min_size=8)
    try:
        k13 = resident.calls['prod']
        small = F(np.array([2, 3, 4], dtype=object))
        assert int(np.prod(small)) == 24 and np.all(small) is np.True_
        assert resident.calls['prod'] == k13                                   # plain and below min_size
        assert int(np.prod(limb(F, ctx, [2, 3, 4], (3,)))) == 24              # limb-backed: any size
        assert resident.calls['prod'] == k13 + 1
    finally:
        inst.uninstall()
    import oracle_prod
    installed(monkeypatch, thresha, finfields)
    try:
        for name in oracle_prod.METHODS:
            monkeypatch.delattr(resident.backend, name)
        assert not resident._prod_backend()
        k13 = resident.calls['prod']
        x = limb(F, ctx, [2, 3, 0, 5], (2, 2))
        assert [int(v) for v in np.prod(x, axis=0).value] == [0, 15]
        assert np.any(x) is np.True_ and int(x.prod()) == 0
        assert [int(v) for v in np.cumprod(x, axis=1).value.reshape(-1)] == [2, 6, 0, 0]
        assert resident.calls['prod'] == k13
    finally:
        inst.uninstall()


def test_uninstall_restores_prod(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    cls = finfields.FiniteFieldArray
    orig_prod, orig_af = cls.__dict__['prod'], cls.__dict__['__array_function__']
    inst = installed(monkeypatch, thresha, finfields)
    assert cls.__dict__['prod'] is not orig_prod
    inst.uninstall()
    assert cls.__dict__['prod'] is orig_prod and cls.__dict__['__array_function__'] is orig_af


def test_k13_abi_argument_errors():
    """Null buffers, sizes that overflow, overlapping buffers and a non-canonical initial are rejected before any CUDA
    call; binary fields are unsupported; a valid call without a device fails with a CUDA error."""
    import mpyc_b200
    from mpyc_b200._cabi import lib, check, u64_array
    torch = pytest.importorskip('torch')
    p = 2**128 - 173
    ctx = mpyc_b200.context_for(p)                                    # 16-byte elements
    a, c = ctypes.c_void_p(1 << 30), ctypes.c_void_p(1 << 34)
    ok = u64_array([5, 0])
    bad = u64_array([p & (2**64 - 1), p >> 64])
    big = 1 << 62
    prod, cum, aa = lib.mpyc_b200_ff_prod_axis, lib.mpyc_b200_ff_cumprod_axis, lib.mpyc_b200_ff_all_any_axis
    calls = [lambda: prod(ctx.handle, a, 2, 3, 4, bad, c, None),                              # non-canonical initial
             lambda: prod(ctx.handle, None, 2, 3, 4, ok, c, None),
             lambda: prod(ctx.handle, a, 2, 3, 4, None, None, None),
             lambda: prod(ctx.handle, a, big, big, 4, None, c, None),                         # overflow
             lambda: prod(ctx.handle, a, 2, 3, 4, None, ctypes.c_void_p((1 << 30) + 8 * 16), None),   # overlap
             lambda: prod(ctx.handle, a, 2, 3, 4, None, ctypes.c_void_p((1 << 30) - 16), None),
             lambda: cum(ctx.handle, None, 2, 3, 4, 0, c, None),
             lambda: cum(ctx.handle, a, 2, 3, 4, 1, None, None),
             lambda: cum(ctx.handle, a, 2, 2**64 - 1, 4, 1, c, None),                         # len + 1 overflows
             lambda: cum(ctx.handle, a, 4, big, 4, 0, c, None),
             lambda: cum(ctx.handle, a, 2, 3, 4, 1, ctypes.c_void_p((1 << 30) + 16 * 23), None),
             lambda: aa(ctx.handle, None, 2, 3, 4, 0, c, None),
             lambda: aa(ctx.handle, a, 2, 3, 4, 1, None, None),
             lambda: aa(ctx.handle, a, big, 4, big, 1, c, None),
             lambda: aa(ctx.handle, a, 2, 3, 4, 0, ctypes.c_void_p((1 << 30) + 16), None)]
    for call in calls:
        with pytest.raises(ValueError):
            check(call())
    check(prod(ctx.handle, None, 0, 3, 4, None, None, None))                 # empty output: nothing to do
    check(cum(ctx.handle, None, 2, 0, 4, 0, None, None))
    check(aa(ctx.handle, None, 2, 3, 0, 1, None, None))
    g = mpyc_b200.context_for(283, binary=True)
    for call in (lambda: prod(g.handle, a, 2, 3, 4, None, c, None), lambda: cum(g.handle, a, 2, 3, 4, 0, c, None),
                 lambda: aa(g.handle, a, 2, 3, 4, 0, c, None)):
        with pytest.raises(mpyc_b200.UnsupportedFieldError):
            check(call())
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(prod(ctx.handle, a, 2, 3, 4, ok, c, None))
