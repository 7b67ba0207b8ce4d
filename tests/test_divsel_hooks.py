"""Division, powers, square roots, is_sqr and np.where behind install(operators=True) on the reference's own finfields (K11
and K1b through mpyc_b200.resident, answered here by the CPU stand-in of tests/oracle_divsel.py): every hooked form
reproduces tests/golden/divsel.json -- the unmodified reference's values, and its exception type and message for zero
divisors -- without turning limb-backed inputs into Python ints or modifying them; `/=` leaves arrays that share the old
store unchanged; the calls left to the reference reach it with its own result or error; a backend without K11 leaves
everything to the reference.  Also ModValue's `== 0`, np.count_nonzero and np.where against NumPy object arithmetic, and the
argument errors of the K11 C-ABI entry points, which need no GPU."""
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
_spec = importlib.util.spec_from_file_location('make_golden_divsel', os.path.join(HERE, 'golden', 'make_golden_divsel.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'divsel.json')) as _fh:
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


def outcome(fn):
    """('bool', values) / ('array', class, shape, values) / ('element', value) / ('raises', type, message)"""
    try:
        r = fn()
    except Exception as e:   # noqa: BLE001
        return ('raises', type(e).__name__, str(e))
    if isinstance(r, np.ndarray):
        return ('ndarray', r.dtype.kind, r.shape, r.tolist())
    if hasattr(r, 'field') and hasattr(r, 'shape'):
        return ('array', type(r).__name__, r.shape, [int(v) for v in np.asarray(r.value, dtype=object).reshape(-1)])
    return ('other', repr(r))


def encoded(fn):
    try:
        r = fn()
    except Exception as e:   # noqa: BLE001
        return {'error': [type(e).__name__, str(e)]}
    return gold.encode(r)


def limb(F, ctx, vals, shape=None):
    from mpyc_b200 import resident, codec
    return F(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), shape or (len(vals),)), check=False)


def test_hooks_reproduce_the_golden_fixtures(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_divsel
    oracle_device.patch(monkeypatch)
    oracle_divsel.patch_resident(monkeypatch)
    assert len(FIXTURES) > 300 and sum('error' in c for c in FIXTURES) > 70
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for c in FIXTURES:
            p = int(c['p'], 16)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            names, fn = gold.CASES[c['case']]
            ops = [limb(F, ctx, gold.operand(p, k)) for k in names]
            keep = [resident.raw_value(x) for x in ops]
            mat, lops = resident.calls['materialised'], resident.calls['limb_ops']
            res = [None]

            def run():
                res[0] = fn(F, *ops)
                return res[0]
            try:
                run()
            except Exception:   # noqa: BLE001
                pass
            assert resident.calls['materialised'] == mat, c['case']
            if 'error' not in c:
                assert resident.calls['limb_ops'] > lops, c['case']
                assert isinstance(res[0], np.ndarray) or type(resident.raw_value(res[0])) is resident.LimbValue, c['case']
            got = encoded(lambda: res[0] if 'error' not in c else fn(F, *ops))
            want = {k: v for k, v in c.items() if k in ('hex', 'bool', 'error')}
            assert got == want, c['case']
            for k, v in zip(names, keep):       # inputs, and arrays sharing their stores, keep their values
                assert [int(e) for e in v._materialise().reshape(-1)] == gold.operand(p, k), c['case']
    finally:
        inst.uninstall()


def test_plain_object_arrays_are_packed_and_give_the_fixtures(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_divsel
    oracle_device.patch(monkeypatch)
    oracle_divsel.patch_resident(monkeypatch)
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for c in FIXTURES[:120]:
            p = int(c['p'], 16)
            F = finfields.GF(p).array
            names, fn = gold.CASES[c['case']]
            ops = [F(np.array(gold.operand(p, k), dtype=object)) for k in names]
            assert encoded(lambda: fn(F, *ops)) == {k: v for k, v in c.items() if k in ('hex', 'bool', 'error')}, c['case']
    finally:
        inst.uninstall()


def test_in_place_division_leaves_sharers_unchanged(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_divsel
    oracle_device.patch(monkeypatch)
    oracle_divsel.patch_resident(monkeypatch)
    p = 2**127 - 1
    F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        a = limb(F, ctx, [3, 4, 5, 6])
        view = a.reshape(2, 2)                     # shares a's store
        b = limb(F, ctx, [2, 2, 5, 3])
        a /= b
        assert [int(v) for v in a.value] == [3 * pow(2, -1, p) % p, 2, 1, 2]
        assert [int(v) for v in view.value.reshape(-1)] == [3, 4, 5, 6]
        c = limb(F, ctx, [2, 3])
        alias = c.copy()
        c **= -1
        assert [int(v) for v in c.value] == [pow(2, -1, p), pow(3, -1, p)]
        assert [int(v) for v in alias.value] == [2, 3]
    finally:
        inst.uninstall()


def reference_cases(F, G, H):
    """Calls the hooks leave to the reference (name, fn(make) -> result); make(vals, shape=None, cls=F) builds an operand"""
    return [('broadcast_div', lambda m: m([1, 2, 3, 4, 5, 6], (2, 3)) / m([1, 2, 3])),
            ('broadcast_where', lambda m: np.where(np.array([True, False, True]), m([1, 2, 3, 4, 5, 6], (2, 3)), m([7, 8, 9]))),
            ('where_one_arg', lambda m: np.where(m([0, 1, 2]))),
            ('where_keywords', lambda m: np.where(np.array([True, False]), x=m([1, 2]), y=m([3, 4]))),
            ('where_other_field', lambda m: np.where(np.array([True, False]), m([1, 2]), m([3, 4], cls=H))),
            ('where_float', lambda m: np.where(np.array([True, False]), m([1, 2]), 1.5)),
            ('where_bad_mask_shape', lambda m: np.where(np.array([True, False, True]), m([1, 2]), m([3, 4]))),
            ('pow_float', lambda m: m([1, 2, 3]) ** 2.0),
            ('pow_ndarray', lambda m: m([1, 2, 3]) ** np.array([1, 2, 3])),
            ('pow_np_int', lambda m: m([1, 2, 3]) ** np.int64(3)),
            ('pow_bool', lambda m: m([1, 2, 3]) ** True),
            ('div_other_field', lambda m: m([1, 2]) / m([3, 4], cls=H)),
            ('div_float', lambda m: m([1, 2]) / 2.5),
            ('div_bool', lambda m: m([1, 2]) / True),
            ('div_complex', lambda m: m([1, 2]) / 1j),
            ('div_int_ndarray', lambda m: m([1, 2]) / np.array([3, 4])),
            ('rdiv_float', lambda m: 2.5 / m([1, 2])),
            ('binary_div', lambda m: m([3, 5, 7], cls=G) / m([1, 2, 3], cls=G)),
            ('binary_where', lambda m: np.where(np.array([True, False, True]), m([3, 5, 7], cls=G), m([1, 2, 3], cls=G))),
            ('binary_reciprocal', lambda m: m([3, 5, 7], cls=G).reciprocal()),
            ('empty_div', lambda m: m([], (0,)) / m([], (0,)))]


def test_calls_left_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst
    import oracle_device
    import oracle_divsel
    oracle_device.patch(monkeypatch)
    oracle_divsel.patch_resident(monkeypatch)
    P, Q = 2**127 - 1, 2**61 - 1
    F, H = finfields.GF(P).array, finfields.GF(Q).array
    G = finfields.GF(gfpx.GFpX(2)(283)).array

    def plain(vals, shape=None, cls=F):
        return cls(np.array(vals, dtype=object).reshape(shape or (len(vals),)))

    def limbed(vals, shape=None, cls=F):
        if cls is G or not vals:
            return plain(vals, shape, cls)
        return limb(cls, mpyc_b200.context_for(cls.field.modulus), vals, shape)
    table = reference_cases(F, G, H)
    want = [outcome(lambda: fn(plain)) for _, fn in table]
    assert sum(w[0] == 'raises' for w in want) >= 5
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for (name, fn), w in zip(table, want):
            assert outcome(lambda: fn(limbed)) == w, name
    finally:
        inst.uninstall()


def test_non_blum_sqrt_and_a_backend_without_k11_stay_with_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_conv
    import oracle_divsel
    oracle_device.patch(monkeypatch)
    p = 2**64 - 59                                       # p % 4 == 1
    assert p & 3 == 1
    F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
    sq = [v * v % p for v in (3, 5, 7)]
    want = outcome(lambda: F(np.array(sq, dtype=object)).sqrt())
    oracle_divsel.patch_resident(monkeypatch)
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        mat = resident.calls['materialised']
        assert outcome(lambda: limb(F, ctx, sq).sqrt()) == want
        assert resident.calls['materialised'] > mat
    finally:
        inst.uninstall()
    oracle_conv.patch_resident(monkeypatch)
    for name in oracle_divsel.METHODS:
        if name != 'nonzero':
            monkeypatch.delattr(resident.backend, name, raising=False)
    assert not resident._divsel_backend()
    calls = [lambda a, b: a / b, lambda a, b: 3 / a, lambda a, b: a.reciprocal(), lambda a, b: a ** -2, lambda a, b: a.is_sqr(),
             lambda a, b: np.where(np.array([True, False, True]), a, b)]
    want = [outcome(lambda: fn(F(np.array([2, 3, 4], dtype=object)), F(np.array([5, 6, 7], dtype=object)))) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for fn, w in zip(calls, want):
            a, b = limb(F, ctx, [2, 3, 4]), limb(F, ctx, [5, 6, 7])
            mat = resident.calls['materialised']
            assert outcome(lambda: fn(a, b)) == w
            assert resident.calls['materialised'] > mat
    finally:
        inst.uninstall()


def test_modvalue_zero_tests_count_and_where_match_numpy(monkeypatch):
    """The expressions of _np_is_zero, np_reciprocal and np_lsb on ModValues against NumPy object arithmetic mod p."""
    import mpyc_b200
    from mpyc_b200 import resident, codec
    import oracle_device
    import oracle_divsel
    import oracle_conv
    oracle_conv.patch_resident(monkeypatch)
    for name, fn in oracle_divsel.METHODS.items():
        monkeypatch.setattr(resident.backend, name, fn.__get__(resident.backend), raising=False)
    p = 2**61 - 1
    ctx = mpyc_b200.context_for(p)
    rng = np.random.default_rng(3)
    c = [0, 5, 0, p - 1, 2, 0, 7, 1]
    z = [int(v) for v in rng.integers(0, 2, size=8)]
    mk = lambda vals, exact=True: resident.ModValue(ctx, codec.ints_to_limbs(vals, ctx), (len(vals),), exact=exact)   # noqa: E731
    C, Z = np.array(c, dtype=object), np.array(z, dtype=object)

    def ints(v):
        return [int(e) % p for e in np.asarray(v._materialise() if type(v) is resident.ModValue else v, dtype=object).reshape(-1)]
    assert (mk(c) == 0).tolist() == (C == 0).tolist()
    assert np.count_nonzero(mk(c)) == np.count_nonzero(C) == 5
    mask = mk(c) == 0
    r = np.where(mask, 0, mk(z))                                     # runtime.py:3614
    assert type(r) is resident.ModValue and ints(r) == ints(np.where(C == 0, 0, Z))
    zz = mk(z)
    r = np.where(np.array([True, False] * 4), 1 - zz, zz)            # runtime.py:3615, a pending affine map
    assert ints(r) == ints(np.where(np.array([True, False] * 4), 1 - Z, Z))
    r = np.where(mk(c) & 1, 3 * zz + 4, -2)                          # a device mask: c & 1 != 0
    assert ints(r) == ints(np.where(C & 1, 3 * Z + 4, -2))
    r = np.where(mk(c) & 1, mk(z, exact=False) * mk(c), mk(c) ** 2)  # pending square on one side
    assert ints(r) == ints(np.where(C & 1, Z * C, C ** 2))
    with pytest.raises(AssertionError):
        np.where(mk(c) + 1, zz, zz)                                  # not an exact value: no truth value
    oracle_device.patch_resident(monkeypatch)                        # no K11: np.where settles, == 0 still runs on limbs
    r = np.where(mk(c) == 0, 0, mk(z))
    assert type(r) is np.ndarray and ints(r) == ints(np.where(C == 0, 0, Z))


def test_k11_abi_argument_errors():
    """Null buffers, sizes that overflow, overlapping buffers and non-canonical maps are rejected before any CUDA call;
    binary fields are unsupported; a valid call without a device fails with a CUDA error."""
    import mpyc_b200
    from mpyc_b200._cabi import lib, check, u64_array
    torch = pytest.importorskip('torch')
    p = 2**128 - 173
    ctx = mpyc_b200.context_for(p)                                    # 16-byte elements
    a, b, c, m = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 24), ctypes.c_void_p(1 << 30), ctypes.c_void_p(1 << 34)
    ok = u64_array([1, 0, 5, 0])
    bad = u64_array([p & (2**64 - 1), p >> 64, 0, 0])
    big = 1 << 62
    for call in [lambda: lib.mpyc_b200_ff_div(ctx.handle, None, b, c, 4, None),
                 lambda: lib.mpyc_b200_ff_div(ctx.handle, a, None, c, 4, None),
                 lambda: lib.mpyc_b200_ff_div(ctx.handle, a, b, None, 4, None),
                 lambda: lib.mpyc_b200_ff_div(ctx.handle, a, b, c, big, None),
                 lambda: lib.mpyc_b200_ff_div(ctx.handle, a, b, a, 4, None),
                 lambda: lib.mpyc_b200_ff_div(ctx.handle, a, b, ctypes.c_void_p((1 << 24) + 16), 4, None),
                 lambda: lib.mpyc_b200_ff_div(ctx.handle, a, b, ctypes.c_void_p((1 << 20) - 16), 4, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, None, 0, a, ok, b, ok, c, 4, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, m, 0, a, ok, b, ok, None, 4, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, m, 0, a, None, b, ok, c, 4, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, m, 0, a, ok, b, bad, c, 4, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, m, 0, a, ok, b, ok, c, big, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, m, 0, a, ok, b, ok, a, 4, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, m, 0, None, ok, b, ok, ctypes.c_void_p((1 << 24) + 32), 4, None),
                 lambda: lib.mpyc_b200_ff_select(ctx.handle, m, 1, a, ok, None, ok, ctypes.c_void_p((1 << 34) - 16), 4, None)]:
        with pytest.raises(ValueError):
            check(call())
    check(lib.mpyc_b200_ff_div(ctx.handle, None, None, None, 0, None))                 # n == 0: nothing to do
    check(lib.mpyc_b200_ff_select(ctx.handle, None, 0, None, ok, None, ok, None, 0, None))
    g = mpyc_b200.context_for(283, binary=True)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(lib.mpyc_b200_ff_div(g.handle, a, b, c, 4, None))
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(lib.mpyc_b200_ff_select(g.handle, m, 0, a, ok, b, ok, c, 4, None))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(lib.mpyc_b200_ff_div(ctx.handle, a, b, c, 4, None))
    with pytest.raises(RuntimeError):
        check(lib.mpyc_b200_ff_select(ctx.handle, m, 0, a, ok, b, ok, c, 4, None))
