"""Per-element exponents behind install() on the reference's own finfields and gmpy (K12 through mpyc_b200.resident and
mpyc_b200.finfields, answered here by the CPU stand-in of tests/oracle_powexp.py): x ** e and x **= e with an exponent array
of x's shape, PrimeFieldArray._pow on plain object arrays, and gmpy.powmod_exp_list reproduce tests/golden/powexp.json --
the unmodified reference's values, and its exception type and message where it raises -- without turning limb-backed inputs
into Python ints or modifying them.  The calls left to the reference reach it with its own result or error; uninstall()
restores gmpy.powmod_exp_list; the C-ABI entry point rejects bad arguments without a GPU."""
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
_spec = importlib.util.spec_from_file_location('make_golden_powexp', os.path.join(HERE, 'golden', 'make_golden_powexp.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'powexp.json')) as _fh:
    FIXTURES = json.load(_fh)


@pytest.fixture(scope='module')
def mpyc_mods():
    if REF is None:
        pytest.skip('reference not present ($MPYC_REFERENCE, or the copy build() makes in oracle/_ref)')
    sys.dont_write_bytecode = True
    sys.path.insert(0, REF)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import thresha, finfields, gfpx, gmpy
    finally:
        sys.argv = argv
    yield thresha, finfields, gfpx, gmpy
    sys.path.remove(REF)


def outcome(fn):
    try:
        r = fn()
    except Exception as e:   # noqa: BLE001
        return ('raises', type(e).__name__, str(e))
    if isinstance(r, list):
        return ('list', r)
    return ('array', type(r).__name__, r.shape, [int(v) for v in np.asarray(r.value, dtype=object).reshape(-1)])


def encoded(fn):
    try:
        r = fn()
    except Exception as e:   # noqa: BLE001
        return {'error': [type(e).__name__, str(e)]}
    return gold.encode(r)


def limb(F, ctx, vals, shape=None):
    from mpyc_b200 import resident, codec
    return F(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), shape or (len(vals),)), check=False)


def want_of(c):
    return {k: v for k, v in c.items() if k in ('hex', 'error')}


def installed(monkeypatch, thresha, finfields, min_size=1):
    from mpyc_b200 import install as inst
    import oracle_device
    import oracle_powexp
    oracle_device.patch(monkeypatch)
    oracle_powexp.patch_resident(monkeypatch)
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=min_size, finfields_min_size=1)
    return inst


def test_hooks_reproduce_the_golden_fixtures(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx, gmpy = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    assert len(FIXTURES) == 168 and sum('error' in c for c in FIXTURES) == 54
    inst = installed(monkeypatch, thresha, finfields)
    try:
        assert getattr(gmpy.powmod_exp_list, '__mpyc_b200__', False)
        for c in FIXTURES:
            p = int(c['p'], 16)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            b, e, fn = gold.CASES[c['case']]
            ex = gold.exponents(p, e)
            mat, pe = resident.calls['materialised'], resident.calls['pow_exp']
            if fn is None:
                got = encoded(lambda: gmpy.powmod_exp_list(gold.list_base(p, b), ex.tolist() if e == 'obj' else ex, p))
            else:
                x = limb(F, ctx, gold.bases(p, b))
                keep = resident.raw_value(x)
                res = [None]

                def run():
                    res[0] = fn(F, x, ex)
                    return res[0]
                try:
                    run()
                except Exception:   # noqa: BLE001
                    pass
                # negative per-element exponents go to the reference, which reads x's values
                assert resident.calls['materialised'] == mat or e == 'neg', c['case']
                if e != 'neg':
                    assert type(resident.raw_value(res[0])) is resident.LimbValue, c['case']
                got = encoded(lambda: res[0] if 'error' not in c else fn(F, x, ex))
                assert [int(v) for v in keep._materialise()] == gold.bases(p, b), c['case']   # the input's store is intact
            assert got == want_of(c), c['case']
            # every call without an error ran on K12 except negative per-element exponents and NumPy-int exponent lists
            on_device = 'error' not in c and e != 'neg' or (fn is None and e == 'neg' and 'error' not in c)
            assert resident.calls['pow_exp'] == pe + on_device, c['case']
    finally:
        inst.uninstall()


def test_plain_object_arrays_take_the_pow_hook(mpyc_mods, monkeypatch):
    """PrimeFieldArray._pow on plain object arrays (install(finfields_module=...)): x ** e with e an exponent array."""
    thresha, finfields, gfpx, gmpy = mpyc_mods
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_powexp
    oracle_device.patch(monkeypatch)
    oracle_powexp.patch_resident(monkeypatch)
    inst.install(thresha, finfields_module=finfields, finfields_min_size=1)
    try:
        for c in FIXTURES:
            b, e, fn = gold.CASES[c['case']]
            if fn is None:
                continue
            p = int(c['p'], 16)
            F = finfields.GF(p).array
            pe = resident.calls['pow_exp']
            assert encoded(lambda: fn(F, F(np.array(gold.bases(p, b), dtype=object)), gold.exponents(p, e))) == want_of(c), c['case']
            assert resident.calls['pow_exp'] == pe + (e != 'neg'), c['case']
    finally:
        inst.uninstall()


def test_in_place_power_leaves_sharers_unchanged(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx, gmpy = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    p = 2**64 - 189
    F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
    inst = installed(monkeypatch, thresha, finfields)
    try:
        x = limb(F, ctx, [3, 4, 5, 6])
        y = F(resident.raw_value(x), check=False)            # shares x's store
        x **= np.array([2, 0, 2**70, 1], dtype=object)
        assert type(resident.raw_value(x)) is resident.LimbValue
        assert [int(v) for v in x.value] == [9, 1, pow(5, 2**70, p), 6]
        assert [int(v) for v in y.value] == [3, 4, 5, 6]
    finally:
        inst.uninstall()


def test_calls_left_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx, gmpy = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    P = 2**127 - 1
    F = finfields.GF(P).array
    G = finfields.GF(gfpx.GFpX(2)(283)).array
    mpyc_b200.context_for(P)
    vals = [2, 3, 0, 5]
    table = [
        ('broadcast', F, lambda x: x ** np.array([3], dtype=object)),
        ('broadcast_2d', F, lambda x: x ** np.array([[1, 2, 3, 4]], dtype=np.int64)),
        ('bool', F, lambda x: x ** np.array([True, False, True, True])),
        ('float', F, lambda x: x ** np.array([1.0, 2.0, 3.0, 4.0])),
        ('int32', F, lambda x: x ** np.array([1, 2, 3, 4], dtype=np.int32)),
        ('wide', F, lambda x: x ** np.array([2**256, 1, 2, 3], dtype=object)),
        ('negative', F, lambda x: x ** np.array([-1, 1, 2, 3], dtype=np.int64)),
        ('negative_nonzero', F, lambda x: (x + 1) ** np.array([-1, 1, -2, 3], dtype=object)),
        ('binary', G, lambda x: x ** np.array([1, 2, 3, 4], dtype=object)),
    ]

    def make(cls, limbed):
        if limbed and cls is F:
            return limb(F, mpyc_b200.context_for(P), vals)
        return cls(np.array(vals, dtype=object))
    want = [outcome(lambda: fn(make(cls, False))) for _, cls, fn in table]
    from mpyc_b200 import field
    assert (2**89 - 1, False) not in field._contexts
    lists = [(3, [1, 2, 3], 2**89 - 1),                           # a prime the engine holds no context for
             (3, [1, 2, 3], 2**64),                               # composite
             (0, [1, -2, 3], P), (P, [-1], P),                    # a zero base with a negative exponent
             (3, np.array([1, 2, 3], dtype=np.int64), P),         # NumPy ints
             (3, np.array([[1, 2]], dtype=object), P),            # not 1-D
             (3, [1.5, 2], P), (3, [2**256, 1], P), (3.0, [1, 2], P), (True, [1, 2], P), (3, range(1, 3), P)]
    want_lists = [outcome(lambda: gmpy.powmod_exp_list(*args)) for args in lists]
    assert sum(w[0] == 'raises' for w in want + want_lists) >= 6
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for (name, cls, fn), w in zip(table, want):
            pe = resident.calls['pow_exp']
            assert outcome(lambda: fn(make(cls, True))) == w, name
            assert resident.calls['pow_exp'] == pe, name
        for args, w in zip(lists, want_lists):
            pe = resident.calls['pow_exp']
            assert outcome(lambda: gmpy.powmod_exp_list(*args)) == w, args
            assert resident.calls['pow_exp'] == pe, args
    finally:
        inst.uninstall()


def test_min_size_and_a_backend_without_k12(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx, gmpy = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    P = 2**127 - 1
    mpyc_b200.context_for(P)
    inst = installed(monkeypatch, thresha, finfields, min_size=4)
    try:
        pe = resident.calls['pow_exp']
        assert gmpy.powmod_exp_list(3, [1, 2, 3], P) == [3, 9, 27]
        assert resident.calls['pow_exp'] == pe
        assert gmpy.powmod_exp_list(3, [1, 2, 3, -1], P) == [3, 9, 27, pow(3, -1, P)]
        assert resident.calls['pow_exp'] == pe + 1
    finally:
        inst.uninstall()
    monkeypatch.delattr(resident.backend, 'pow_exp')
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=1, finfields_min_size=1)
    try:
        assert not resident._powexp_backend()
        pe = resident.calls['pow_exp']
        F = finfields.GF(P).array
        x = limb(F, mpyc_b200.context_for(P), [2, 3])
        assert [int(v) for v in (x ** np.array([5, 7], dtype=object)).value] == [32, 3**7]
        assert gmpy.powmod_exp_list(3, [1, 2, 3, 4], P) == [3, 9, 27, 81]
        assert resident.calls['pow_exp'] == pe
    finally:
        inst.uninstall()


def test_uninstall_restores_powmod_exp_list(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx, gmpy = mpyc_mods
    orig = gmpy.powmod_exp_list
    inst = installed(monkeypatch, thresha, finfields)
    assert gmpy.powmod_exp_list is not orig
    inst.uninstall()
    assert gmpy.powmod_exp_list is orig
    inst.install(thresha, operators=True, finfields_module=finfields)      # not resident: left alone
    try:
        assert gmpy.powmod_exp_list is orig
    finally:
        inst.uninstall()
    assert gmpy.powmod_exp_list is orig


def test_exponent_packing():
    from mpyc_b200 import codec
    limbs, signs, bits = codec.exponents_to_limbs(np.array([0, 5, -(2**63), 2**63 - 1], dtype=np.int64))
    assert limbs.shape == (4, 1) and bits == 64 and signs.tolist() == [0, 0, 1, 0]
    assert limbs[:, 0].tolist() == [0, 5, 2**63, 2**63 - 1]
    limbs, signs, bits = codec.exponents_to_limbs(np.array([2**64 - 1, 3], dtype=np.uint64))
    assert signs is None and bits == 64 and limbs[:, 0].tolist() == [2**64 - 1, 3]
    vals = [0, 1, -(2**130 + 7), 2**255 + 3]
    limbs, signs, bits = codec.exponents_to_limbs(np.array(vals, dtype=object))
    assert limbs.shape == (4, 4) and bits == 256 and signs.tolist() == [0, 0, 1, 0]
    assert [sum(int(w) << (64 * i) for i, w in enumerate(r)) for r in limbs] == [abs(v) for v in vals]
    limbs, signs, bits = codec.exponents_to_limbs([0, 0])
    assert limbs.shape == (2, 1) and bits == 0 and signs is None
    assert codec.exponents_to_limbs([]) is not None
    for bad in (np.array([True]), np.array([1.0]), np.array([1], dtype=np.int32), [2**256], [1, 2.0], [True], 'ab', 3):
        assert codec.exponents_to_limbs(bad) is None


def test_k12_abi_argument_errors():
    """Null buffers, bases given twice or not at all, signs with per-element bases, a non-canonical base, bad exponent widths,
    sizes that overflow and overlapping buffers are rejected before any CUDA call; binary fields are unsupported; a valid
    call without a device fails with a CUDA error."""
    import mpyc_b200
    from mpyc_b200._cabi import lib, check, u64_array
    torch = pytest.importorskip('torch')
    p = 2**128 - 173
    ctx = mpyc_b200.context_for(p)                                    # 16-byte elements
    a, e, c, s = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 24), ctypes.c_void_p(1 << 30), ctypes.c_void_p(1 << 34)
    ok = u64_array([5, 0])
    bad = u64_array([p & (2**64 - 1), p >> 64])
    big = 1 << 62
    f = lib.mpyc_b200_ff_pow_exp
    for call in [lambda: f(ctx.handle, a, ok, e, 1, 64, None, 4, c, None),          # both bases
                 lambda: f(ctx.handle, None, None, e, 1, 64, None, 4, c, None),     # neither
                 lambda: f(ctx.handle, a, None, e, 1, 64, s, 4, c, None),           # signs with per-element bases
                 lambda: f(ctx.handle, None, bad, e, 1, 64, None, 4, c, None),      # non-canonical base
                 lambda: f(ctx.handle, None, ok, e, 0, 0, None, 4, c, None),
                 lambda: f(ctx.handle, None, ok, e, 5, 64, None, 4, c, None),
                 lambda: f(ctx.handle, None, ok, e, 1, 65, None, 4, c, None),
                 lambda: f(ctx.handle, None, ok, e, 2, -1, None, 4, c, None),
                 lambda: f(ctx.handle, None, ok, None, 1, 64, None, 4, c, None),
                 lambda: f(ctx.handle, None, ok, e, 1, 64, None, 4, None, None),
                 lambda: f(ctx.handle, None, ok, e, 4, 256, None, big, c, None),
                 lambda: f(ctx.handle, None, ok, e, 1, 64, None, 4, ctypes.c_void_p((1 << 24) + 8), None),
                 lambda: f(ctx.handle, None, ok, e, 1, 64, None, 4, ctypes.c_void_p((1 << 24) - 32), None),
                 lambda: f(ctx.handle, None, ok, e, 1, 64, s, 4, ctypes.c_void_p((1 << 34) - 16), None),
                 lambda: f(ctx.handle, a, None, e, 1, 64, None, 4, ctypes.c_void_p((1 << 20) + 16), None)]:
        with pytest.raises(ValueError):
            check(call())
    check(f(ctx.handle, None, ok, None, 1, 64, None, 0, None, None))                 # n == 0: nothing to do
    g = mpyc_b200.context_for(283, binary=True)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(f(g.handle, None, ok, e, 1, 64, None, 4, c, None))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(f(ctx.handle, a, None, e, 1, 64, None, 4, c, None))
