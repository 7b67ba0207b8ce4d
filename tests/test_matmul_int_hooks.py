"""Prime-field matrices times public integer matrices behind install() on the reference's own finfields (K14 through
mpyc_b200.resident, answered here by the CPU stand-in of tests/oracle_matmul_int.py): `x @ W`, `W @ x` and np.matmul
reproduce tests/golden/matmul_int.json -- the unmodified reference's values and result types, and its exception type and
message where it raises -- without turning limb-backed operands into Python ints.  np.matmul of two field arrays and
object-int operands take K1c; the calls left to the reference reach it with its own result or error; uninstall() restores
__array_ufunc__ and __matmul__; the C-ABI entry point rejects bad arguments without a GPU."""
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import pytest

from oracle import reference

REF = reference.path()
pytestmark = pytest.mark.filterwarnings('ignore::PendingDeprecationWarning')     # np.matrix operands
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden_matmul_int', os.path.join(HERE, 'golden', 'make_golden_matmul_int.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'matmul_int.json')) as _fh:
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


def want_of(c):
    return {k: v for k, v in c.items() if k not in ('p', 'case')}


def limb(F, ctx, vals, shape):
    from mpyc_b200 import resident, codec
    return F(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), shape), check=False)


def installed(monkeypatch, thresha, finfields, min_size=1, public=True):
    from mpyc_b200 import install as inst
    import oracle_device
    import oracle_matmul_int
    oracle_device.patch(monkeypatch)
    oracle_matmul_int.patch_resident(monkeypatch)
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=min_size, public_matmul=public)
    return inst


def k14_case(name):
    """Cases with a NumPy integer operand that K14 computes."""
    return name.startswith(('xW_', 'Wx_', 'np_xW_', 'np_Wx_'))


def inner(name):
    """1-D @ 1-D: the one-element result is settled, as for field @ field."""
    return name in ('xW_v_v', 'Wx_v_v', 'np_xW_v_v', 'np_ff_v_v', 'obj_Wx_v') or name.startswith('xW_pm1v_')


def _terms(c):
    """r * k * c of an integer-operand case, from the result's shape and the field operand's k (the size rule for plain
    operands)"""
    xs = gold.SHAPES[gold.CASES[c['case']][0]]
    k = xs[0] if c['case'].startswith(('Wx_', 'np_Wx_')) else xs[-1]
    return int(np.prod(c['shape'])) * k


def outcome(fn):
    try:
        return gold.encode(fn())
    except Exception as e:   # noqa: BLE001
        return {'error': [type(e).__name__, str(e)]}


def test_fixture_inventory():
    assert len(FIXTURES) == 6 * len(gold.CASES) == 504
    assert sum('error' in c for c in FIXTURES) == 6 * 6
    assert {c.get('kind') for c in FIXTURES} == {'array', 'element', None}
    assert sum(k14_case(n) for n in gold.CASES) == 65


def test_hooks_reproduce_the_golden_fixtures(mpyc_mods, monkeypatch):
    """Limb-backed field operands: every integer-operand case runs on K14 (one call) and settles nothing but a 1-D @ 1-D
    result; np.matmul of field arrays and object-int operands run on K1c; the calls left to the reference give its own
    results and errors.  The operand's store is never modified."""
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
            mat, k14 = resident.calls['materialised'], resident.calls['matmul_int']
            name = c['case']
            try:
                res = fn(F, x)
            except Exception as e:   # noqa: BLE001
                assert [type(e).__name__, str(e)] == c['error'], name
                assert resident.calls['matmul_int'] == k14, name
                continue
            assert resident.calls['matmul_int'] == k14 + k14_case(name), name
            if not name.startswith('ref_'):
                assert resident.calls['materialised'] == mat + inner(name), name
            if not name.startswith('ref_'):
                if c['kind'] == 'element':
                    assert type(res) is F.field, name
                elif c['shape']:
                    assert type(res) is F and type(resident.raw_value(res)) is resident.LimbValue, name
                else:
                    assert type(res) is F, name                        # np.matmul's 0-d array
            assert gold.encode(res) == want_of(c), name
            assert [int(v) for v in np.reshape(keep._materialise(), -1)] == vals, name
    finally:
        inst.uninstall()


def test_plain_object_arrays_match_the_fixtures(mpyc_mods, monkeypatch):
    """Plain object-array field operands take the same hooks when r * k * c reaches operators_min_size * 8."""
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import resident
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for c in FIXTURES:
            if c['p'] not in (hex(gold.P61), hex(gold.P64G), hex(gold.P256)):
                continue
            F = finfields.GF(int(c['p'], 16)).array
            d, fn = gold.CASES[c['case']]
            k14 = resident.calls['matmul_int']
            assert outcome(lambda: fn(F, gold.operand(F, d))) == want_of(c), c['case']
            hooked = resident.calls['matmul_int'] - k14
            assert hooked == (k14_case(c['case']) and _terms(c) >= 8), c['case']
    finally:
        inst.uninstall()


def test_calls_left_to_the_reference(mpyc_mods, monkeypatch):
    """Binary fields, a backend without matmul_int, small plain operands, @= and other ufuncs keep the reference's code."""
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    P = 2**64 - 189
    F = finfields.GF(P).array
    G = finfields.GF(gfpx.GFpX(2)(283)).array
    ctx = mpyc_b200.context_for(P)
    vals = [2, 3, 0, 5, 7, 1]
    W = np.array([[1, -2], [3, 4], [5, -6]], dtype=np.int64)
    table = [
        ('binary_xW', lambda: G(np.array(vals, dtype=object).reshape(2, 3)) @ W),
        ('binary_Wx', lambda: W.T @ G(np.array(vals, dtype=object).reshape(2, 3))),
        ('imatmul', lambda: _imatmul(limb(F, ctx, vals, (2, 3)), np.ones((3, 3), dtype=np.int64))),
        ('add_ufunc', lambda: np.add(np.ones((2, 3), dtype=np.int64), limb(F, ctx, vals, (2, 3)))),
        ('matmul_at', lambda: np.matmul.reduce(limb(F, ctx, vals, (2, 3)))),
    ]
    want = {name: outcome(fn) for name, fn in table}
    assert want['matmul_at'].get('error')
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for name, fn in table:
            k14 = resident.calls['matmul_int']
            assert outcome(fn) == want[name], name
            assert resident.calls['matmul_int'] == k14, name
    finally:
        inst.uninstall()
    inst = installed(monkeypatch, thresha, finfields, min_size=8)
    try:
        k14 = resident.calls['matmul_int']
        small = F(np.array(vals, dtype=object).reshape(2, 3))
        assert [int(v) for v in (small @ W).value.reshape(-1)] == [(a % P) for a in (np.array(vals, dtype=object).reshape(2, 3) @ W).reshape(-1)]
        assert resident.calls['matmul_int'] == k14                  # plain and r * k * c < 8 * min_size
        limb(F, ctx, vals, (2, 3)) @ W                              # limb-backed: any size
        assert resident.calls['matmul_int'] == k14 + 1
        monkeypatch.delattr(resident.backend, 'matmul_int')
        x = limb(F, ctx, vals, (2, 3))
        assert [int(v) for v in (x @ W).value.reshape(-1)] == [(a % P) for a in (np.array(vals, dtype=object).reshape(2, 3) @ W).reshape(-1)]
        assert resident.calls['matmul_int'] == k14 + 1
    finally:
        inst.uninstall()


def test_without_public_matmul_integer_operands_keep_the_reference_path(mpyc_mods, monkeypatch):
    """install() without public_matmul: a limb-backed operand of @ / np.matmul with an integer ndarray is settled and the
    reference's code computes, exactly as before K14 (so existing programs keep their conversion counts); np.matmul of two
    field arrays still runs on K1c.  uninstall() clears the option."""
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import resident
    P = 2**64 - 189
    F = finfields.GF(P).array
    ctx = mpyc_b200.context_for(P)
    vals = [2, 3, 0, 5, 7, 1]
    W = np.array([[1, -2], [3, 4], [5, -6]], dtype=np.int64)
    want = [int(a) % P for a in (np.array(vals, dtype=object).reshape(2, 3) @ W).reshape(-1)]
    inst = installed(monkeypatch, thresha, finfields, public=False)
    try:
        assert resident.public_matmul is False
        for fn in (lambda x: x @ W, lambda x: np.matmul(x, W), lambda x: np.matmul(W.T.copy(), x.T)):
            x = limb(F, ctx, vals, (2, 3))
            k14, mat = resident.calls['matmul_int'], resident.calls['materialised']
            r = fn(x)
            assert resident.calls['matmul_int'] == k14 and resident.calls['materialised'] == mat + 1
            got = [int(v) for v in np.reshape(r.value, -1)]
            assert got in (want, [int(a) % P for a in (np.array(want, dtype=object).reshape(2, 2).T).reshape(-1)])
        x = limb(F, ctx, vals, (2, 3))
        mat = resident.calls['materialised']
        y = np.matmul(x, limb(F, ctx, vals, (2, 3)).T)
        assert resident.calls['materialised'] == mat and type(resident.raw_value(y)) is resident.LimbValue
    finally:
        inst.uninstall()
    inst = installed(monkeypatch, thresha, finfields)
    assert resident.public_matmul is True
    inst.uninstall()
    assert resident.public_matmul is False


def _imatmul(x, w):
    x @= w
    return x


def test_uninstall_restores_array_ufunc_and_matmul(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    cls = finfields.FiniteFieldArray
    orig = {n: cls.__dict__[n] for n in ('__array_ufunc__', '__matmul__', '__rmatmul__')}
    inst = installed(monkeypatch, thresha, finfields)
    assert all(cls.__dict__[n] is not m for n, m in orig.items())
    inst.uninstall()
    assert all(cls.__dict__[n] is m for n, m in orig.items())


def test_k14_abi_argument_errors():
    """Null buffers, sizes that overflow, misaligned and overlapping buffers are rejected before any CUDA call; binary
    fields are unsupported; a valid call without a device fails with a CUDA error."""
    import mpyc_b200
    from mpyc_b200._cabi import lib, check
    torch = pytest.importorskip('torch')
    p = 2**128 - 173
    ctx = mpyc_b200.context_for(p)                                    # 16-byte elements
    mm = lib.mpyc_b200_ff_matmul_int
    x, w, c = ctypes.c_void_p(1 << 30), ctypes.c_void_p(1 << 32), ctypes.c_void_p(1 << 34)
    big = 1 << 62
    calls = [lambda: mm(ctx.handle, None, w, 0, 0, c, 2, 3, 4, None),
             lambda: mm(ctx.handle, x, None, 0, 1, c, 2, 3, 4, None),
             lambda: mm(ctx.handle, x, w, 0, 0, None, 2, 3, 4, None),
             lambda: mm(ctx.handle, x, w, 0, 0, c, big, big, 4, None),                            # r * k overflows
             lambda: mm(ctx.handle, x, w, 1, 1, c, 4, big, big, None),
             lambda: mm(ctx.handle, x, w, 0, 0, c, 2, 1 << 60, 1, None),                          # bytes overflow
             lambda: mm(ctx.handle, ctypes.c_void_p((1 << 30) + 4), w, 0, 0, c, 2, 3, 4, None),   # misaligned
             lambda: mm(ctx.handle, x, ctypes.c_void_p((1 << 32) + 2), 0, 0, c, 2, 3, 4, None),
             lambda: mm(ctx.handle, x, w, 0, 0, ctypes.c_void_p((1 << 34) + 1), 2, 3, 4, None),
             lambda: mm(ctx.handle, x, w, 0, 0, ctypes.c_void_p((1 << 30) + 16 * 5), 2, 3, 4, None),  # c overlaps x
             lambda: mm(ctx.handle, x, w, 0, 1, ctypes.c_void_p((1 << 32) - 16), 2, 3, 4, None)]      # c overlaps w
    for call in calls:
        with pytest.raises(ValueError):
            check(call())
    check(mm(ctx.handle, None, None, 0, 0, None, 0, 3, 4, None))      # empty output: nothing to do
    check(mm(ctx.handle, None, None, 1, 1, None, 2, 3, 0, None))
    g = mpyc_b200.context_for(283, binary=True)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(mm(g.handle, x, w, 0, 0, c, 2, 3, 4, None))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(mm(ctx.handle, x, w, 0, 0, c, 2, 3, 4, None))
