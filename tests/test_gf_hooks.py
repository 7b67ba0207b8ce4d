"""GF(2^8) bit composition, broadcasts, stacked products and integer-array sums behind install() on the reference's own
finfields (K15 through mpyc_b200.resident, answered here by the CPU stand-in of tests/oracle_gf.py): the expressions of
tests/golden/gf_local.json reproduce the unmodified reference's values, result types and errors, without turning
limb-backed operands into Python ints where the hooks cover them.  Plain operands are packed; the calls left to the
reference reach it with its own result or error; a backend without K15 leaves every GF(2^8) case to the reference;
uninstall() restores the methods; the C-ABI entry points reject bad arguments without a GPU."""
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
_spec = importlib.util.spec_from_file_location('make_golden_gf', os.path.join(HERE, 'golden', 'make_golden_gf.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'gf_local.json')) as _fh:
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


def installed(monkeypatch, thresha, finfields, k15=True):
    from mpyc_b200 import install as inst
    import oracle_device
    import oracle_gf
    import oracle_matmul_int
    oracle_device.patch(monkeypatch)
    (oracle_gf if k15 else oracle_matmul_int).patch_resident(monkeypatch)
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=1)
    return inst


def field(finfields, gfpx, poly):
    import mpyc_b200
    G = finfields.GF(gfpx.GFpX(2)(poly))
    return G.array, mpyc_b200.context_for(poly, binary=True)


def limb_maker(F, ctx):
    from mpyc_b200 import resident, codec

    def make(shape, salt):
        return F(resident.LimbValue(ctx, codec.ints_to_limbs(gold.values(shape, salt), ctx), shape, type(F.field.modulus)),
                 check=False)
    return make


def run(F, ctx, name, make):
    """The case on operands from make; compose cases run on a ModValue, as np_to_bits / np_from_bits see the raw value."""
    from mpyc_b200 import resident
    specs = gold.CASES[name][0]
    if gold.CASES[name][1] != 'compose':
        return gold.run_case(F, name, make)
    shape = specs[0][1]
    x = make(shape, 0) if make else F(np.array(gold.values(shape, 0), dtype=object).reshape(shape))
    lv = resident.as_limb_value(resident.raw_value(x))
    v = resident.ModValue(ctx, lv.store, lv.shape, exact=True) if lv is not None else x.value
    return F(np.sum(v << np.arange(shape[-1]), axis=len(shape) - 1))


def test_fixture_inventory():
    assert len(FIXTURES) == len(gold.POLYS) * len(gold.CASES) == 82
    assert {c['poly'] for c in FIXTURES} == {283, 285}
    assert sum(c['want'][0] == 'raises' for c in FIXTURES) == 2 * 4
    assert sum(covered for _, _, covered in gold.CASES.values()) == 32


def test_limb_backed_operands_reproduce_the_fixtures(mpyc_mods, monkeypatch):
    """Every covered case runs on K15 (or K1's same-shape kernels) and settles nothing; the others give the reference's
    result or error."""
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import resident
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for c in FIXTURES:
            F, ctx = field(finfields, gfpx, c['poly'])
            name = c['case']
            mat, ops = resident.calls['materialised'], resident.calls['limb_ops']
            r = run(F, ctx, name, limb_maker(F, ctx))
            if gold.CASES[name][2]:
                assert resident.calls['materialised'] == mat and resident.calls['limb_ops'] > ops, name
                assert type(r) is F and resident.as_limb_value(resident.raw_value(r)) is not None, name
            else:
                assert resident.calls['materialised'] > mat or resident.calls['limb_ops'] == ops, name
            assert gold.outcome(r) == c['want'], name
    finally:
        inst.uninstall()


def test_plain_operands_are_packed_and_match_the_fixtures(mpyc_mods, monkeypatch):
    """Plain field arrays (and public object arrays) take the same hooks: they are packed, the result is limb-backed.  An
    integer ndarray is added on the device to a limb-backed array only, so with a plain one the reference adds them."""
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import resident
    inst = installed(monkeypatch, thresha, finfields)
    try:
        for c in FIXTURES:
            F, _ = field(finfields, gfpx, c['poly'])
            name = c['case']
            packed = resident.calls['packed']
            r = run(F, None, name, None)
            if gold.CASES[name][2] and gold.CASES[name][1] != 'compose' and not name.startswith('int'):
                assert resident.calls['packed'] > packed, name
                assert resident.as_limb_value(resident.raw_value(r)) is not None, name
            assert gold.outcome(r) == c['want'], name
    finally:
        inst.uninstall()


def test_a_backend_without_k15_leaves_gf256_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import resident
    inst = installed(monkeypatch, thresha, finfields, k15=False)
    try:
        for c in FIXTURES:
            F, ctx = field(finfields, gfpx, c['poly'])
            name = c['case']
            if gold.CASES[name][1] == 'compose' or name in ('sq4',):
                continue                    # ModValues are made only with K15; 2-D products of two arrays run on K1c as before
            ops = resident.calls['limb_ops']
            r = run(F, ctx, name, limb_maker(F, ctx))
            assert resident.calls['limb_ops'] == ops, name
            assert gold.outcome(r) == c['want'], name
    finally:
        inst.uninstall()


def test_modvalue_over_gf256_xors_and_settles_the_rest(mpyc_mods, monkeypatch):
    """np_to_bits' `a + r_modl` is XOR on the device; ring steps that are not + of two arrays settle to the reference's
    polynomial arithmetic."""
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import resident, codec
    inst = installed(monkeypatch, thresha, finfields)
    try:
        F, ctx = field(finfields, gfpx, 283)
        x, y = gold.values((6,), 0), gold.values((6,), 3)
        a = F(resident.LimbValue(ctx, codec.ints_to_limbs(x, ctx), (6,), type(F.field.modulus)), check=False)
        m = resident.ModValue(ctx, codec.ints_to_limbs(y, ctx), (6,), exact=True)
        mat = resident.calls['materialised']
        r = a + m
        assert resident.calls['materialised'] == mat
        assert [int(v) for v in r.value] == [u ^ v for u, v in zip(x, y)]
        m2 = resident.ModValue(ctx, codec.ints_to_limbs(y, ctx), (6,), exact=True)
        assert [int(v) for v in (m2 + m2)] == [0] * 6
        m3 = resident.ModValue(ctx, codec.ints_to_limbs(y, ctx), (6,), exact=True)
        want = np.array([F.field(v).value for v in y], dtype=object) * 3
        assert list(m3 * 3) == list(want)
    finally:
        inst.uninstall()


def test_uninstall_restores_the_patched_methods(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    cls = finfields.FiniteFieldArray
    names = ('__array_ufunc__', '__add__', '__radd__', '__mul__', '__matmul__', '__rmatmul__')
    orig = {n: cls.__dict__[n] for n in names}
    inst = installed(monkeypatch, thresha, finfields)
    assert all(cls.__dict__[n] is not m for n, m in orig.items())
    inst.uninstall()
    assert all(cls.__dict__[n] is m for n, m in orig.items())


def test_k15_abi_argument_errors():
    """Null buffers, l == 0, bad shapes and strides, sizes that overflow and overlapping buffers are rejected before any CUDA
    call; prime fields are unsupported; a valid call without a device fails with a CUDA error."""
    import mpyc_b200
    from mpyc_b200 import _cabi
    from mpyc_b200._cabi import lib, check
    torch = pytest.importorskip('torch')
    g = mpyc_b200.context_for(283, binary=True)
    p = mpyc_b200.context_for(2**64 - 189)
    x, y, z = ctypes.c_void_p(1 << 30), ctypes.c_void_p(1 << 32), ctypes.c_void_p(1 << 34)
    bc, mm, bv = lib.mpyc_b200_gf_bits_compose, lib.mpyc_b200_gf_matmul_batched, lib.mpyc_b200_gf_binop_view

    def view(shape, strides, offset=0):
        v = _cabi.View()
        v.offset, v.rank, v.index_axis = offset, len(shape), -1
        for k, (e, s) in enumerate(zip(shape, strides)):
            v.extent[k], v.stride[k] = e, s
        return ctypes.byref(v)
    big = 1 << 62
    calls = [lambda: bc(g.handle, None, 4, 8, z, None), lambda: bc(g.handle, x, 4, 8, None, None),
             lambda: bc(g.handle, x, 4, 0, z, None),                                        # l == 0
             lambda: bc(g.handle, x, big, big, z, None),                                    # n * l overflows
             lambda: bc(g.handle, x, 4, 8, ctypes.c_void_p((1 << 30) + 31), None),          # out overlaps the bits
             lambda: mm(g.handle, None, 0, y, 8, z, 5, 8, 8, 1, None),
             lambda: mm(g.handle, x, 0, y, 8, None, 5, 8, 8, 1, None),
             lambda: mm(g.handle, x, 3, y, 8, z, 5, 8, 8, 1, None),                         # stride neither 0 nor r k
             lambda: mm(g.handle, x, 0, y, 7, z, 5, 8, 8, 1, None),
             lambda: mm(g.handle, x, 0, y, 8, z, big, big, 8, 1, None),                     # sizes overflow
             lambda: mm(g.handle, x, 0, y, 8, ctypes.c_void_p((1 << 32) + 39), 5, 8, 8, 1, None),   # c overlaps b
             lambda: bv(g.handle, 0, None, 20, view((4, 5), (5, 1)), y, 5, view((4, 5), (0, 1)), z, None),
             lambda: bv(g.handle, 3, x, 20, view((4, 5), (5, 1)), y, 5, view((4, 5), (0, 1)), z, None),   # op
             lambda: bv(g.handle, 0, x, 20, view((4, 5), (5, 1)), y, 4, view((4, 5), (0, 1)), z, None),   # outside b
             lambda: bv(g.handle, 0, x, 20, view((4, 5), (5, 1)), y, 5, view((4, 4), (0, 1)), z, None),   # extents
             lambda: bv(g.handle, 0, x, 20, view((4, 5), (5, 1)), y, 5, view((4, 5), (0, 1)), ctypes.c_void_p((1 << 30) + 3), None)]
    for call in calls:
        with pytest.raises(ValueError):
            check(call())
    check(bc(g.handle, None, 0, 8, None, None))                          # nothing to do
    check(mm(g.handle, None, 0, None, 0, None, 0, 8, 8, 1, None))
    for call in (lambda: bc(p.handle, x, 4, 8, z, None), lambda: mm(p.handle, x, 0, y, 8, z, 5, 8, 8, 1, None),
                 lambda: bv(p.handle, 0, x, 20, view((4, 5), (5, 1)), y, 5, view((4, 5), (0, 1)), z, None)):
        with pytest.raises(mpyc_b200.UnsupportedFieldError):
            check(call())
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(bc(g.handle, x, 4, 8, z, None))


def test_prime_fields_keep_their_integer_sums_and_gf256_joins_pack_plain_pieces(mpyc_mods, monkeypatch):
    """An integer ndarray plus a plain prime-field array goes to the reference without packing (the np.add branch of
    __array_ufunc__ serves GF(2^8) only); over GF(2^8) a join of a limb-backed and a plain piece packs the plain one."""
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import resident
    inst = installed(monkeypatch, thresha, finfields)
    try:
        P = finfields.GF(2**61 - 1).array
        x = P(np.array(gold.values((3, 4), 1), dtype=object).reshape(3, 4))
        c = np.arange(12, dtype=np.int64).reshape(3, 4)
        packed = resident.calls['packed']
        r = c + x
        assert resident.calls['packed'] == packed
        assert [int(v) for v in np.reshape(r.value, -1)] == [(a + b) % (2**61 - 1) for a, b in zip(range(12), gold.values((3, 4), 1))]
        F, ctx = field(finfields, gfpx, 283)
        a = limb_maker(F, ctx)((2, 3), 0)
        b = F(np.array(gold.values((2, 2), 1), dtype=object).reshape(2, 2))
        mat, packed = resident.calls['materialised'], resident.calls['packed']
        j = np.concatenate((a, b), axis=1)
        assert resident.calls['materialised'] == mat and resident.calls['packed'] == packed + 1
        want = np.concatenate((np.array(gold.values((2, 3), 0)).reshape(2, 3), np.array(gold.values((2, 2), 1)).reshape(2, 2)), axis=1)
        assert [int(v) for v in np.reshape(j.value, -1)] == want.reshape(-1).tolist()
    finally:
        inst.uninstall()
