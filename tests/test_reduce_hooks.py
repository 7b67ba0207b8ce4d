"""np.sum / FiniteFieldArray.sum / np.cumsum / np.cumulative_sum / np.outer behind install(operators=True) on the
reference's own finfields (K7 / K1c through mpyc_b200.resident, answered here by the CPU oracle stand-in): every result
equals the uninstalled reference's in type, shape and value, limb-backed inputs are never turned into Python ints, and
every call the hooks leave alone still returns the reference's result or raises its error.  Also the argument errors of
the two K7 C-ABI entry points, which need no GPU."""
import ctypes
import sys

import numpy as np
import pytest

from oracle import reference

REF = reference.path()
P = 2**128 - 173


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


def call(fn):
    """fn()'s result, or the type of the exception it raised"""
    try:
        return fn()
    except Exception as e:   # noqa: BLE001
        return ('raises', type(e))


def outcome(r):
    """('array', class, shape, values) / ('element', class, value) / ('raises', exception type) of a call's result"""
    if isinstance(r, tuple) and r[0] == 'raises':
        return r
    if isinstance(r, np.ndarray):
        return ('ndarray', r.shape, r.tolist())
    if hasattr(r, 'field'):
        return ('array', type(r).__name__, r.shape, [int(v) for v in np.asarray(r.value, dtype=object).reshape(-1)])
    return ('element', type(r).__name__, int(r))


SHAPES = [(), (5,), (3, 4), (2, 3, 4), (2, 1, 3, 2), (0, 3)]


def axis_forms(ndim):
    forms = [None, (), 0, -1, ndim, (0, 0), 1.5]
    forms += [(a,) for a in range(ndim)] + [(a, b) for a in range(ndim) for b in range(a + 1, ndim)]
    forms += [(-1, 0), tuple(range(ndim))] + ([(0, 2), (1, 3), (0, 1, 3)] if ndim == 4 else [])
    return forms


def sum_cases(F, ints):
    """(name, covered, fn(make)) -- make(shape) builds the operand; covered: the hooks must take the call"""
    cases = []
    for shape in SHAPES:
        nd = len(shape)
        for axis in axis_forms(nd):
            try:
                from mpyc_b200 import axes
                axes.sum_plan(shape, axis, False)
                ok = True
            except (TypeError, ValueError):
                ok = False
            for keepdims in (False, True):
                for initial in (0, 5, -3, P + 2):
                    if initial and keepdims and axis not in (None, 0, (0, 1)):
                        continue
                    cases.append((f'sum{shape}{axis}{keepdims}{initial}', ok, shape,
                                  lambda a, axis=axis, k=keepdims, i=initial: np.sum(a, axis=axis, keepdims=k, initial=i)))
        if nd:
            cases.append((f'method{shape}', True, shape, lambda a: a.sum()))
            cases.append((f'method0{shape}', True, shape, lambda a: a.sum(0)))
            cases.append((f'method_kw{shape}', True, shape, lambda a: a.sum(axis=-1, keepdims=True, initial=7)))
            cases.append((f'np_sum_pos{shape}', True, shape, lambda a: np.sum(a, 0)))
        for axis in (None, 0, -1, 1, (0,), nd):
            ok = axis is None or (isinstance(axis, int) and -nd <= axis < nd)
            cases.append((f'cumsum{shape}{axis}', ok, shape, lambda a, axis=axis: np.cumsum(a, axis=axis)))
            for inc in (False, True):
                ok2 = ok and (axis is not None or nd <= 1)
                cases.append((f'cumulative{shape}{axis}{inc}', ok2, shape,
                              lambda a, axis=axis, inc=inc: np.cumulative_sum(a, axis=axis, include_initial=inc)))
        # left to the reference: dtype= / where= / a non-int initial
        cases.append((f'dtype{shape}', False, shape, lambda a: np.sum(a, dtype=object)))
        cases.append((f'where{shape}', False, shape, lambda a: np.sum(a, where=np.ones(np.shape(a), dtype=bool))))
        cases.append((f'init_elem{shape}', False, shape, lambda a: np.sum(a, initial=F(3))))
        cases.append((f'cumsum_dtype{shape}', False, shape, lambda a: np.cumsum(a, dtype=object)))
    return cases


def test_sums_and_scans_equal_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_reduce
    oracle_device.patch(monkeypatch)
    oracle_reduce.patch_resident(monkeypatch)
    F = finfields.GF(P)
    ctx = mpyc_b200.context_for(P)

    def values(shape):
        n = int(np.prod(shape, dtype=object))
        return [(7 * i * i + 3 * i + (P - 1 if i % 3 == 0 else 0)) % P for i in range(n)]

    def plain(shape):
        return F.array(np.array(values(shape), dtype=object).reshape(shape))

    def limb(shape):
        return F.array(resident.LimbValue(ctx, codec.ints_to_limbs(values(shape), ctx), shape), check=False)

    cases = sum_cases(F, values)
    want = [outcome(call(lambda: fn(plain(shape)))) for _, _, shape, fn in cases]
    assert sum(w[0] == 'raises' for w in want) > 10 and sum(w[0] == 'element' for w in want) > 10
    before = F.array.__mro__[2].__dict__.get('sum')
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for (name, covered, shape, fn), w in zip(cases, want):
            for make in (limb, plain):
                a = make(shape)
                ops, mat = resident.calls['limb_ops'], resident.calls['materialised']
                r = call(lambda: fn(a))
                if make is limb and covered:
                    assert resident.calls['materialised'] == mat, name
                    assert resident.calls['limb_ops'] > ops, name
                if not covered:
                    assert resident.calls['limb_ops'] == ops, name
                assert outcome(r) == w, (name, make.__name__)
    finally:
        inst.uninstall()
    assert F.array.__mro__[2].__dict__.get('sum') is before


def test_outer_equals_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    oracle_device.patch(monkeypatch)
    oracle_device.patch_resident(monkeypatch)
    F = finfields.GF(P)
    ctx = mpyc_b200.context_for(P)
    va, vb = [(5 * i + 1) * (P // 7) % P for i in range(6)], [(i * i + 2) % P for i in range(4)] + [P - 1, 0]

    def limb(v, shape):
        return F.array(resident.LimbValue(ctx, codec.ints_to_limbs(v, ctx), shape), check=False)

    def plain(v, shape):
        return F.array(np.array(v, dtype=object).reshape(shape))
    pub = np.array([-1, P + 3, 2, 0, 5, 7], dtype=object)                # public ints: not canonical, not reduced
    cases = [(lambda mk: np.outer(mk(va, (6,)), mk(vb, (6,))), True), (lambda mk: np.outer(mk(va, (2, 3)), mk(vb, (3, 2))), True),
             (lambda mk: np.outer(mk(va, (6,)), plain(vb, (6,))), True), (lambda mk: np.outer(mk(va[:1], (1,)), mk(vb, (6,))), True),
             (lambda mk: np.outer(mk(va, (6,)), pub), False), (lambda mk: np.outer(pub, mk(vb, (6,))), False),
             (lambda mk: np.outer(mk(va, (6,)), 3), False)]
    want = [outcome(call(lambda: fn(plain))) for fn, _ in cases]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for i, ((fn, covered), w) in enumerate(zip(cases, want)):
            mat, ops = resident.calls['materialised'], resident.calls['limb_ops']
            r = call(lambda: fn(limb))
            if covered:
                assert resident.calls['materialised'] == mat and resident.calls['limb_ops'] > ops, i
            assert outcome(r) == w, i
            assert outcome(call(lambda: fn(plain))) == w, i
    finally:
        inst.uninstall()


def test_a_backend_without_k7_leaves_sums_to_the_reference(mpyc_mods, monkeypatch):
    """The CPU stand-in backend alone (no sum_axis / cumsum_axis): the reference's code answers, unchanged."""
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    oracle_device.patch(monkeypatch)
    oracle_device.patch_resident(monkeypatch)
    F = finfields.GF(P)
    ctx = mpyc_b200.context_for(P)
    vals = [(3 * i + 1) % P for i in range(12)]
    plain = F.array(np.array(vals, dtype=object).reshape(3, 4))
    calls = [lambda a: np.sum(a, axis=1), lambda a: a.sum(), lambda a: np.cumsum(a, axis=0),
             lambda a: np.cumulative_sum(a, axis=1, include_initial=True)]
    want = [outcome(call(lambda: fn(plain))) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for fn, w in zip(calls, want):
            a = F.array(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), (3, 4)), check=False)
            ops, packed = resident.calls['limb_ops'], resident.calls['packed']
            r = call(lambda: fn(a))
            assert resident.calls['limb_ops'] == ops and resident.calls['packed'] == packed
            assert outcome(r) == w
    finally:
        inst.uninstall()


def test_binary_fields_are_left_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import install as inst, resident
    import oracle_device
    oracle_device.patch(monkeypatch)
    oracle_device.patch_resident(monkeypatch)
    G = finfields.GF(gfpx.GFpX(2)(283))
    a = G.array(np.array([1, 2, 3, 0x53, 7, 9], dtype=object).reshape(2, 3))
    calls = [lambda: np.sum(a), lambda: np.sum(a, axis=0), lambda: a.sum(1), lambda: np.cumsum(a, axis=1),
             lambda: np.outer(a, a)]
    want = [outcome(call(fn)) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        ops = resident.calls['limb_ops']
        assert [outcome(call(fn)) for fn in calls] == want
        assert resident.calls['limb_ops'] == ops
    finally:
        inst.uninstall()


def test_axis_plans():
    from mpyc_b200 import axes
    assert axes.sum_plan((2, 3, 4), None) == ([(1, 24, 1)], ())
    assert axes.sum_plan((2, 3, 4), (0, 1), keepdims=True) == ([(1, 6, 4)], (1, 1, 4))
    # non-adjacent axes: one run at a time, the largest reduction first
    assert axes.sum_plan((2, 3, 4), (0, 2)) == ([(6, 4, 1), (1, 2, 3)], (3,))
    assert axes.sum_plan((5, 3), ()) == ([(15, 1, 1)], (5, 3))
    assert axes.sum_plan((), None) == ([(1, 1, 1)], ())
    assert axes.scan_plan((2, 3, 4), -2, True) == ((2, 3, 4), (2, 4, 4))
    assert axes.scan_plan((2, 3), None) == ((1, 6, 1), (6,))
    for bad in ((0, 0), 3, -4, 1.0, (True,)):
        with pytest.raises((TypeError, ValueError)):
            axes.sum_plan((2, 3, 4), bad)


def test_k7_abi_argument_errors():
    """Bad arguments are rejected before any CUDA call; valid ones without a device fail with a CUDA error."""
    import mpyc_b200
    from mpyc_b200._cabi import lib, check, u64_array
    torch = pytest.importorskip('torch')
    ctx = mpyc_b200.context_for(2**64 - 189)
    buf = ctypes.c_void_p(64)                                      # never dereferenced: every call below fails first
    with pytest.raises(ValueError):                                # null input
        check(lib.mpyc_b200_ff_sum_axis(ctx.handle, None, 2, 3, 4, None, buf, None))
    with pytest.raises(ValueError):                                # null output
        check(lib.mpyc_b200_ff_sum_axis(ctx.handle, buf, 2, 3, 4, None, None, None))
    with pytest.raises(ValueError):                                # size overflow
        check(lib.mpyc_b200_ff_sum_axis(ctx.handle, buf, 2**40, 2**20, 2**10, None, buf, None))
    with pytest.raises(ValueError):                                # initial not a canonical residue
        check(lib.mpyc_b200_ff_sum_axis(ctx.handle, buf, 2, 3, 4, u64_array([2**64 - 1]), buf, None))
    with pytest.raises(ValueError):
        check(lib.mpyc_b200_ff_sum_axis(None, buf, 2, 3, 4, None, buf, None))
    with pytest.raises(ValueError):
        check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, None, 2, 3, 4, 0, buf, None))
    with pytest.raises(ValueError):                                # len + 1 overflows
        check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, buf, 1, 2**64 - 1, 1, 1, buf, None))
    with pytest.raises(ValueError):
        check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, buf, 2**33, 2**33, 1, 0, buf, None))
    g = mpyc_b200.context_for(283, binary=True)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):           # prime fields only
        check(lib.mpyc_b200_ff_sum_axis(g.handle, buf, 2, 3, 4, None, buf, None))
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(lib.mpyc_b200_ff_cumsum_axis(g.handle, buf, 2, 3, 4, 0, buf, None))
    check(lib.mpyc_b200_ff_sum_axis(ctx.handle, None, 0, 3, 4, None, None, None))      # nothing to do
    check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, None, 2, 0, 4, 0, None, None))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(lib.mpyc_b200_ff_sum_axis(ctx.handle, buf, 2, 3, 4, None, buf, None))
    with pytest.raises(RuntimeError):
        check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, buf, 2, 3, 4, 1, buf, None))
