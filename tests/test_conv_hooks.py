"""np.convolve behind install(operators=True) on the reference's own finfields (K10 through mpyc_b200.resident, answered
here by the CPU stand-in of tests/oracle_conv.py): every hooked form -- field x field and field x each public integer
form, in all three modes and both argument orders, the reference's own test_finfields cases among them -- equals the
uninstalled reference in kind, shape and value; the calls left to the reference reach it with its own result or error;
limb-backed inputs are never turned into Python ints and are not modified; a backend without K10 leaves np.convolve to
the reference.  Also the stand-in against tests/golden/conv.json and the argument errors of the K10 C-ABI entry point,
which need no GPU."""
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import pytest

from oracle import reference
from test_reduce_hooks import call, outcome

REF = reference.path()
HERE = os.path.dirname(os.path.abspath(__file__))
PRIMES = [2**61 - 1, 2**64 - 189, 9409569905028393239, 2**128 - 173, 0x80000004f1bbcdcbfa53e0af9ce60302e76e423f, 2**256 - 189]
_spec = importlib.util.spec_from_file_location('make_golden_conv', os.path.join(HERE, 'golden', 'make_golden_conv.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'conv.json')) as _fh:
    CASES = json.load(_fh)


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


def values(p):
    rng = np.random.default_rng(p % 1000)
    return {k: [int(v) % p for v in rng.integers(-2**62, 2**62, size=k)] for k in (1, 2, 3, 4, 5, 7, 9)}


def cases(p):
    """(name, covered, operand names, fn(*operands)); operand names 'f<k>' are field arrays of length k (limb-backed
    or plain), anything else a public operand built by public()"""
    out = []
    for m, n in ((1, 1), (1, 7), (7, 1), (2, 3), (3, 2), (4, 4), (5, 9), (9, 5)):
        for mode in ('full', 'same', 'valid'):
            out.append((f'ff_{m}x{n}_{mode}', True, [f'f{m}', f'f{n}'], lambda a, b, mode=mode: np.convolve(a, b, mode=mode)))
    out.append(('ff_mode_positional', True, ['f5', 'f3'], lambda a, b: np.convolve(a, b, 'same')))
    for form in ('list', 'tuple', 'range', 'int64', 'uint64', 'object', 'list_big'):
        for mode in ('full', 'same', 'valid'):
            out.append((f'{form}_right_{mode}', True, ['f5', form], lambda a, b, mode=mode: np.convolve(a, b, mode=mode)))
            out.append((f'{form}_left_{mode}', True, [form, 'f4'], lambda a, b, mode=mode: np.convolve(a, b, mode=mode)))
    # test_finfields.py's own cases: a slice that shares its store, lists, tuples, ranges, 'same' and 'valid'
    out += [('ref_slice', True, ['f7', 'f4'], lambda a, b: np.convolve(a[:-2], b)),
            ('ref_list', True, ['f7', 'ref_list'], lambda a, b: np.convolve(a, b)),
            ('ref_tuple', True, ['f7', 'ref_tuple'], lambda a, b: np.convolve(a, b)),
            ('ref_range', True, ['f7', 'ref_range'], lambda a, b: np.convolve(a, b)),
            ('ref_same', True, ['f7', 'f4'], lambda a, b: np.convolve(a, b, mode='same')),
            ('ref_valid', True, ['f7', 'f4'], lambda a, b: np.convolve(a, b, mode='valid'))]
    # left to the reference
    out += [('operand_keywords', False, ['f3', 'f5'], lambda a, b: np.convolve(v=b, a=a, mode='valid')),
            ('element', False, ['f5'], lambda a: np.convolve(a, type(a).field(3))),
            ('zero_d', False, ['f5'], lambda a: np.convolve(a, type(a)(np.array(4, dtype=object)))),
            ('two_d', False, ['f4', 'f4'], lambda a, b: np.convolve(a.reshape(2, 2), b)),
            ('empty', False, ['f5', 'empty'], lambda a, b: np.convolve(a, b)),
            ('empty_field', False, ['f5'], lambda a: np.convolve(a[:0], a)),
            ('int_mode', False, ['f5', 'f3'], lambda a, b: np.convolve(a, b, 1)),
            ('bad_mode', False, ['f5', 'f3'], lambda a, b: np.convolve(a, b, mode='bogus')),
            ('short_mode', False, ['f5', 'f3'], lambda a, b: np.convolve(a, b, mode='f')),
            ('float_list', False, ['f5', 'floats'], lambda a, b: np.convolve(a, b)),
            ('float_array', False, ['f5', 'float64'], lambda a, b: np.convolve(a, b)),
            ('bool_array', False, ['f5', 'bools'], lambda a, b: np.convolve(a, b)),
            ('bool_list', False, ['f5', 'bool_list'], lambda a, b: np.convolve(a, b)),
            ('complex_array', False, ['f5', 'complex'], lambda a, b: np.convolve(a, b)),
            ('two_d_public', False, ['f5', 'int2d'], lambda a, b: np.convolve(a, b))]
    return out


def is_field(k):
    return k[0] == 'f' and k[1:].isdigit()


def public(name, p):
    rng = np.random.default_rng(5)
    ints = [int(v) for v in rng.integers(-10**6, 10**6, size=3)]
    obj = np.empty(3, dtype=object)
    obj[:] = [p + 5, -p - 7, 3 * p**3 + 1]
    return {'list': ints, 'tuple': tuple(ints), 'range': range(2, 5), 'int64': np.array([-2**63, 2**63 - 1, -5], dtype=np.int64),
            'uint64': np.array([2**64 - 1, 0, 2**63 + 11], dtype=np.uint64), 'object': obj, 'list_big': [p, -1, 2 * p + 3, -p**2],
            'empty': [], 'floats': [1.5, 2.0], 'float64': np.array([1.0, 2.0]), 'bools': np.array([True, False]),
            'bool_list': [True, False, True], 'complex': np.array([1 + 2j]),
            'int2d': np.array([[1, 2], [3, 4]]), 'ref_list': [1, 2, 3], 'ref_tuple': (1, 2, 3), 'ref_range': range(3)}[name]


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_convolve_hooks_equal_the_reference(mpyc_mods, monkeypatch, p):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_conv
    oracle_device.patch(monkeypatch)
    oracle_conv.patch_resident(monkeypatch)
    F = finfields.GF(p).array
    ctx = mpyc_b200.context_for(p)
    data = values(p)

    def plain(k):
        return F(np.array(data[int(k[1:])], dtype=object)) if is_field(k) else public(k, p)

    def limb(k):
        if not is_field(k):
            return public(k, p)
        v = data[int(k[1:])]
        return F(resident.LimbValue(ctx, codec.ints_to_limbs(v, ctx), (len(v),)), check=False)
    table = cases(p)
    want = [outcome(call(lambda: fn(*[plain(k) for k in ks]))) for _, _, ks, fn in table]
    assert sum(w[0] == 'raises' for w in want) >= 5
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for (name, covered, ks, fn), w in zip(table, want):
            args = [limb(k) for k in ks]
            mat, ops, packed = resident.calls['materialised'], resident.calls['limb_ops'], resident.calls['packed']
            r = call(lambda: fn(*args))
            if covered:
                assert resident.calls['materialised'] == mat, name
                assert resident.calls['limb_ops'] > ops, name
                assert resident.calls['packed'] == packed + sum(not is_field(k) for k in ks), name
                assert type(resident.raw_value(r)) is resident.LimbValue, name
            elif name != 'operand_keywords':  # the reference's code: it reads .value, which settles a limb-backed input
                assert resident.calls['materialised'] > mat, name
            assert outcome(r) == w, (name, outcome(r), w)
            if covered:
                assert outcome(call(lambda: fn(*[plain(k) for k in ks]))) == w, name      # plain arrays: packed
        a, b = limb('f5'), limb('f3')                                                   # inputs stay as they were
        before = outcome(a), outcome(b)
        np.convolve(a, b)
        np.convolve(b, a, mode='valid')
        assert (outcome(a), outcome(b)) == before
    finally:
        inst.uninstall()


def test_small_object_arrays_and_binary_fields_stay_with_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_conv
    oracle_device.patch(monkeypatch)
    oracle_conv.patch_resident(monkeypatch)
    F = finfields.GF(2**127 - 1).array
    G = finfields.GF(gfpx.GFpX(2)(283)).array
    H = finfields.GF(2**61 - 1).array
    calls = [lambda: np.convolve(F(np.array([1, 2, 3], dtype=object)), F(np.array([4, 5], dtype=object))),
             lambda: np.convolve(F(np.array([1, 2, 3], dtype=object)), [4, 5]),
             lambda: np.convolve(G(np.array([1, 2, 3], dtype=object)), G(np.array([4, 5], dtype=object))),
             lambda: np.convolve(G(np.array([1, 2, 3], dtype=object)), [4, 5], mode='same'),
             lambda: np.convolve(F(np.array([1, 2, 3], dtype=object)), H(np.array([4, 5], dtype=object)))]
    want = [outcome(call(fn)) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1024)
    try:
        for fn, w in zip(calls, want):
            ops = resident.calls['limb_ops']
            assert outcome(call(fn)) == w
            assert resident.calls['limb_ops'] == ops
    finally:
        inst.uninstall()


def test_other_field_and_binary_limb_arrays_stay_with_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_conv
    oracle_device.patch(monkeypatch)
    oracle_conv.patch_resident(monkeypatch)
    P, Q = 2**127 - 1, 2**61 - 1
    F, H = finfields.GF(P).array, finfields.GF(Q).array
    G = finfields.GF(gfpx.GFpX(2)(283)).array
    fv, hv, gv = [3, 1, 4, 1, 5], [9, 2, 6], [7, 0, 1, 200]
    want = [outcome(call(lambda: np.convolve(F(np.array(fv, dtype=object)), H(np.array(hv, dtype=object))))),
            outcome(call(lambda: np.convolve(G(np.array(gv, dtype=object)), G(np.array(gv[:2], dtype=object)))))]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        ctx_f, ctx_h = mpyc_b200.context_for(P), mpyc_b200.context_for(Q)
        a = F(resident.LimbValue(ctx_f, codec.ints_to_limbs(fv, ctx_f), (5,)), check=False)
        b = H(resident.LimbValue(ctx_h, codec.ints_to_limbs(hv, ctx_h), (3,)), check=False)
        mat = resident.calls['materialised']
        assert outcome(call(lambda: np.convolve(a, b))) == want[0]
        assert resident.calls['materialised'] > mat          # the reference's code read a's values
        ops = resident.calls['limb_ops']
        g = G(np.array(gv, dtype=object))
        assert outcome(call(lambda: np.convolve(g, g[:2]))) == want[1]
        assert resident.calls['limb_ops'] == ops
    finally:
        inst.uninstall()


def test_a_backend_without_k10_leaves_convolve_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_linalg
    oracle_device.patch(monkeypatch)
    oracle_linalg.patch_resident(monkeypatch)                          # K7, K8 and K9 but no K10
    P = 2**128 - 173
    F = finfields.GF(P).array
    ctx = mpyc_b200.context_for(P)
    vals = [(5 * i * i + 3) % P for i in range(6)]
    calls = [lambda a: np.convolve(a, a), lambda a: np.convolve(a, [1, -2, 3], mode='same'),
             lambda a: np.convolve(range(4), a, mode='valid')]
    want = [outcome(call(lambda: fn(F(np.array(vals, dtype=object))))) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for fn, w in zip(calls, want):
            a = F(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), (6,)), check=False)
            mat = resident.calls['materialised']
            r = call(lambda: fn(a))
            assert resident.calls['materialised'] > mat
            assert outcome(r) == w
    finally:
        inst.uninstall()


def window(m, n, mode):
    s, g = min(m, n), max(m, n)
    return {'full': (0, m + n - 1), 'same': ((s - 1) // 2, g), 'valid': (s - 1, g - s + 1)}[mode]


def case_operands(c):
    p = int(c['p'], 16)
    return p, [gold.operand(p, length, form, c['seed'] + k) for k, (length, form) in enumerate(zip((c['m'], c['n']), c['forms']))]


def expected(c, vals):
    return [hex(v) for v in vals] if c['len'] <= gold.STORE_LIMIT else gold.digest(vals)


def test_stand_in_reproduces_the_golden_fixtures():
    """tests/oracle_conv.py's definition on every conv.json case up to 20000 products (the rest are replayed on the GPU)."""
    import oracle_conv
    assert len(CASES) > 600
    done = 0
    for c in CASES:
        if c['m'] * c['n'] > 20000:
            continue
        p, (a, b) = case_operands(c)
        lo, count = window(c['m'], c['n'], c['mode'])
        assert count == c['len']
        a, b = [int(v) % p for v in a], [int(v) % p for v in b]
        assert expected(c, oracle_conv.convolve_ints(a, b, lo, count, p)) == c['result'], c
        done += 1
    assert done > 500


def test_golden_fixtures_through_the_hook(mpyc_mods, monkeypatch):
    """The small conv.json cases through install's np.convolve hook on the stand-in: operands limb-backed where they are
    field arrays, the public forms as generated."""
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_conv
    oracle_device.patch(monkeypatch)
    oracle_conv.patch_resident(monkeypatch)
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for c in CASES:
            if c['m'] * c['n'] > 2000:
                continue
            p, ops = case_operands(c)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            ops = [F(resident.LimbValue(ctx, codec.ints_to_limbs(x, ctx), (len(x),)), check=False) if form in ('field', 'max') else x
                   for x, form in zip(ops, c['forms'])]
            ops_before = resident.calls['limb_ops']
            r = np.convolve(ops[0], ops[1], mode=c['mode'])
            assert resident.calls['limb_ops'] > ops_before
            assert expected(c, [int(v) for v in np.asarray(r.value, dtype=object)]) == c['result'], c
    finally:
        inst.uninstall()


def test_k10_abi_argument_errors():
    """Empty operands, windows past the full result, sizes that overflow and overlapping buffers are rejected before any
    CUDA call; a valid call without a device fails with a CUDA error."""
    import mpyc_b200
    from mpyc_b200._cabi import lib, check
    torch = pytest.importorskip('torch')
    ctx = mpyc_b200.context_for(2**128 - 173)                  # 16-byte elements
    a, b, c = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 24), ctypes.c_void_p(1 << 30)   # never dereferenced
    big = 1 << 62
    for bad in [lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 0, b, 4, 0, 1, c, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 0, 0, 1, c, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 0, 7, c, None),        # 6 outputs
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 6, 1, c, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 7, 0, c, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 2**64 - 1, 2, c, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, big, b, big, 0, 1, c, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 2**64 - 1, b, 2, 0, 1, c, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 0, 6, ctypes.c_void_p((1 << 20) + 16 * 3), None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 0, 6, ctypes.c_void_p((1 << 24) - 16 * 5), None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 0, 6, a, None),
                lambda: lib.mpyc_b200_ff_convolve(ctx.handle, None, 4, b, 3, 0, 6, c, None)]:
        with pytest.raises(ValueError):
            check(bad())
    check(lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 6, 0, c, None))         # count == 0: nothing to do
    g = mpyc_b200.context_for(283, binary=True)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(lib.mpyc_b200_ff_convolve(g.handle, a, 4, b, 3, 0, 6, c, None))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(lib.mpyc_b200_ff_convolve(ctx.handle, a, 4, b, 3, 0, 6, c, None))
