"""np.linalg.det / solve / inv / matrix_power behind install(operators=True) on the reference's own finfields (K9 and K1c
through mpyc_b200.resident, answered here by the CPU stand-in of tests/oracle_linalg.py, which restates the kernels'
division-free algorithm): every result equals the uninstalled reference's in kind, shape and value -- the determinant's
sign rule for row swaps included -- errors are the reference's, limb-backed inputs are never turned into Python ints,
the calls left to the reference reach it, and a backend without K9 leaves everything to the reference.  Also the argument
errors of the two K9 C-ABI entry points, which need no GPU."""
import ctypes
import sys

import numpy as np
import pytest

from oracle import reference
from test_reduce_hooks import call, outcome

REF = reference.path()
PRIMES = [2**61 - 1, 2**64 - 189, 9409569905028393239, 2**128 - 173, 0x80000004f1bbcdcbfa53e0af9ce60302e76e423f, 2**256 - 189]


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


def matrices(p):
    """name -> list of values and shape: random, swap-forcing, singular and the reference's documented oddities"""
    rng = np.random.default_rng(p % 1000)

    def rand(*shape):
        return [int(v) % p for v in rng.integers(-2**62, 2**62, size=shape).reshape(-1)], shape
    swaps = [[0, 1, 2, 3], [0, 0, 4, 5], [6, 7, 8, 9], [1, 2, 3, 5]]        # zero pivots at steps 0 and 1
    out = {
        'r1': rand(1, 1), 'r2': rand(2, 2), 'r3': rand(3, 3), 'r5': rand(5, 5), 'r8': rand(8, 8),
        'swap2': ([0, 1, 1, 0], (2, 2)), 'swap4': ([v % p for r in swaps for v in r], (4, 4)),
        'zero_col': ([1, 0, 3, 4, 0, 6, 7, 0, 9], (3, 3)), 'dep_rows': ([1, 2, 3, 2, 4, 6, 5, 7, 9], (3, 3)),
        'late_singular': ([1, 2, 3, 4, 5, 6, 7, 8, 9], (3, 3)), 'zero1': ([0], (1, 1)),
        'stack_doc': ([0, 1, 2, 3, 4, 5, 6, 7], (2, 2, 2)), 'stack3': rand(2, 3, 3, 3), 'stack1': rand(4, 1, 1),
        'neg': ([(-v) % p for v in range(1, 10)], (3, 3)),
    }
    return out


def cases(p):
    """(name, covered, builder names, fn(*arrays))"""
    m = matrices(p)
    out = []
    for k in m:
        out.append((f'det_{k}', True, [k], lambda a: np.linalg.det(a)))
    for k in ('r1', 'r3', 'r8', 'swap4', 'swap2'):
        out.append((f'inv_{k}', True, [k], lambda a: np.linalg.inv(a)))
        for e in (-5, 0, 1, 3):
            out.append((f'pow{e}_{k}', True, [k], lambda a, e=e: np.linalg.matrix_power(a, e)))
    out += [('inv_singular', True, ['dep_rows'], lambda a: np.linalg.inv(a)),
            ('inv_late_singular', True, ['late_singular'], lambda a: np.linalg.inv(a)),
            ('pow_neg_singular', True, ['zero_col'], lambda a: np.linalg.matrix_power(a, -2)),
            ('pow0_singular', True, ['zero_col'], lambda a: np.linalg.matrix_power(a, 0)),
            ('solve_r3', True, ['r3', 'b3x2'], lambda a, b: np.linalg.solve(a, b)),
            ('solve_swap4', True, ['swap4', 'b4x1'], lambda a, b: np.linalg.solve(a, b)),
            ('pow_kw', True, ['r3'], lambda a: np.linalg.matrix_power(a, n=3)),
            ('det_kw', True, ['r3'], lambda a: np.linalg.det(a=a)),
            ('solve_singular', True, ['zero_col', 'b3x2'], lambda a, b: np.linalg.solve(a, b)),
            # left to the reference
            ('solve_numpy_kw', False, ['r3', 'b3x2'], lambda a, b: np.linalg.solve(a=a, b=b)),
            ('det_rect', False, ['rect'], lambda a: np.linalg.det(a)), ('det_1d', False, ['vec3'], lambda a: np.linalg.det(a)),
            ('det_empty', False, ['empty'], lambda a: np.linalg.det(a)),
            ('inv_stack', False, ['stack3'], lambda a: np.linalg.inv(a)), ('inv_rect', False, ['rect'], lambda a: np.linalg.inv(a)),
            ('solve_vec', False, ['r3', 'vec3'], lambda a, b: np.linalg.solve(a, b)),
            ('solve_rows', False, ['r3', 'b4x1'], lambda a, b: np.linalg.solve(a, b)),
            ('pow_np_int', False, ['r3'], lambda a: np.linalg.matrix_power(a, np.int64(2)))]
    return out


def builders(p):
    m = matrices(p)
    rng = np.random.default_rng(7)
    extra = {'b3x2': ([int(v) % p for v in rng.integers(0, 2**62, size=6)], (3, 2)),
             'b4x1': ([int(v) % p for v in rng.integers(0, 2**62, size=4)], (4, 1)),
             'rect': (list(range(1, 7)), (2, 3)), 'vec3': ([1, 2, 3], (3,)), 'empty': ([], (0, 0))}
    return dict(m, **extra)


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_linalg_hooks_equal_the_reference(mpyc_mods, monkeypatch, p):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_linalg
    oracle_device.patch(monkeypatch)
    oracle_linalg.patch_resident(monkeypatch)
    F = finfields.GF(p).array
    ctx = mpyc_b200.context_for(p)
    data = builders(p)

    def plain(k):
        v, shape = data[k]
        return F(np.array(v, dtype=object).reshape(shape))

    def limb(k):
        v, shape = data[k]
        return F(resident.LimbValue(ctx, codec.ints_to_limbs(v, ctx), shape), check=False)
    table = cases(p)
    want = [outcome(call(lambda: fn(*[plain(k) for k in ks]))) for _, _, ks, fn in table]
    assert sum(w[0] == 'raises' for w in want) >= 12
    assert want[[t[0] for t in table].index('det_swap2')] == ('element', F.field.__name__, 1)
    assert want[[t[0] for t in table].index('det_stack_doc')][3] == [2, p - 2]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for (name, covered, ks, fn), w in zip(table, want):
            args = [limb(k) for k in ks]
            mat, ops = resident.calls['materialised'], resident.calls['limb_ops']
            r = call(lambda: fn(*args))
            if covered:
                assert resident.calls['materialised'] == mat, name
                assert resident.calls['limb_ops'] > ops or r[0] == 'raises', name
            else:                            # the reference's code: it reads .value, which settles a limb-backed input
                assert resident.calls['limb_ops'] == ops, name
            assert outcome(r) == w, (name, outcome(r), w)
            if covered:
                assert outcome(call(lambda: fn(*[plain(k) for k in ks]))) == w, name      # plain arrays: packed
            if name == 'solve_r3':                                                      # a plain b with a limb-backed a
                packed = resident.calls['packed']
                assert outcome(call(lambda: fn(limb(ks[0]), plain(ks[1])))) == w
                assert resident.calls['packed'] == packed + 1
        a = limb('r3')                                                                  # inputs stay as they were
        before = outcome(a)
        np.linalg.inv(limb('r3'))
        np.linalg.det(a)
        assert outcome(a) == before
    finally:
        inst.uninstall()


def test_small_object_arrays_and_binary_fields_stay_with_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import install as inst, resident
    import oracle_device
    import oracle_linalg
    oracle_device.patch(monkeypatch)
    oracle_linalg.patch_resident(monkeypatch)
    F = finfields.GF(2**127 - 1).array
    G = finfields.GF(gfpx.GFpX(2)(283)).array
    calls = [lambda: np.linalg.det(F(np.array([[1, 2], [3, 4]], dtype=object))),
             lambda: np.linalg.inv(F(np.array([[1, 2], [3, 4]], dtype=object))),
             lambda: np.linalg.det(G(np.array([[1, 2], [3, 4]], dtype=object))),
             lambda: np.linalg.inv(G(np.array([[1, 2], [3, 4]], dtype=object)))]
    want = [outcome(call(fn)) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1024)
    try:
        for fn, w in zip(calls, want):
            ops = resident.calls['limb_ops']
            assert outcome(call(fn)) == w
            assert resident.calls['limb_ops'] == ops
    finally:
        inst.uninstall()


def test_a_backend_without_k9_leaves_linalg_to_the_reference(mpyc_mods, monkeypatch):
    thresha, finfields, gfpx = mpyc_mods
    import mpyc_b200
    from mpyc_b200 import install as inst, resident, codec
    import oracle_device
    import oracle_layout
    oracle_device.patch(monkeypatch)
    oracle_layout.patch_resident(monkeypatch)                          # K7 and K8 but no K9
    P = 2**128 - 173
    F = finfields.GF(P).array
    ctx = mpyc_b200.context_for(P)
    vals = [(5 * i * i + 3) % P for i in range(9)]
    calls = [lambda a: np.linalg.det(a), lambda a: np.linalg.inv(a), lambda a: np.linalg.matrix_power(a, 3),
             lambda a: np.linalg.solve(a, a)]
    want = [outcome(call(lambda: fn(F(np.array(vals, dtype=object).reshape(3, 3))))) for fn in calls]
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for fn, w in zip(calls, want):
            a = F(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), (3, 3)), check=False)
            mat = resident.calls['materialised']
            r = call(lambda: fn(a))
            assert resident.calls['materialised'] > mat
            assert outcome(r) == w
    finally:
        inst.uninstall()


def test_k9_abi_argument_errors():
    """Bad sizes and overlapping buffers are rejected before any CUDA call; valid ones without a device fail with a CUDA
    error."""
    import mpyc_b200
    from mpyc_b200._cabi import lib, check
    torch = pytest.importorskip('torch')
    ctx = mpyc_b200.context_for(2**128 - 173)                  # 16-byte elements
    a, b = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 30)  # never dereferenced: every call below fails first
    big = 1 << 40
    for bad in [lambda: lib.mpyc_b200_ff_det(ctx.handle, a, 1, 0, b, None),
                lambda: lib.mpyc_b200_ff_det(ctx.handle, a, big, big, b, None),
                lambda: lib.mpyc_b200_ff_det(ctx.handle, a, 2, 4, ctypes.c_void_p((1 << 20) + 16 * 31), None),
                lambda: lib.mpyc_b200_ff_det(ctx.handle, None, 2, 4, b, None),
                lambda: lib.mpyc_b200_ff_solve(ctx.handle, a, 0, None, 0, b, None),
                lambda: lib.mpyc_b200_ff_solve(ctx.handle, a, big, None, big, b, None),
                lambda: lib.mpyc_b200_ff_solve(ctx.handle, a, 4, None, 3, b, None),
                lambda: lib.mpyc_b200_ff_solve(ctx.handle, a, 4, b, 2, ctypes.c_void_p((1 << 30) + 16), None),
                lambda: lib.mpyc_b200_ff_solve(ctx.handle, a, 4, None, 4, ctypes.c_void_p((1 << 20) + 16 * 15), None)]:
        with pytest.raises(ValueError):
            check(bad())
    check(lib.mpyc_b200_ff_det(ctx.handle, a, 0, 4, b, None))                     # an empty stack: nothing to do
    g = mpyc_b200.context_for(283, binary=True)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(lib.mpyc_b200_ff_det(g.handle, a, 1, 2, b, None))
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        check(lib.mpyc_b200_ff_solve(g.handle, a, 2, None, 2, b, None))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError):
        check(lib.mpyc_b200_ff_det(ctx.handle, a, 1, 4, b, None))


def test_stand_in_algorithm_reproduces_the_golden_fixtures():
    """The restated algorithm on tests/golden/linalg.json's cases up to n = 33 (the larger ones are replayed on the GPU)."""
    import importlib.util
    import json
    import os
    import oracle_linalg
    here = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location('make_golden_linalg', os.path.join(here, 'golden', 'make_golden_linalg.py'))
    gold = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gold)
    with open(os.path.join(here, 'golden', 'linalg.json')) as fh:
        cases = json.load(fh)
    assert len(cases) > 500
    for c in cases:
        p, n = int(c['p'], 16), c['n']
        if n > 33:
            continue
        mats = [[v for r in gold.matrix(p, n, k, c['seed'] + 100 * j) for v in r] for j, k in enumerate(c['kinds'])]
        try:
            if c['op'] == 'det':
                got = [str(oracle_linalg.det_ints(m, n, p)) for m in mats]
            elif c['op'] == 'inv':
                got = gold.digest(oracle_linalg.solve_ints(mats[0], n, None, n, p))
            elif c['op'] == 'solve':
                B = [v for r in gold.rhs(p, n, c['nrhs'], c['seed']) for v in r]
                got = gold.digest(oracle_linalg.solve_ints(mats[0], n, B, c['nrhs'], p))
            else:
                continue
        except ZeroDivisionError:
            got = 'ZeroDivisionError'
        assert got == c['result'], c


def test_stand_in_algorithm_matches_textbook_determinant_up_to_swap_sign():
    """The restated algorithm against a Leibniz expansion: |det| agrees with the signed determinant up to the sign of the
    swap permutation the reference's pivot rule makes (none for a matrix without zero pivots)."""
    from itertools import permutations
    import oracle_linalg
    p = 2**61 - 1
    rng = np.random.default_rng(3)
    for n in (1, 2, 3, 4):
        v = [int(x) for x in rng.integers(1, 2**60, size=n * n)]
        leib = 0
        for perm in permutations(range(n)):
            sgn = 1
            for i in range(n):
                for j in range(i + 1, n):
                    if perm[i] > perm[j]:
                        sgn = -sgn
            term = sgn
            for i in range(n):
                term *= v[i * n + perm[i]]
            leib += term
        assert oracle_linalg.det_ints(v, n, p) == leib % p
        X = oracle_linalg.solve_ints(v, n, None, n, p)
        A = np.array(v, dtype=object).reshape(n, n)
        assert ((A @ np.array(X, dtype=object).reshape(n, n)) % p == np.eye(n, dtype=object)).all()
