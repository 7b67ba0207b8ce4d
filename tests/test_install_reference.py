"""install() against the REAL reference (only where it is available, see oracle/reference.py):
attribute swap, pass-through for fields the engine does not cover, host-only helpers equal to the
reference's, and no silent CPU computation for covered fields."""
import sys

import pytest

from oracle import reference

REF = reference.path()
if REF is None:
    pytest.skip('reference not present ($MPYC_REFERENCE, or the copy build() makes in oracle/_ref)', allow_module_level=True)


@pytest.fixture(scope='module')
def mpyc_thresha():
    sys.dont_write_bytecode = True
    sys.path.insert(0, REF)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import thresha, finfields, gfpx
    finally:
        sys.argv = argv
    yield thresha, finfields, gfpx
    sys.path.remove(REF)


def test_install_swaps_and_restores(mpyc_thresha):
    thresha, finfields, gfpx = mpyc_thresha
    from mpyc_b200 import install as inst
    orig = {n: getattr(thresha, n) for n in inst._NAMES}
    names = inst.install(thresha)
    assert set(names) == set(inst._NAMES)
    assert all(getattr(getattr(thresha, n), '__mpyc_b200__', False) for n in names)
    inst.uninstall()
    assert all(getattr(thresha, n) is orig[n] for n in names)


def test_host_helpers_equal_reference_and_uncovered_fields_pass_through(mpyc_thresha):
    thresha, finfields, gfpx = mpyc_thresha
    from mpyc_b200 import install as inst
    ref_rv, ref_fsi = thresha._recombination_vector, thresha._f_S_i
    fields = [finfields.GF(p) for p in (19, 101, 2**61 - 1, 2**64 - 189, 2**69 - 93, 2**128 - 173, 2**256 - 189,
                                         9409569905028393239)]
    f256 = finfields.GF(gfpx.GFpX(2)(283))
    from itertools import combinations
    cases_rv = [(F, xs, x_r) for F in fields + [f256]
                for xs in ((1,), (1, 2, 3), (2, 3, 5), (1, 2, 3, 4, 5, 6, 7), tuple(range(1, 18))) for x_r in (0, 1, 18)
                if not (F.order == 19 and (len(xs) > 16 or x_r == 18))]
    cases_fs = [(F, m, i, S) for F in fields + [f256] for m, t in ((3, 1), (5, 2), (7, 3))
                for S in combinations(range(m), m - t) for i in S]
    want_rv = [ref_rv(F, xs, x_r) for F, xs, x_r in cases_rv]      # the unmodified reference, before install()
    want_fs = [ref_fsi(F, m, i, S) for F, m, i, S in cases_fs]
    inst.install(thresha)
    try:
        for (F, xs, x_r), want in zip(cases_rv, want_rv):
            assert thresha._recombination_vector(F, xs, x_r) == want
        for (F, m, i, S), want in zip(cases_fs, want_fs):
            got = thresha._f_S_i(F, m, i, S)
            if F is f256:
                assert got == want
            else:
                assert got % F.modulus == want % F.modulus
        # fields the engine does not cover run on the reference's own code, unchanged
        f2, f27 = finfields.GF(2), finfields.GF(gfpx.GFpX(3)(46))
        for F in (f2, f27):
            a = [F(0), F(1), F(1)]
            sh = thresha.random_split(F, a, 1, 3) if F is f27 else thresha.random_split(F, a, 0, 1)
            assert a == thresha.recombine(F, [(j + 1, sh[j]) for j in range(len(sh))])   # order as in tests/test_thresha.py:21
        # covered field, no GPU here: the call must fail loudly, never compute on the CPU
        import torch
        if not torch.cuda.is_available():
            with pytest.raises(RuntimeError):
                thresha.random_split(fields[2], [1, 2, 3], 1, 3)
    finally:
        inst.uninstall()


def test_finfields_hooks_installed_and_small_arrays_untouched(mpyc_thresha):
    """PrimeFieldArray's batched hot spots are swapped in; arrays below the size threshold (and per-element
    exponents) still run the reference's own code, so this part can be checked without a GPU."""
    thresha, finfields, gfpx = mpyc_thresha
    import numpy as np
    from mpyc_b200 import install as inst
    F = finfields.GF(2**61 - 1)
    a = F.array(np.array([1, 2, 3, 12345], dtype=object))
    want_inv, want_sqr = a.reciprocal().value.tolist(), a.is_sqr().tolist()
    orig = finfields.PrimeFieldArray.__dict__['_reciprocal']
    inst.install(thresha, finfields_module=finfields, finfields_min_size=100)
    try:
        assert finfields.PrimeFieldArray.__dict__['_reciprocal'] is not orig
        assert a.reciprocal().value.tolist() == want_inv          # 4 elements < 100: reference path
        assert a.is_sqr().tolist() == want_sqr
        assert (a ** np.array([1, 2, 3, 4], dtype=object)).value.tolist() == [1, 4, 27, pow(12345, 4, 2**61 - 1)]
        with pytest.raises(ZeroDivisionError):
            F.array(np.array([0, 1], dtype=object)).reciprocal()
    finally:
        inst.uninstall()
    assert finfields.PrimeFieldArray.__dict__['_reciprocal'] is orig


def test_share_rows_interoperate_with_the_reference_field_arrays(mpyc_thresha):
    """What runtime.py does with a received row over the limb wire (runtime.py:506-509): unmarshal = pickle.loads,
    then field.array(row, check=False).reshape(shape) -- with the REAL FiniteFieldArray, for a prime field and GF(2^8)."""
    import pickle
    import numpy as np
    thresha, finfields, gfpx = mpyc_thresha
    import mpyc_b200
    from mpyc_b200 import codec, wire
    p = 2**128 - 173
    F = finfields.GF(p)
    ctx = mpyc_b200.context_for(p)
    vals = [3, 1, 4, 1, 5, p - 1]
    row = pickle.loads(pickle.dumps(wire.ShareRow(ctx, codec.ints_to_limbs(vals, ctx))))
    a = F.array(row, check=False).reshape(2, 3)
    assert isinstance(a, F.array) and a.value.tolist() == [[3, 1, 4], [1, 5, p - 1]]
    assert ((a + a) * 2).value.tolist() == [[(4 * v) % p for v in r] for r in a.value.tolist()]     # ordinary field arithmetic afterwards
    f256 = finfields.GF(gfpx.GFpX(2)(283))
    ctx8 = mpyc_b200.context_for(283, binary=True)
    row8 = pickle.loads(pickle.dumps(wire.ShareRow(ctx8, np.array([0, 1, 0x53, 0xCA], dtype=np.uint8))))
    b = f256.array(row8, check=False)
    assert [int(v) for v in b.value] == [0, 1, 0x53, 0xCA]
    assert int((b * b).value[2]) == int((f256(0x53) * f256(0x53)).value)


def test_min_size_routes_small_calls_to_the_reference(mpyc_thresha):
    """install(min_size=n): calls on fewer elements run the reference's own code (no GPU needed here), larger ones go
    to the engine (which, without a GPU, must raise rather than compute)."""
    thresha, finfields, gfpx = mpyc_thresha
    from mpyc_b200 import install as inst
    F = finfields.GF(2**61 - 1)
    inst.install(thresha, min_size=8)
    try:
        a = [F(3), F(1), F(4)]
        sh = thresha.random_split(F, a, 1, 3)                      # 3 < 8 elements: reference path
        assert thresha.recombine(F, [(1, sh[0]), (2, sh[1])]) == a
        import torch
        if not torch.cuda.is_available():
            with pytest.raises(RuntimeError):
                thresha.random_split(F, [F(i) for i in range(8)], 1, 3)   # 8 >= 8: engine, no CPU fallback
    finally:
        inst.uninstall()


def test_install_sets_and_clears_the_limb_wire_flag(mpyc_thresha):
    thresha, finfields, gfpx = mpyc_thresha
    from mpyc_b200 import install as inst, thresha as engine
    assert engine.limb_wire is False
    inst.install(thresha, limb_wire=True)
    try:
        assert engine.limb_wire is True
    finally:
        inst.uninstall()
    assert engine.limb_wire is False


def test_coverage_is_decided_per_call_never_raises_where_the_reference_computes(mpyc_thresha, monkeypatch):
    """A covered field with an argument outside the kernels' range -- a PRF bound above 2^256, more than 64 recombination
    points -- is computed by the reference's own function (round 1 raised UnsupportedFieldError in the middle of
    runtime._convert).  strict=True keeps raising.  The device round trips are answered by the oracle here."""
    thresha, finfields, gfpx = mpyc_thresha
    import mpyc_b200
    from mpyc_b200 import install as inst
    import oracle_device
    oracle_device.patch(monkeypatch)
    F = finfields.GF(2**61 - 1)
    key = bytes(range(16))
    big = (1 << 300) + 7
    prfs = {(0,): thresha.PRF(key, big)}
    want = thresha.np_pseudorandom_share(F, 1, 0, prfs, b'uci', 9).value.tolist()
    want_l = [a.value for a in thresha.pseudorandom_share(F, 1, 0, prfs, b'uci', 9)]
    xs = list(range(1, 71))                                   # 70 points > MPYC_B200_MAX_POINTS
    rows = [[(x * 7 + h) % F.modulus for h in range(5)] for x in xs]
    want_rec = thresha.recombine(F, list(zip(xs, rows)))
    inst.install(thresha)
    try:
        assert thresha.np_pseudorandom_share(F, 1, 0, prfs, b'uci', 9).value.tolist() == want
        assert [a.value for a in thresha.pseudorandom_share(F, 1, 0, prfs, b'uci', 9)] == want_l
        got = thresha.recombine(F, list(zip(xs, rows)))
        assert [int(v) % F.modulus for v in got] == [int(v) % F.modulus for v in want_rec]
    finally:
        inst.uninstall()
    inst.install(thresha, strict=True)
    try:
        with pytest.raises(mpyc_b200.UnsupportedFieldError):
            thresha.np_pseudorandom_share(F, 1, 0, prfs, b'uci', 9)
    finally:
        inst.uninstall()


def test_limb_backed_field_arrays_keep_their_limbs_through_the_hooked_operators(mpyc_thresha, monkeypatch):
    """install(resident=True) on the reference's own finfields: << >> (+ in place), contiguous __getitem__, np.concatenate
    (axis 0), == / != with a scalar and + - * on limb-backed arrays give what the reference gives on object arrays, without
    turning the operands into Python ints; uninstall() restores every method."""
    thresha, finfields, gfpx = mpyc_thresha
    import numpy as np
    from mpyc_b200 import install as inst, resident, codec
    import mpyc_b200
    import oracle_device
    oracle_device.patch(monkeypatch)
    oracle_device.patch_resident(monkeypatch)
    p = 2**128 - 173
    F = finfields.GF(p)
    ctx = mpyc_b200.context_for(p)
    vals = [(7 * i * i + 3) % p for i in range(12)] + [0, p - 1]
    plain = F.array(np.array(vals, dtype=object).reshape(7, 2))
    before = {name: F.array.__mro__[2].__dict__.get(name) for name in ('__getitem__', '__eq__', '__lshift__')}
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=1)
    try:
        def limb():
            return F.array(resident.LimbValue(ctx, codec.ints_to_limbs(vals, ctx), (7, 2)), check=False)

        def backed(a):
            return resident.as_limb_value(resident.raw_value(a)) is not None
        start = resident.calls['materialised']
        pairs = [(limb() << 5, plain << 5), (limb() >> 3, plain >> 3), (limb()[2:5], plain[2:5]), (limb()[-1], plain[-1]),
                 (limb()[1:], plain[1:]), (np.concatenate((limb()[:1], limb()[3:]), axis=0), np.concatenate((plain[:1], plain[3:]), axis=0)),
                 (limb() * limb() + limb() - 5, plain * plain + plain - 5)]
        row = F.array(resident.LimbValue(ctx, codec.ints_to_limbs(vals[:2], ctx), (2,)), check=False)
        prow = F.array(np.array(vals[:2], dtype=object))
        pairs += [(limb() - row, plain - prow), (row - limb(), prow - plain), (limb() * row, plain * prow), (row + limb(), prow + plain)]
        x = limb()
        x <<= 2
        x >>= 7
        y = plain.copy()
        y <<= 2
        y >>= 7
        pairs.append((x, y))
        assert all(backed(g) for g, _ in pairs)
        assert resident.calls['materialised'] == start               # nothing became a Python int so far
        for g, w in pairs:
            assert g.shape == w.shape and [int(v) for v in g.value.reshape(-1)] == [int(v) for v in w.value.reshape(-1)]
        for k in (0, p - 1, vals[3], -1):
            assert ((limb() == k) == (plain == k)).all() and ((limb() != k) == (plain != k)).all()
        assert (limb() == 0).dtype == bool and (limb() == 0).shape == (7, 2)
        # selections that are not one contiguous run, and other axes, are the reference's business (object arrays)
        assert [int(v) for v in limb()[::2].value.reshape(-1)] == [int(v) for v in plain[::2].value.reshape(-1)]
        assert [int(v) for v in limb()[:, 1].value] == [int(v) for v in plain[:, 1].value]
        assert np.concatenate((limb(), limb()), axis=1).shape == (7, 4)
    finally:
        inst.uninstall()
    assert all(F.array.__mro__[2].__dict__.get(name) is fn for name, fn in before.items())
