"""K13 on the GPU: k_prod_*, k_cumprod_* and k_allany_*.  The golden fixtures (tests/golden/prod.json, the unmodified
reference's values, result types and errors) through install's hooks and the C ABI; for every limb count and reduction
kind prod(a) prod(b) = prod(a b) and cumprod(a)[-1] = prod(a) at 10^7 elements, running products against Python ints on
sampled columns, all / any with zeros planted first, last and inside slices, shapes on both sides of each form's split
decision, and operands that start mid-allocation (8-byte alignment only)."""
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import device as dev                # noqa: E402
from mpyc_b200._cabi import lib, check             # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from oracle import reference                       # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden_prod', os.path.join(HERE, 'golden', 'make_golden_prod.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'prod.json')) as _fh:
    FIXTURES = json.load(_fh)

# (p, limbs, kind): every limb count with each reduction kind (1: pseudo-Mersenne aligned, 2: shifted, 0: generic)
CELLS = [(2**61 - 1, 1, 2), (2**64 - 189, 1, 1), (9409569905028393239, 1, 0),
         (2**127 - 1, 2, 2), (2**128 - 173, 2, 1), (0xd1b54a32d192ed03a5c2a0c9b1f0e7ed, 2, 0),
         (2**189 - 25, 3, 2), (2**192 - 237, 3, 1), (gold.P192, 3, 0),
         (2**255 - 19, 4, 2), (2**256 - 189, 4, 1), (2**256 - 2**32 - 977, 4, 0)]
BIG = 10**7


def cell_id(c):
    return f'L{c[1]}k{c[2]}'


def ctx_of(cell):
    p, L, kind = cell
    ctx = mpyc_b200.context_for(p)
    assert (ctx.nlimbs, ctx.kind) == (L, kind)
    return ctx


def ints(a):
    return [int(v) for v in a.to_ints()]


def host_prod(p, vals, shape, axis):
    x = np.array(vals, dtype=object).reshape(shape)
    return [int(v) for v in np.reshape(np.frompyfunc(lambda a, b: a * b % p, 2, 1).reduce(x, axis=axis, initial=1), -1)]


def host_cumprod(p, vals, shape, axis):
    x = np.array(vals, dtype=object).reshape(shape)
    return [int(v) for v in np.reshape(np.frompyfunc(lambda a, b: a * b % p, 2, 1).accumulate(x, axis=axis, dtype=object), -1)]


def host_all_any(vals, shape, axis, any):
    x = np.array(vals, dtype=object).reshape(shape) != 0
    return [int(v) for v in np.reshape((np.any if any else np.all)(x, axis=axis), -1)]


@pytest.fixture(scope='module')
def mpyc_mods():
    path = reference.path()
    if path is None:
        pytest.skip('reference not present')
    sys.dont_write_bytecode = True
    sys.path.insert(0, path)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import thresha, finfields
    finally:
        sys.argv = argv
    yield thresha, finfields
    sys.path.remove(path)


def test_fixtures_through_the_hooks(mpyc_mods):
    """Every fixture on limb-backed operands in HBM (CudaBackend): the reference's values, types and errors, one K13 call
    per case without an error and nothing settled."""
    thresha, finfields = mpyc_mods
    from mpyc_b200 import install as inst, resident
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=1)
    try:
        for c in FIXTURES:
            p = int(c['p'], 16)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            d, fn = gold.CASES[c['case']]
            vals = gold.values(p, d)
            x = F(resident.LimbValue(ctx, DeviceArray.from_ints(ctx, vals), gold.SHAPES[d]), check=False)
            mat, k13 = resident.calls['materialised'], resident.calls['prod']
            try:
                r = fn(F, x)
            except Exception as e:   # noqa: BLE001
                assert 'error' in c and [type(e).__name__, str(e)] == c['error'], c['case']
                continue
            assert 'error' not in c, c['case']
            assert resident.calls['materialised'] == mat and resident.calls['prod'] == k13 + 1, c['case']
            if c['kind'] == 'bool':
                assert r is (np.True_ if c['bool'] else np.False_), c['case']
            got = gold.encode(r)
            assert got == {k: v for k, v in c.items() if k not in ('p', 'case')}, c['case']
    finally:
        inst.uninstall()


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_product_identities_at_1e7(cell):
    """prod(a) prod(b) = prod(a b) over 10^7 elements (rows form, split), the same as a (10^4, 10^3) array reduced along
    axis 0 then 1 (columns form, split), and the last running product equals the product."""
    ctx = ctx_of(cell)
    a, b = DeviceArray.random(ctx, BIG, 11), DeviceArray.random(ctx, BIG, 12)
    pa = ints(dev.prod_axis(a, (BIG,))[0])[0]
    pb = ints(dev.prod_axis(b, (BIG,))[0])[0]
    pab = ints(dev.prod_axis(a * b, (BIG,))[0])[0]
    assert pa * pb % ctx.modulus == pab
    cols, _ = dev.prod_axis(a, (10**4, 10**3), axis=0)
    assert ints(dev.prod_axis(cols, (10**3,))[0])[0] == pa
    run, shape = dev.cumprod_axis(a, (BIG,))
    assert shape == (BIG,) and ints(DeviceArray(ctx, run.t[BIG - 1:]))[0] == pa
    run, shape = dev.cumprod_axis(a, (10**4, 10**3), axis=0, include_initial=True)
    last = ints(DeviceArray(ctx, run.t[10**4 * 10**3:]))
    assert shape == (10**4 + 1, 10**3) and len(last) == 10**3 and ints(dev.prod_axis(DeviceArray.from_ints(ctx, last), (10**3,))[0])[0] == pa


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_running_products_on_sampled_columns(cell):
    """Split running products in both forms against Python ints: every column of a sample, every row."""
    ctx = ctx_of(cell)
    p = ctx.modulus
    for shape, axis in (((4000, 40), 0), ((3, 5000, 7), 1), ((2, 3, 33), 2)):
        n = int(np.prod(shape))
        a = DeviceArray.random(ctx, n, 21)
        vals = ints(a)
        got = np.array(ints(dev.cumprod_axis(a, shape, axis=axis)[0]), dtype=object).reshape(shape)
        x = np.array(vals, dtype=object).reshape(shape)
        for idx in list(np.ndindex(*(s for k, s in enumerate(shape) if k != axis)))[::5][:8]:
            sl = list(idx)
            sl.insert(axis, slice(None))
            acc, want = 1, []
            for v in x[tuple(sl)]:
                acc = acc * int(v) % p
                want.append(acc)
            assert list(got[tuple(sl)]) == want, (shape, idx)


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_all_any_with_planted_zeros(cell):
    """Columns with a zero first, last, inside and in the middle of R, and none, in both forms, split and not."""
    ctx = ctx_of(cell)
    for shape, axis in (((4096, 64), 0), ((3, 9000, 5), 1), ((50, 40), 0)):
        n = int(np.prod(shape))
        vals = [v or 1 for v in ints(DeviceArray.random(ctx, n, 31))]
        x = np.array(vals, dtype=object).reshape(shape)
        R = shape[axis]
        for j, r in enumerate((0, R - 1, min(64, R - 2), R // 2 + 1, 1)):
            sl = [0] * len(shape)
            sl[axis] = r
            sl[-1 if axis != len(shape) - 1 else 0] = j
            x[tuple(sl)] = 0
        vals = [int(v) for v in x.reshape(-1)]
        a = DeviceArray.from_ints(ctx, vals)
        for any_ in (False, True):
            got = ints(dev.all_any_axis(a, shape, axis=axis, any=any_)[0])
            assert got == host_all_any(vals, shape, axis, any_), (shape, any_)
            assert set(got) <= {0, 1}


# (shape, axis) on both sides of prod_plan's split (unsplit: R < 128 for columns, R * I < 2048 for rows) and of the form
# decision (columns for I >= 32 and for R * I < 32)
SPLIT_SHAPES = [((63, 32), 0), ((640, 32), 0), ((33, 31), 0), ((2000, 31), 0), ((1, 70, 1), 1), ((1, 5000, 1), 1),
                ((999, 7, 3), 1), ((4000, 31, 1), 1), ((3, 32, 1), 1)]


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_both_sides_of_the_split(cell):
    ctx = ctx_of(cell)
    p = ctx.modulus
    for shape, axis in SPLIT_SHAPES:
        n = int(np.prod(shape))
        a = DeviceArray.random(ctx, n, 41)
        vals = ints(a)
        init = p - 2
        want = [v * init % p for v in host_prod(p, vals, shape, axis)]
        assert ints(dev.prod_axis(a, shape, axis=axis, initial=init)[0]) == want, shape
        assert ints(dev.cumprod_axis(a, shape, axis=axis)[0]) == host_cumprod(p, vals, shape, axis), shape
        assert ints(dev.all_any_axis(a, shape, axis=axis)[0]) == host_all_any(vals, shape, axis, False), shape


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_mid_buffer_views(cell):
    """Operands and outputs that start one element into an allocation (8-byte aligned, not 16)."""
    ctx = ctx_of(cell)
    p = ctx.modulus
    shape = (300, 40)
    n = shape[0] * shape[1]
    base = DeviceArray.random(ctx, n + 1, 51)
    a = DeviceArray(ctx, base.t[1:])
    vals = ints(a)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = DeviceArray.empty(ctx, n + 2 + 1)
    dst = DeviceArray(ctx, out.t[1:])
    for axis in (0, 1):
        O, R, I = (1, shape[0], shape[1]) if axis == 0 else (shape[0], shape[1], 1)
        check(lib.mpyc_b200_ff_prod_axis(ctx.handle, a.ptr, O, R, I, None, dst.ptr, stream))
        assert ints(DeviceArray(ctx, dst.t[:O * I])) == host_prod(p, vals, shape, axis)
        check(lib.mpyc_b200_ff_cumprod_axis(ctx.handle, a.ptr, O, R, I, 0, dst.ptr, stream))
        assert ints(DeviceArray(ctx, dst.t[:n])) == host_cumprod(p, vals, shape, axis)
        check(lib.mpyc_b200_ff_all_any_axis(ctx.handle, a.ptr, O, R, I, 1, dst.ptr, stream))
        assert ints(DeviceArray(ctx, dst.t[:O * I])) == host_all_any(vals, shape, axis, True)


def test_abi_rejects_overlap_on_the_device():
    ctx = mpyc_b200.context_for(2**127 - 1)
    a = DeviceArray.random(ctx, 64, 1)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    with pytest.raises(ValueError):
        check(lib.mpyc_b200_ff_cumprod_axis(ctx.handle, a.ptr, 1, 32, 1, 0, ctypes.c_void_p(a.t[16:].data_ptr()), stream))
