"""K14 on the GPU: k_matmul_int_cols and k_matmul_int_rows.  The golden fixtures (tests/golden/matmul_int.json, the
unmodified reference's values, result types and errors) through install's hooks; for every limb count and reduction kind,
products against Python ints on both sides of the columns / rows and split decisions, with operands that start
mid-allocation (8-byte alignment only) and every integer dtype; k past the 2^20 fold with extreme entries against all-(p - 1)
field operands; K14 against K1c on the same matrix converted to limbs at about 10^7 products; and linearity
X@W1 + X@W2 == X@(W1+W2) with K1 additions."""
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
from mpyc_b200._cabi import OP_ADD                 # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from oracle import reference                       # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden_matmul_int', os.path.join(HERE, 'golden', 'make_golden_matmul_int.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'matmul_int.json')) as _fh:
    FIXTURES = json.load(_fh)

# (p, limbs, kind): every limb count with each reduction kind (1: pseudo-Mersenne aligned, 2: shifted, 0: generic);
# 2^57 - 13 is a 1-limb shifted field below 2^61, where the lazy sums fold every 2^12 terms
CELLS = [(2**61 - 1, 1, 2), (2**64 - 189, 1, 1), (9409569905028393239, 1, 0),
         (2**127 - 1, 2, 2), (2**128 - 173, 2, 1), (0xd1b54a32d192ed03a5c2a0c9b1f0e7ed, 2, 0),
         (2**189 - 25, 3, 2), (2**192 - 237, 3, 1), (gold.P192, 3, 0),
         (2**255 - 19, 4, 2), (2**256 - 189, 4, 1), (2**256 - 2**32 - 977, 4, 0)]
SHORT = (2**57 - 13, 1, 2)


def cell_id(c):
    return f'L{c[1]}k{c[2]}'


def ctx_of(cell):
    p, L, kind = cell
    ctx = mpyc_b200.context_for(p)
    assert (ctx.nlimbs, ctx.kind) == (L, kind)
    return ctx


def field_vals(p, n, seed):
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 2**63, size=(n, 5), dtype=np.int64)
    v = [sum(int(x) << (63 * i) for i, x in enumerate(row)) % p for row in w]
    v[:min(n, 3)] = [p - 1, 0, 1][:min(n, 3)]
    return v


def host(p, X, W, r, k, c, w_left):
    Xo = np.array(X, dtype=object)
    Wo = np.array([int(v) for v in np.asarray(W).reshape(-1)], dtype=object)
    if k == 0:
        return [0] * (r * c)
    C = Wo.reshape(r, k) @ Xo.reshape(k, c) if w_left else Xo.reshape(r, k) @ Wo.reshape(k, c)
    return [int(v) % p for v in np.reshape(C, -1)]


def filled(ctx, value, n):
    a = DeviceArray.empty(ctx, n)
    row = torch.from_numpy(mpyc_b200.codec.ints_to_limbs([value], ctx).view(np.int64)).to(a.t.device)
    a.t.copy_(row.expand(n, -1))
    return a


def mid(ctx, vals):
    """A DeviceArray view that starts one element into its allocation (8-byte but not 16-byte aligned for L = 1, 3)."""
    a = DeviceArray.from_ints(ctx, [0] + vals)
    return DeviceArray(ctx, a.t[1:])


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
    """Every fixture on limb-backed operands in HBM (CudaBackend): the reference's values, types and errors, one K14 call
    per integer-operand case."""
    thresha, finfields = mpyc_mods
    from mpyc_b200 import install as inst, resident
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=1, public_matmul=True)
    try:
        for c in FIXTURES:
            p = int(c['p'], 16)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            d, fn = gold.CASES[c['case']]
            vals = gold.values(p, d)
            x = F(resident.LimbValue(ctx, DeviceArray.from_ints(ctx, vals), gold.SHAPES[d]), check=False)
            k14 = resident.calls['matmul_int']
            try:
                r = fn(F, x)
            except Exception as e:   # noqa: BLE001
                assert 'error' in c and [type(e).__name__, str(e)] == c['error'], c['case']
                continue
            kernel = c['case'].startswith(('xW_', 'Wx_', 'np_xW_', 'np_Wx_'))
            assert resident.calls['matmul_int'] == k14 + kernel, c['case']
            if kernel and c['kind'] == 'array' and c['shape']:
                assert type(resident.raw_value(r)) is resident.LimbValue, c['case']
            assert gold.encode(r) == {k: v for k, v in c.items() if k not in ('p', 'case')}, c['case']
    finally:
        inst.uninstall()


# (r, k, c): columns form (c >= 32) with TM = 1 and 4 and partial tiles, rows form (c < 32) with c = 1, a divisor of 32 and
# not, and shapes on both sides of the split decision (few outputs, long k)
SHAPES = [(1, 300, 40), (3, 70, 257), (5, 130, 33), (6, 3000, 64), (1, 6000, 300),
          (1, 2000, 1), (7, 50, 1), (3, 33, 16), (9, 200, 31), (2, 5000, 5), (4000, 40, 1)]


@pytest.mark.parametrize('cell', CELLS + [SHORT], ids=cell_id)
def test_shapes_against_python_ints(cell):
    p = cell[0]
    ctx = ctx_of(cell)
    dtypes = ['int64', 'uint64', 'int8', 'uint32']
    for h, (r, k, c) in enumerate(SHAPES):
        for w_left in (False, True):
            dt = dtypes[(h + w_left) % len(dtypes)]
            W = gold.ints((r, k) if w_left else (k, c), dt, h)
            xs = (k, c) if w_left else (r, k)
            X = field_vals(p, xs[0] * xs[1], 7 * h + w_left)
            out = dev.matmul_int(ctx, mid(ctx, X), W, r, k, c, w_left)
            assert [int(v) for v in out.to_ints()] == host(p, X, W, r, k, c, w_left), (r, k, c, w_left, dt)


@pytest.mark.parametrize('cell', CELLS + [SHORT], ids=cell_id)
def test_extreme_entries_past_the_fold_and_split(cell):
    """Every term at its largest (p - 1 times -2^63, 2^63 - 1 or 2^64 - 1): dot products of 9000 terms, past the lazy sums'
    fold every 2^12 terms, on shapes that fill the GPU without a split (rows form with c = 1, columns form with TM = 4), and
    of 2^20 + 77 terms, split into slices and summed by K7 (rows form with c = 1, columns form with r = 1)."""
    p = cell[0]
    ctx = ctx_of(cell)
    want = {v: (p - 1) * v % p for v in (-2**63, 2**63 - 1, 2**64 - 1)}
    for r, k, c in ((2200, 9000, 1), (1100, 9000, 256), (1, (1 << 20) + 77, 1), (1, (1 << 20) + 77, 32)):
        for w_left in (False, True):
            X = filled(ctx, p - 1, k * c if w_left else r * k)
            for val, dt in ((-2**63, 'int64'), (2**63 - 1, 'int64'), (2**64 - 1, 'uint64')):
                W = np.full((r, k) if w_left else (k, c), val, dtype=dt)
                out = dev.matmul_int(ctx, X, W, r, k, c, w_left).to_ints()
                assert set(int(v) for v in out) == {want[val] * k % p}, (r, k, c, w_left, val)


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_equals_k1c_on_the_same_matrix(cell):
    """About 10^7 products: K14 equals K1c given W converted to limbs (entries reduced mod p), on both sides."""
    p = cell[0]
    ctx = ctx_of(cell)
    r, k, c = 100, 1000, 100
    X = DeviceArray.random(ctx, r * k, seed=11)
    W = gold.ints((k, c), 'int64', 5)
    Wl = DeviceArray.from_ints(ctx, [int(v) % p for v in W.reshape(-1)])
    a = dev.matmul_int(ctx, X, W, r, k, c)
    b = dev.matmul(ctx, X, Wl, r, k, c)
    assert torch.equal(a.t, b.t)
    Wt = np.ascontiguousarray(W.T)                                  # (c, k) @ (k, r)
    Xt = DeviceArray.random(ctx, k * r, seed=12)
    Wtl = DeviceArray.from_ints(ctx, [int(v) % p for v in Wt.reshape(-1)])
    assert torch.equal(dev.matmul_int(ctx, Xt, Wt, c, k, r, w_left=True).t, dev.matmul(ctx, Wtl, Xt, c, k, r).t)


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_linearity(cell):
    """X@W1 + X@W2 == X@(W1 + W2) (K1 additions), W1 + W2 kept within int64 by halving the entries."""
    ctx = ctx_of(cell)
    for r, k, c in ((64, 3000, 48), (5000, 300, 1)):
        X = DeviceArray.random(ctx, r * k, seed=r + c)
        W1 = gold.ints((k, c), 'int64', 1) >> 1
        W2 = gold.ints((k, c), 'int64', 2) >> 1
        lhs = dev.matmul_int(ctx, X, W1, r, k, c)._binop(dev.matmul_int(ctx, X, W2, r, k, c), OP_ADD)
        assert torch.equal(lhs.t, dev.matmul_int(ctx, X, W1 + W2, r, k, c).t)
