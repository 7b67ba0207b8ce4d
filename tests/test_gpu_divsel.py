"""K11 on the GPU: ff_div (k_inv_batch with a numerator) and k_select.  The golden fixtures (tests/golden/divsel.json, the
unmodified reference's values and errors) through the C ABI and through install's hooks; (a / b) * b == a and select
against NumPy at 10^7 elements for every limb count and reduction kind; sizes on both sides of k_inv_batch's T x B
layout; views that start mid-buffer (8-byte alignment only); all four side forms with non-trivial affine maps and both
mask polarities; a zero divisor first, last and inside a batch."""
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
from mpyc_b200 import codec, device as dev         # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from oracle import reference                       # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden_divsel', os.path.join(HERE, 'golden', 'make_golden_divsel.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'divsel.json')) as _fh:
    FIXTURES = json.load(_fh)
# the fixtures' six primes (L = 1..4, pseudo-Mersenne and generic) and 2^255 - 19
PRIMES = gold.PRIMES + [2**255 - 19]


def rand_array(ctx, n, seed):
    return DeviceArray.random(ctx, n, seed)


def limbs_of(vals, ctx):
    return DeviceArray.from_ints(ctx, vals)


@pytest.mark.parametrize('p', gold.PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_golden_division_through_the_abi(p):
    ctx = mpyc_b200.context_for(p)
    b = gold.operand(p, 'b')
    for x, y in (('a', 'b'), ('max', 'b'), ('a', 'max'), ('b', 'b')):
        want = next(c for c in FIXTURES if c['case'] == f'div_{x}_{y}' and int(c['p'], 16) == p)['hex']
        got = dev.divide(limbs_of(gold.operand(p, x), ctx), limbs_of(gold.operand(p, y), ctx)).to_ints()
        assert [hex(int(v)) for v in got] == want
    for z in ('z0', 'zm', 'zl'):
        with pytest.raises(ZeroDivisionError):
            dev.divide(limbs_of(gold.operand(p, 'a'), ctx), limbs_of(gold.operand(p, z), ctx))
    a, mx = gold.operand(p, 'a'), gold.operand(p, 'max')
    want = next(c for c in FIXTURES if c['case'] == 'where_a_b' and int(c['p'], 16) == p)['hex']
    got = dev.select(np.array(gold.COND), limbs_of(a, ctx), (1, 0), limbs_of(b, ctx), (1, 0)).to_ints()
    assert [hex(int(v)) for v in got] == want
    want = next(c for c in FIXTURES if c['case'] == 'where_max_p+3' and int(c['p'], 16) == p)['hex']
    got = dev.select(np.array(gold.COND), limbs_of(mx, ctx), (1, 0), None, (1, p + 3)).to_ints()
    assert [hex(int(v)) for v in got] == want


@pytest.fixture(scope='module')
def mpyc_mods():
    ref = reference.path()
    if ref is None:
        pytest.skip('reference not present (the copy build() makes in oracle/_ref)')
    sys.dont_write_bytecode = True
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import thresha, finfields
    finally:
        sys.argv = argv
    yield thresha, finfields
    sys.path.remove(ref)


def test_golden_fixtures_through_the_hooks(mpyc_mods):
    thresha, finfields = mpyc_mods
    from mpyc_b200 import install as inst, resident
    inst.install(thresha, operators=True, finfields_module=finfields, operators_min_size=1)
    try:
        for c in FIXTURES:
            p = int(c['p'], 16)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            names, fn = gold.CASES[c['case']]
            ops = [F(resident.LimbValue(ctx, limbs_of(gold.operand(p, k), ctx), (gold.N,)), check=False) for k in names]
            mat = resident.calls['materialised']
            try:
                r = fn(F, *ops)
                got = None
            except Exception as e:   # noqa: BLE001
                got = {'error': [type(e).__name__, str(e)]}
            assert resident.calls['materialised'] == mat, c['case']
            if got is None:
                got = gold.encode(r)
            assert got == {k: v for k, v in c.items() if k in ('hex', 'bool', 'error')}, c['case']
    finally:
        inst.uninstall()


def check_sample(ctx, got: DeviceArray, want_fn, n, k=2000, seed=0):
    """want_fn(indices) -> expected ints; a random sample of k indices plus both ends"""
    rng = np.random.default_rng(seed)
    idx = np.unique(np.concatenate([rng.integers(0, n, size=k), [0, n - 1]]))
    t = got.t[torch.from_numpy(idx).to(got.t.device)]
    vals = codec.limbs_to_ints(t.cpu().numpy().view(np.uint64) if not ctx.binary else t.cpu().numpy(), ctx)
    assert [int(v) for v in vals] == want_fn(idx)


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_division_times_divisor_is_the_numerator_at_1e7(p):
    ctx = mpyc_b200.context_for(p)
    n = 10**7
    a, b = rand_array(ctx, n, 1), rand_array(ctx, n, 2)
    if b.count_mismatch(DeviceArray(ctx, torch.zeros_like(b.t))) != n:
        pytest.skip('a random zero')
    q = dev.divide(a, b)
    assert (q * b).count_mismatch(a) == 0
    check_sample(ctx, q, lambda idx: [int(x) * pow(int(y), -1, p) % p for x, y in zip(
        codec.limbs_to_ints(a.t[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.uint64), ctx),
        codec.limbs_to_ints(b.t[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.uint64), ctx))], n)
    r = dev.divide(b, b)                                        # num aliasing den
    assert r.count_mismatch(DeviceArray(ctx, torch.zeros_like(r.t)).__add__(1)) == 0


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_select_matches_numpy_at_1e7(p):
    ctx = mpyc_b200.context_for(p)
    n = 10**7
    x, y = rand_array(ctx, n, 3), rand_array(ctx, n, 4)
    mask = torch.randint(0, 2, (n,), dtype=torch.uint8, device='cuda')
    out = dev.select(mask, x, (1, 0), y, (1, 0))
    both = dev.select(mask, x, (1, 0), x, (1, 0))
    assert both.count_mismatch(x) == 0
    inv = dev.select(mask, y, (1, 0), x, (1, 0), invert=True)
    assert inv.count_mismatch(out) == 0
    m = mask.cpu().numpy().astype(bool)

    def want(idx):
        t = torch.from_numpy(idx).cuda()
        xs = codec.limbs_to_ints(x.t[t].cpu().numpy().view(np.uint64), ctx)
        ys = codec.limbs_to_ints(y.t[t].cpu().numpy().view(np.uint64), ctx)
        return [int(u) if m[i] else int(v) for i, u, v in zip(idx, xs, ys)]
    check_sample(ctx, out, want, n)


@pytest.mark.parametrize('p', [2**61 - 1, 2**128 - 173, gold.P160, 2**256 - 189], ids=lambda p: f'p{p.bit_length()}')
def test_every_side_form_both_polarities_and_mid_buffer_views(p):
    ctx = mpyc_b200.context_for(p)
    rng = np.random.default_rng(p % 1000)
    n = 1237
    xv = [int(v) % p for v in rng.integers(0, 2**62, size=n + 1)]
    yv = [int(v) % p for v in rng.integers(0, 2**62, size=n + 1)]
    X, Y = limbs_of(xv, ctx), limbs_of(yv, ctx)
    x, y = DeviceArray(ctx, X.t[1:]), DeviceArray(ctx, Y.t[1:])          # start one element in: 8-byte alignment for L = 1, 3
    xv, yv = xv[1:], yv[1:]
    m = rng.integers(0, 2, size=n).astype(bool)
    sx, tx, sy, ty = p - 3, 12345, 7, p - 1
    for invert in (False, True):
        pick = m != invert
        for xs in (x, None):
            for ys in (y, None):
                if xs is None and ys is None:
                    got = dev.select(m, None, (sx, tx), y, (sy, ty), n=n, invert=invert)
                    want = [tx if c else (v * sy + ty) % p for c, v in zip(pick, yv)]
                else:
                    got = dev.select(m, xs, (sx, tx), ys, (sy, ty), n=n, invert=invert)
                    want = [((u * sx + tx) % p if xs is not None else tx) if c else ((v * sy + ty) % p if ys is not None else ty)
                            for c, u, v in zip(pick, xv, yv)]
                assert [int(v) for v in got.to_ints()] == want
    for off in (1, 3):                                         # division of views that start mid-buffer
        a, b = DeviceArray(ctx, X.t[off:]), DeviceArray(ctx, Y.t[off:])
        if 0 in yv[off - 1:]:
            continue
        got = dev.divide(a, b)
        assert [int(v) for v in got.to_ints()] == [u * pow(v, -1, p) % p for u, v in zip(xv[off - 1:], yv[off - 1:])]


@pytest.mark.parametrize('p', [2**64 - 189, 2**128 - 173, gold.P160, 2**256 - 189], ids=lambda p: f'p{p.bit_length()}')
def test_sizes_around_the_batch_layout_and_zero_divisors(p, monkeypatch):
    ctx = mpyc_b200.context_for(p)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_wave = sms * 1024
    for n in (1, 2, 255, 2 * per_wave - 1, 2 * per_wave, 2 * per_wave + 1, 4 * per_wave + 7):
        a, b = rand_array(ctx, n, 5), rand_array(ctx, n, 6)
        q = dev.divide(a, b)
        assert (q * b).count_mismatch(a) == 0, n
    monkeypatch.setenv('MPYC_B200_INV_BATCH', '7')             # long batches on a small array
    n = 1000
    vals = [(i * 7919 + 1) % p or 1 for i in range(n)]
    for z in (0, n - 1, 7 * 13 + 3, 500):
        den = list(vals)
        den[z] = 0
        with pytest.raises(ZeroDivisionError):
            dev.divide(limbs_of(vals, ctx), limbs_of(den, ctx))
    got = dev.divide(limbs_of(vals[::-1], ctx), limbs_of(vals, ctx))
    assert [int(v) for v in got.to_ints()] == [u * pow(v, -1, p) % p for u, v in zip(vals[::-1], vals)]
