"""K12 on the GPU: k_powexp_fixed and k_powexp_elem.  The golden fixtures (tests/golden/powexp.json, the unmodified
reference's values and errors) through the C ABI and through install's hooks; for every limb count and reduction kind at
10^7 elements x^(e1 + e2) = x^e1 x^e2, x^(p - 1) = 1, the two forms agreeing and base^-e base^e = 1; exponent widths from
1 to 256 bits against Python's pow; sizes on both sides of a CTA and of one wave; buffers that start mid-allocation (8-byte
alignment only)."""
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
from mpyc_b200 import codec, device as dev         # noqa: E402
from mpyc_b200._cabi import lib, check             # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from oracle import reference                       # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden_powexp', os.path.join(HERE, 'golden', 'make_golden_powexp.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'powexp.json')) as _fh:
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


def host(a):
    return a.to_limbs().reshape(a.n, -1)


def ones(ctx, n):
    r = np.zeros((n, ctx.nlimbs), dtype=np.uint64)
    r[:, 0] = 1
    return r


def rand_u64(n, seed, bits=64):
    g = np.random.default_rng(seed)
    e = g.integers(0, 2**64 - 1, size=n, dtype=np.uint64, endpoint=True)
    return e >> np.uint64(64 - bits) if bits < 64 else e


@pytest.mark.parametrize('p', gold.PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_golden_fixtures_through_the_abi(p):
    ctx = mpyc_b200.context_for(p)
    done = 0
    for c in FIXTURES:
        if int(c['p'], 16) != p:
            continue
        b, e, fn = gold.CASES[c['case']]
        ex = gold.exponents(p, e)
        packed = codec.exponents_to_limbs(ex)
        if fn is None:
            if 'error' in c:
                continue
            got = dev.pow_exp(ctx, gold.list_base(p, b) % p, *packed).to_ints()
        else:
            if 'error' in c or e == 'neg':
                continue
            got = dev.pow_exp(ctx, DeviceArray.from_ints(ctx, gold.bases(p, b)), *packed).to_ints()
        assert [hex(int(v)) for v in got] == c['hex'], c['case']
        done += 1
    assert done == 18
    with pytest.raises(ZeroDivisionError):
        dev.pow_exp(ctx, 0, *codec.exponents_to_limbs([1, -1, 2]))


def test_golden_fixtures_through_the_hooks():
    ref = reference.path()
    if ref is None:
        pytest.skip('reference not present')
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import thresha, finfields, gmpy
    finally:
        sys.argv = argv
    from mpyc_b200 import install as inst, resident, codec as cd
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=1, finfields_min_size=1)
    try:
        for c in FIXTURES:
            p = int(c['p'], 16)
            F, ctx = finfields.GF(p).array, mpyc_b200.context_for(p)
            b, e, fn = gold.CASES[c['case']]
            ex = gold.exponents(p, e)
            try:
                if fn is None:
                    got = {'hex': [hex(v) for v in gmpy.powmod_exp_list(gold.list_base(p, b), ex.tolist() if e == 'obj' else ex, p)]}
                else:
                    x = F(resident.LimbValue(ctx, cd.ints_to_limbs(gold.bases(p, b), ctx), (gold.N,)), check=False)
                    got = gold.encode(fn(F, x, ex))
            except Exception as err:   # noqa: BLE001
                got = {'error': [type(err).__name__, str(err)]}
            assert got == {k: v for k, v in c.items() if k in ('hex', 'error')}, c['case']
    finally:
        inst.uninstall()
        sys.path.remove(ref)


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_identities_at_1e7(cell):
    """Compared on the device (count_mismatch), so that no 10^7-element array crosses to the host."""
    ctx = ctx_of(cell)
    p = cell[0]
    x = DeviceArray.random(ctx, BIG, 12)
    e1, e2 = rand_u64(BIG, 1), rand_u64(BIG, 2)
    s = e1 + e2
    e12 = np.stack([s, (s < e1).astype(np.uint64)], axis=1)               # e1 + e2 as 65-bit exponents
    a, b, ab = (dev.pow_exp(ctx, x, e1.reshape(-1, 1), None, 64), dev.pow_exp(ctx, x, e2.reshape(-1, 1), None, 64),
                dev.pow_exp(ctx, x, e12, None, 65))
    assert (a * b).count_mismatch(ab) == 0
    # Fermat: x^(p - 1) = 1 for x != 0 (and x^0 = 1, 0^0 included)
    one = dev.pow_exp(ctx, x, np.zeros((BIG, 1), dtype=np.uint64), None, 0)
    assert (one * x).count_mismatch(x) == 0
    pm1 = codec.exponents_to_limbs([p - 1])[0]
    r = dev.pow_exp(ctx, x, np.repeat(pm1, BIG, axis=0), None, (p - 1).bit_length())
    zeros = BIG - dev.nonzero(x, want_mask=False)[1]
    assert zeros <= 2 and r.count_mismatch(one) == zeros
    # the two forms agree; a negative exponent times base^|e| is 1
    base = int(codec.limbs_to_ints(host(DeviceArray(ctx, x.t[:1])), ctx)[0]) or 3
    xb = DeviceArray.from_limbs(ctx, np.repeat(codec.ints_to_limbs([base], ctx), BIG, axis=0))
    fixed = dev.pow_exp(ctx, base, e1.reshape(-1, 1), None, 64)
    assert fixed.count_mismatch(dev.pow_exp(ctx, xb, e1.reshape(-1, 1), None, 64)) == 0
    signs = (rand_u64(BIG, 3) & np.uint64(1)).astype(np.uint8)
    neg = dev.pow_exp(ctx, base, e1.reshape(-1, 1), signs, 64)
    want = dev.select(signs.astype(bool), one, (1, 0), fixed * fixed, (1, 0))
    assert (neg * fixed).count_mismatch(want) == 0


@pytest.mark.parametrize('cell', CELLS, ids=cell_id)
def test_exponent_widths_against_python_pow(cell):
    ctx = ctx_of(cell)
    p = cell[0]
    n, k = 1 << 17, 10**4
    g = np.random.default_rng(cell[0] % 2**32)
    x = DeviceArray.random(ctx, n, 5)
    xv = codec.limbs_to_ints(host(x), ctx)
    idx = g.choice(n, size=k, replace=False)
    for w in (1, 31, 63, 64, 65, 128, 255, 256):
        vals = [int.from_bytes(g.bytes(32), 'little') >> (256 - w) for _ in range(n)]
        vals[int(idx[0])] |= 1 << (w - 1)
        packed = codec.exponents_to_limbs(vals)
        assert packed[2] == w
        elem = codec.limbs_to_ints(host(dev.pow_exp(ctx, x, *packed)), ctx)
        base = int(xv[1]) or 7
        fixed = codec.limbs_to_ints(host(dev.pow_exp(ctx, base, *packed)), ctx)
        for i in idx:
            assert int(elem[i]) == pow(int(xv[i]), vals[i], p), (w, int(i))
            assert int(fixed[i]) == pow(base, vals[i], p), (w, int(i))


@pytest.mark.parametrize('cell', [CELLS[1], CELLS[5], CELLS[9]], ids=cell_id)
def test_sizes_around_a_cta_and_a_wave(cell):
    ctx = ctx_of(cell)
    p = cell[0]
    wave = torch.cuda.get_device_properties(0).multi_processor_count * 256 * 2
    for n in (1, 255, 256, 257, wave - 1, wave, wave + 1, 2 * wave + 3):
        vals = [int(v) for v in rand_u64(n, n, 40)]
        x = DeviceArray.random(ctx, n, n)
        xv = codec.limbs_to_ints(host(x), ctx)
        packed = codec.exponents_to_limbs([-v if i % 3 == 0 else v for i, v in enumerate(vals)])
        got = codec.limbs_to_ints(host(dev.pow_exp(ctx, 5, *packed)), ctx)
        assert [int(v) for v in got] == [pow(5, -v if i % 3 == 0 else v, p) for i, v in enumerate(vals)], n
        got = codec.limbs_to_ints(host(dev.pow_exp(ctx, x, *codec.exponents_to_limbs(vals))), ctx)
        assert [int(v) for v in got] == [pow(int(a), v, p) for a, v in zip(xv, vals)], n


@pytest.mark.parametrize('cell', [CELLS[0], CELLS[4], CELLS[8], CELLS[11]], ids=cell_id)
def test_buffers_that_start_mid_allocation(cell):
    """Bases, exponents, signs and out each start 8 bytes into their allocation (odd 8-byte offsets)."""
    ctx = ctx_of(cell)
    p, L = cell[0], ctx.nlimbs
    n = 5000
    g = np.random.default_rng(9)
    vals = [int.from_bytes(g.bytes(16), 'little') >> 30 for _ in range(n)]
    limbs, _, bits = codec.exponents_to_limbs(vals)
    el = limbs.shape[1]
    xv = [int.from_bytes(g.bytes(32), 'little') % p for _ in range(n)]
    xb = torch.zeros(n * L + 1, dtype=torch.int64, device='cuda')
    xb[1:].copy_(torch.from_numpy(codec.ints_to_limbs(xv, ctx).reshape(-1).view(np.int64)))
    eb = torch.zeros(n * el + 1, dtype=torch.int64, device='cuda')
    eb[1:].copy_(torch.from_numpy(np.ascontiguousarray(limbs).reshape(-1).view(np.int64)))
    sb = torch.zeros(n + 1, dtype=torch.uint8, device='cuda')
    sb[1:] = torch.from_numpy((np.arange(n) % 2).astype(np.uint8))
    ob = torch.zeros(n * L + 1, dtype=torch.int64, device='cuda')

    def at(t, k):
        return ctypes.c_void_p(t.data_ptr() + k)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def result():
        torch.cuda.synchronize()
        return [int(v) for v in codec.limbs_to_ints(ob[1:].cpu().numpy().view(np.uint64).reshape(n, L), ctx)]
    check(lib.mpyc_b200_ff_pow_exp(ctx.handle, at(xb, 8), None, at(eb, 8), el, bits, None, n, at(ob, 8), stream))
    assert result() == [pow(a, v, p) for a, v in zip(xv, vals)]
    check(lib.mpyc_b200_ff_pow_exp(ctx.handle, None, ctx.scalar_limbs(3), at(eb, 8), el, bits, at(sb, 1), n, at(ob, 8), stream))
    assert result() == [pow(3, -v if i % 2 else v, p) for i, v in enumerate(vals)]
