"""K10 (csrc/conv.cuh) on the device: the reference's convolutions (tests/golden/conv.json) replayed through the C ABI and
through install's np.convolve hook; NumPy object convolution mod p up to 2000 x 2000 for every limb count and reduction
kind, in all three modes, on arbitrary windows and on inputs at odd 8-byte offsets; the identity C(r) = A(r) B(r) at a
random r for full results of (2^17, 2^17) and (2^22, 33); a unit-vector convolution at np_roll's shape (10^5, 10^5 + 1)
as an exact shift; worst-case lazy sums for every limb count -- all-(p - 1) operands whose outputs have more than 2^20
terms, in the split form (a 1024-output window) and in the tile form (a window of enough runs to fill the device, where
one work item folds its lazy sums) -- and shapes on both sides of the split decision."""
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
_spec = importlib.util.spec_from_file_location('make_golden_conv', os.path.join(HERE, 'golden', 'make_golden_conv.py'))
gold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gold)
with open(os.path.join(HERE, 'golden', 'conv.json')) as _fh:
    CASES = json.load(_fh)
PRIMES = gold.PRIMES
P61, P128, P256 = gold.P61, gold.P128, gold.P256
SM_COUNT = torch.cuda.get_device_properties(0).multi_processor_count


def window(m, n, mode):
    s, g = min(m, n), max(m, n)
    return {'full': (0, m + n - 1), 'same': ((s - 1) // 2, g), 'valid': (s - 1, g - s + 1)}[mode]


def upload(ctx, vals, offset=0):
    """vals as a DeviceArray; offset: that many spare 64-bit words before the first element (odd: 8-byte aligned only)"""
    limbs = codec.ints_to_limbs([int(v) for v in vals], ctx)
    flat = torch.empty(offset + limbs.size, dtype=torch.int64, device='cuda')
    flat[offset:].copy_(torch.from_numpy(np.ascontiguousarray(limbs).view(np.int64).reshape(-1)))
    return DeviceArray(ctx, flat[offset:].view(len(vals), ctx.nlimbs))


def ints(a):
    return [int(v) for v in a.to_ints()]


def golden_operands(c):
    p = int(c['p'], 16)
    return p, [gold.operand(p, length, form, c['seed'] + k) for k, (length, form) in enumerate(zip((c['m'], c['n']), c['forms']))]


def test_golden_replay_through_the_abi():
    assert len(CASES) > 600
    for c in CASES:
        p, (a, b) = golden_operands(c)
        ctx = mpyc_b200.context_for(p)
        lo, count = window(c['m'], c['n'], c['mode'])
        got = ints(dev.convolve(ctx, upload(ctx, [int(v) % p for v in a]), c['m'], upload(ctx, [int(v) % p for v in b]), c['n'],
                                lo, count))
        assert ([hex(v) for v in got] if count <= gold.STORE_LIMIT else gold.digest(got)) == c['result'], c


@pytest.fixture(scope='module')
def finfields():
    ref = reference.path()
    if ref is None:
        pytest.skip('reference not present ($MPYC_REFERENCE, or the copy build() makes in oracle/_ref)')
    sys.dont_write_bytecode = True
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import thresha, finfields
    finally:
        sys.argv = argv
    yield thresha, finfields
    sys.path.remove(ref)


def test_golden_replay_through_the_hook(finfields):
    thresha, ff = finfields
    from mpyc_b200 import install as inst, resident
    inst.install(thresha, operators=True, finfields_module=ff, operators_min_size=1)
    try:
        for c in CASES:
            p, ops = golden_operands(c)
            F, ctx = ff.GF(p).array, mpyc_b200.context_for(p)
            ops = [F(resident.LimbValue(ctx, upload(ctx, x), (len(x),)), check=False) if form in ('field', 'max') else x
                   for x, form in zip(ops, c['forms'])]
            mat = resident.calls['materialised']
            r = np.convolve(ops[0], ops[1], mode=c['mode'])
            assert type(resident.raw_value(r)) is resident.LimbValue
            assert resident.calls['materialised'] == mat
            vals = [int(v) for v in np.asarray(r.value, dtype=object)]
            assert ([hex(v) for v in vals] if c['len'] <= gold.STORE_LIMIT else gold.digest(vals)) == c['result'], c
    finally:
        inst.uninstall()


def residues(rng, count, p):
    w = rng.integers(0, 2**63, size=(count, 5), dtype=np.int64)
    return [sum(int(x) << (63 * i) for i, x in enumerate(r)) % p for r in w]


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_numpy_object_convolution(p):
    """Every mode, arbitrary windows and operands that are only 8-byte aligned, against np.convolve of Python ints."""
    ctx = mpyc_b200.context_for(p)
    rng = np.random.default_rng(p % 2**32)
    for m, n in ((2000, 1999), (1999, 2000), (1500, 37), (33, 1800), (300, 300), (129, 4100), (4100, 1), (1, 1)):
        a, b = residues(rng, m, p), residues(rng, n, p)
        full = [int(v) % p for v in np.convolve(np.array(a, dtype=object), np.array(b, dtype=object))]
        A, B = upload(ctx, a), upload(ctx, b)
        Ao, Bo = upload(ctx, a, offset=1), upload(ctx, b, offset=3)
        for mode in ('full', 'same', 'valid'):
            lo, count = window(m, n, mode)
            assert ints(dev.convolve(ctx, A, m, B, n, lo, count)) == full[lo:lo + count], (m, n, mode)
        for _ in range(4):
            lo = int(rng.integers(0, m + n - 1))
            count = int(rng.integers(0, m + n - lo))
            want = full[lo:lo + count]
            assert ints(dev.convolve(ctx, A, m, B, n, lo, count)) == want, (m, n, lo, count)
            assert ints(dev.convolve(ctx, Ao, m, Bo, n, lo, count)) == want, (m, n, lo, count, 'offset')
            assert ints(dev.convolve(ctx, Bo, n, A, m, lo, count)) == want, (m, n, lo, count, 'swapped')


def evaluate(vals, r, p):
    acc = 0
    for v in reversed(vals):
        acc = (acc * r + v) % p
    return acc


@pytest.mark.parametrize('p', [P61, P128, P256], ids=lambda p: f'p{p.bit_length()}')
@pytest.mark.parametrize('m,n', [(2**17, 2**17), (2**22, 33)])
def test_polynomial_identity(p, m, n):
    ctx = mpyc_b200.context_for(p)
    A, B = DeviceArray.random(ctx, m, seed=m + 1), DeviceArray.random(ctx, n, seed=n + 7)
    C = dev.convolve(ctx, A, m, B, n, 0, m + n - 1)
    r = int(np.random.default_rng(m ^ n).integers(2, 2**62))
    assert evaluate(ints(C), r, p) == evaluate(ints(A), r, p) * evaluate(ints(B), r, p) % p


@pytest.mark.parametrize('p', [P61, P256], ids=lambda p: f'p{p.bit_length()}')
def test_unit_vector_is_an_exact_shift(p):
    """np_roll's secret shift: a (N) convolved with the unit vector e_s (N + 1) is a moved s places up, zeros elsewhere."""
    N, s = 10**5, 31337
    ctx = mpyc_b200.context_for(p)
    a = DeviceArray.random(ctx, N, seed=5)
    u = torch.zeros((N + 1, ctx.nlimbs), dtype=torch.int64, device='cuda')
    u[s, 0] = 1
    c = dev.convolve(ctx, a, N, DeviceArray(ctx, u), N + 1, 0, 2 * N).t
    assert torch.equal(c[s:s + N], a.t)
    assert not c[:s].any() and not c[s + N:].any()


def check_term_counts(p, m, n, lo, count):
    """all-(p - 1) operands: (p - 1)^2 = 1, so output k is its number of terms mod p"""
    ctx = mpyc_b200.context_for(p)
    A = upload(ctx, [p - 1])                                  # one element, broadcast into a full operand below
    a = DeviceArray(ctx, A.t.expand(m, ctx.nlimbs).contiguous())
    b = DeviceArray(ctx, A.t.expand(n, ctx.nlimbs).contiguous())
    got = ints(dev.convolve(ctx, a, m, b, n, lo, count))
    ks = np.arange(lo, lo + count, dtype=np.int64)
    terms = np.minimum(ks, m - 1) - np.maximum(0, ks - n + 1) + 1
    assert terms.min() > 2**20
    assert got == [int(t) % p for t in terms]


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_lazy_sum_bound_split_form(p):
    """A 1024-output window at the centre of m = n = 2^20 + 515: every output has more than 2^20 terms."""
    m = n = 2**20 + 515
    check_term_counts(p, m, n, (m + n - 1) // 2 - 512, 1024)


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_lazy_sum_bound_tile_form(p):
    """A centre window of 2 * SM_COUNT runs (csrc/inst_conv.cu does not split it): each work item walks all of its more
    than 2^20 taps and folds its lazy sums on the way."""
    count = 2 * SM_COUNT * gold.run_length(p)
    m = n = 2**20 + 3 + count // 2
    check_term_counts(p, m, n, (m + n - 1) // 2 - count // 2, count)


@pytest.mark.parametrize('p', [P61, gold.P64G, P256], ids=lambda p: f'p{p.bit_length()}')
def test_both_sides_of_the_split_decision(p):
    """Windows of 2 * SM_COUNT runs and one run fewer (split), with long and with short (one chunk: never split) taps."""
    ctx = mpyc_b200.context_for(p)
    T = gold.run_length(p)
    rng = np.random.default_rng(11)
    for runs in (2 * SM_COUNT - 1, 2 * SM_COUNT):
        for s in (128, 300):
            count = runs * T
            g = count + s - 1                                   # 'valid' gives count outputs
            a = DeviceArray.random(ctx, s, seed=s)
            b = DeviceArray.random(ctx, g, seed=g)
            got = dev.convolve(ctx, a, s, b, g, s - 1, count)
            # a few sampled outputs against the definition
            av, bv = ints(a), ints(b)
            gv = ints(got)
            for j in [0, 1, count - 1] + [int(x) for x in rng.integers(0, count, size=20)]:
                k = s - 1 + j
                assert gv[j] == sum(av[i] * bv[k - i] for i in range(s)) % p, (runs, s, j)
