"""K15 on the GPU: k_gf_bits_compose, k_gf_binop_view and k_gf_matmul_batched.  The golden fixtures (tests/golden/gf_local.json,
the unmodified reference's values, result types and errors) through install's hooks on limb-backed and plain operands; at
10^7 bytes, bit composition against NumPy, the batched product against K1's k_gf_matmul slice by slice and as one 2-D
product, and broadcast + and * against K1's same-shape k_gf_binop on the materialised broadcast; operands that start at odd
offsets inside their allocation; and the AES S-box of all 256 bytes built from x**254, bits, the stacked product with the
affine matrix, + B and bit composition, against the S-box computed here from its definition."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import device as dev, layout        # noqa: E402
from mpyc_b200._cabi import OP_ADD, OP_MUL         # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import oracle_gf                                   # noqa: E402
import test_gf_hooks as hooks                      # noqa: E402
from test_gf_hooks import mpyc_mods                # noqa: E402,F401  (fixture)

gold = hooks.gold
FIXTURES = hooks.FIXTURES
N = 10**7


def gf(poly=283):
    return mpyc_b200.context_for(poly, binary=True)


def up(ctx, a):
    return DeviceArray.from_limbs(ctx, np.array(a, dtype=np.uint8).reshape(-1))


def down(x):
    return np.asarray(x.to_limbs(), dtype=np.uint8).reshape(-1)


def odd(ctx, a):
    """a uploaded one byte into its allocation: the operand starts at an odd address"""
    a = np.ascontiguousarray(a, dtype=np.uint8).reshape(-1)
    buf = up(ctx, np.concatenate([np.zeros(1, np.uint8), a]))
    return DeviceArray(ctx, buf.t[1:])


@pytest.mark.parametrize('plain', [False, True], ids=['limb', 'plain'])
def test_fixtures_through_the_hooks(mpyc_mods, plain):
    thresha, finfields, gfpx = mpyc_mods
    from mpyc_b200 import install as inst, resident
    inst.install(thresha, resident=True, finfields_module=finfields, operators_min_size=1)
    try:
        for c in FIXTURES:
            F, ctx = hooks.field(finfields, gfpx, c['poly'])
            name = c['case']
            mat = resident.calls['materialised']
            r = hooks.run(F, None if plain else ctx, name, None if plain else hooks.limb_maker(F, ctx))
            if gold.CASES[name][2] and not plain:
                assert resident.calls['materialised'] == mat, name
            assert gold.outcome(r) == c['want'], name
    finally:
        inst.uninstall()


@pytest.mark.parametrize('poly', [283, 285])
def test_bits_compose_against_numpy(poly):
    ctx = gf(poly)
    rng = np.random.default_rng(1)
    bits = rng.integers(0, 2, size=(N // 8, 8), dtype=np.uint8)
    want = np.packbits(bits, axis=-1, bitorder='little').reshape(-1)        # degree < 8: nothing to reduce
    assert np.array_equal(down(dev.gf_bits_compose(up(ctx, bits), N // 8, 8)), want)
    assert np.array_equal(down(dev.gf_bits_compose(odd(ctx, bits), N // 8, 8)), want)
    for l in (1, 3, 13, 30, 300):                                             # general rows: every byte value, reduced
        x = rng.integers(0, 256, size=(N // l // 8, l), dtype=np.uint8)
        want = oracle_gf.gf_bits_compose(None, ctx, x, x.shape[0], l)
        assert np.array_equal(down(dev.gf_bits_compose(up(ctx, x), x.shape[0], l)), want), l
        assert np.array_equal(down(dev.gf_bits_compose(odd(ctx, x), x.shape[0], l)), want), l


@pytest.mark.parametrize('poly', [283, 285])
def test_batched_product_equals_k_gf_matmul(poly):
    ctx = gf(poly)
    rng = np.random.default_rng(2)
    n = N // 8
    A = rng.integers(0, 256, size=(8, 8), dtype=np.uint8)
    X = rng.integers(0, 256, size=(n, 8), dtype=np.uint8)
    got = down(dev.gf_matmul_batched(up(ctx, A), False, up(ctx, X), True, n, 8, 8, 1)).reshape(n, 8)
    whole = down(dev.matmul(ctx, up(ctx, A), up(ctx, X.T), 8, 8, n)).reshape(8, n)          # k_gf_matmul, one 2-D product
    assert np.array_equal(got, whole.T)
    got_odd = down(dev.gf_matmul_batched(odd(ctx, A), False, odd(ctx, X), True, n, 8, 8, 1)).reshape(n, 8)
    assert np.array_equal(got_odd, got)
    for b in (0, 1, n // 2, n - 1):
        assert np.array_equal(got[b], down(dev.matmul(ctx, up(ctx, A), up(ctx, X[b]), 8, 8, 1))), b
    # both sides stacked, a stacked left side with a broadcast right side, and A past the shared-memory size
    for (r, k, c, batch, sa, sb) in ((4, 4, 4, 4096, True, True), (3, 5, 2, 1000, True, False), (80, 60, 3, 7, False, True)):
        P = rng.integers(0, 256, size=((batch if sa else 1), r, k), dtype=np.uint8)
        Q = rng.integers(0, 256, size=((batch if sb else 1), k, c), dtype=np.uint8)
        got = down(dev.gf_matmul_batched(odd(ctx, P), sa, odd(ctx, Q), sb, batch, r, k, c)).reshape(batch, r, c)
        for b in (0, batch // 3, batch - 1):
            want = down(dev.matmul(ctx, up(ctx, P[b if sa else 0]), up(ctx, Q[b if sb else 0]), r, k, c)).reshape(r, c)
            assert np.array_equal(got[b], want), (r, k, c, b)


@pytest.mark.parametrize('op', [OP_ADD, OP_MUL])
def test_broadcasts_equal_k_gf_binop_on_the_materialised_operand(op):
    ctx = gf()
    rng = np.random.default_rng(3)
    for sa, sb in (((N // 8, 8), (8,)), ((N // 1000, 1, 1000), (1, 10, 1)), ((8,), (N // 8, 8)), ((N // 4, 1), (N // 4, 4))):
        a = rng.integers(0, 256, size=sa, dtype=np.uint8)
        b = rng.integers(0, 256, size=sb, dtype=np.uint8)
        shape, va, vb = layout.broadcast_views(sa, sb)
        ca, cb = layout.collapse(va, vb)
        got = down(dev.gf_binop_view(odd(ctx, a), ca, odd(ctx, b), cb, op))
        A, B = np.broadcast_to(a, shape), np.broadcast_to(b, shape)
        want = down(up(ctx, A)._binop(up(ctx, B), op))                       # K1's same-shape k_gf_binop
        assert np.array_equal(got, want), (sa, sb)


def aes_sbox():
    """The AES S-box from its definition: the inverse in GF(2^8) mod 283, then b ^ rotl(b, 1..4) ^ 0x63."""
    def mul(a, b):
        r = 0
        while b:
            if b & 1:
                r ^= a
            a <<= 1
            if a & 0x100:
                a ^= 283
            b >>= 1
        return r
    inv = [0] + [next(y for y in range(1, 256) if mul(x, y) == 1) for x in range(1, 256)]
    rotl = lambda b, s: ((b << s) | (b >> (8 - s))) & 0xFF       # noqa: E731
    return [inv[x] ^ rotl(inv[x], 1) ^ rotl(inv[x], 2) ^ rotl(inv[x], 3) ^ rotl(inv[x], 4) ^ 0x63 for x in range(256)]


def test_batched_sbox_of_all_bytes():
    ctx = gf()
    x = up(ctx, np.arange(256, dtype=np.uint8))
    inv = down(x ** 254)
    bits = ((inv[:, None] >> np.arange(8)) & 1).astype(np.uint8)                      # np_to_bits-style (256, 8)
    A = np.array([np.roll([1, 0, 0, 0, 1, 1, 1, 1], j) for j in range(8)], dtype=np.uint8)   # demos/np_aes.py's circulant
    B = np.array([1, 1, 0, 0, 0, 1, 1, 0], dtype=np.uint8)
    y = dev.gf_matmul_batched(up(ctx, A), False, up(ctx, bits), True, 256, 8, 8, 1)        # A @ x[..., None]
    shape, va, vb = layout.broadcast_views((256, 8), (8,))
    ca, cb = layout.collapse(va, vb)
    y = dev.gf_binop_view(y, ca, up(ctx, B), cb, OP_ADD)                                      # x += B
    s = dev.gf_bits_compose(y, 256, 8)                                                          # np_from_bits
    assert down(s).tolist() == aes_sbox()
