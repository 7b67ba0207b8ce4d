"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle and the golden fixtures
generated from the real reference.  Bit-exact everywhere (integer work).  Run on an H100:
    python -m pytest tests -m gpu -x -q
"""
import itertools
import random

import numpy as np
import pytest

from golden_util import load, unhex
from oracle import shamir_oracle as orc
import fakefield

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('no CUDA device', allow_module_level=True)

import mpyc_b200                                   # noqa: E402
from mpyc_b200 import thresha, device as dev, codec   # noqa: E402
from mpyc_b200.device import DeviceArray, DeviceMatrix   # noqa: E402

SPLIT = load('split_recombine.json')
PRSS = load('prss.json')
FF = load('finfields.json')
G256 = load('gf256.json')

P61, P64, P69, P127, P128, P256 = 2**61 - 1, 2**64 - 189, 2**69 - 93, 2**127 - 1, 2**128 - 173, 2**256 - 189
P64G = 9409569905028393239
GEN = {k: int(v, 16) for k, v in SPLIT['meta']['generic_primes'].items()}


class inject:
    """thresha.coefficient_source <- fixed stream (the role of patching secrets.randbelow in the reference)."""

    def __init__(self, stream):
        self.stream = list(stream)

    def __enter__(self):
        it = iter(self.stream)
        thresha.coefficient_source = lambda order, count: list(itertools.islice(it, count))

    def __exit__(self, *exc):
        thresha.coefficient_source = None


# ---- golden fixtures from the reference ------------------------------------------------------------

@pytest.mark.parametrize('case', SPLIT['cases'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_{c['p'][-4:]}_m{c['m']}t{c['t']}")
def test_golden_split_recombine_dropin(case):
    p, m, t = int(case['p'], 16), case['m'], case['t']
    F = fakefield.make_prime_field(p)
    s, stream = unhex(case['secrets']), unhex(case['stream'])
    with inject(stream):
        sh_np = thresha.np_random_split(F, F.array(np.array(s, dtype=object)), t, m)
    assert sh_np.dtype == object and sh_np.shape == (m, len(s))
    assert sh_np.tolist() == unhex(case['shares_np'])
    with inject(stream):
        sh_li = thresha.random_split(F, list(s), t, m)
    assert sh_li == unhex(case['shares_list'])
    with inject(stream):
        sh_el = thresha.random_split(F, [F(x) for x in s], t, m)   # field elements in
    assert sh_el == unhex(case['shares_list'])
    for rec in case['recombine']:
        xs = rec['xs']
        pts = [(x, sh_np[x - 1]) for x in xs]
        assert thresha._recombination_vector(F, tuple(xs), 0) == unhex(rec['lambda0'])
        y0 = thresha.np_recombine(F, pts)
        assert isinstance(y0, F.array) and y0.value.tolist() == unhex(rec['y0'])
        yw = thresha.np_recombine(F, pts, rec['x_rs'])
        assert yw.value.tolist() == unhex(rec['yw'])
        yl = thresha.recombine(F, [(x, sh_li[x - 1]) for x in xs])
        ylr = thresha.recombine(F, [(x, unhex(case['shares_np'])[x - 1]) for x in xs])
        assert ylr == unhex(rec['y0'])
        if len(xs) >= t + 1:
            assert yl == s and y0.value.tolist() == s
        ye = thresha.recombine(F, [(x, [F(v) for v in sh_li[x - 1]]) for x in xs], [0])
        assert all(isinstance(v, F) for v in ye[0])


@pytest.mark.parametrize('case', FF['cases'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_{c['p'][-4:]}")
def test_golden_finfields_device(case):
    p = int(case['p'], 16)
    ctx = mpyc_b200.context_for(p)
    a, b, nz = unhex(case['a']), unhex(case['b']), unhex(case['nz'])
    A, B, NZ = (DeviceArray.from_ints(ctx, v) for v in (a, b, nz))
    g = lambda x: x.to_ints().tolist()
    assert g(A + B) == unhex(case['add'])
    assert g(A - B) == unhex(case['sub'])
    assert g(A * B) == unhex(case['mul'])
    assert g(-A) == unhex(case['neg'])
    assert g(NZ.reciprocal()) == unhex(case['inv_nz'])
    assert g(A / NZ) == unhex(case['div'])
    assert g(A << 7) == unhex(case['lshift7'])
    assert g(A >> 7) == unhex(case['rshift7'])
    assert g(A ** 5) == unhex(case['pow5'])
    assert g(NZ ** -3) == unhex(case['powm3_nz'])
    assert g(A ** ((p - 1) // 2 + 3)) == unhex(case['pow_big'])
    assert A.is_sqr().cpu().tolist() == case['is_sqr']
    assert [int(x) for x in A.signed_()] == [int(x) for x in case['signed']]
    assert g(A * 12345678901234567890123) == unhex(case['mul_scalar'])
    assert g(A + (p - 5)) == unhex(case['add_scalar'])
    assert g(5 - A) == orc.ff_sub(p, [5] * len(a), a)
    if 'sqrt_a' in case:
        assert g(A.sqrt()) == unhex(case['sqrt_a'])
        assert g((A * A).sqrt()) == unhex(case['sqrt_of_sq'])
        assert g((NZ * NZ).sqrt(INV=True)) == unhex(case['invsqrt_of_nzsq'])
        with pytest.raises(ZeroDivisionError):
            A.sqrt(INV=True)
    with pytest.raises(ZeroDivisionError):
        A.reciprocal()          # a contains 0


@pytest.mark.parametrize('case', PRSS['cases'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_m{c['m']}t{c['t']}")
def test_golden_prss_dropin(case):
    p, m, t, n = int(case['p'], 16), case['m'], case['t'], case['n']
    F = fakefield.make_prime_field(p)
    uci = bytes.fromhex(case['uci'])
    keys = {tuple(int(x) for x in k.split(',')): bytes.fromhex(v) for k, v in case['keys'].items()}
    for party in case['parties']:
        i = party['i']
        prfs = {S: thresha.PRF(k, p) for S, k in keys.items() if i in S}
        for S in prfs:
            assert thresha._f_S_i(F, m, i, S) == int(party['f_S_i'][','.join(map(str, S))], 16) % p
        a_np = thresha.np_pseudorandom_share(F, m, i, prfs, uci, n)
        assert isinstance(a_np, F.array) and a_np.value.tolist() == unhex(party['share_np'])
        a_li = thresha.pseudorandom_share(F, m, i, prfs, uci, n)
        assert [x.value for x in a_li] == unhex(party['share_list'])
        z_li = thresha.pseudorandom_share_zero(F, m, i, prfs, uci, n)
        assert [x.value for x in z_li] == unhex(party['zero_list'])
        if t:
            z_np = thresha.np_pseudorandom_share_0(F, m, i, prfs, uci, n)
            assert z_np.value.tolist() == unhex(party['zero_np'])


BOUNDS = load('prss_bounds.json')


@pytest.mark.parametrize('case', BOUNDS['cases'],
                         ids=lambda c: f"{c['field']}{int(c['modulus'], 16).bit_length()}_b{int(c['bound'], 16).bit_length()}_m{c['m']}t{c['t']}")
def test_golden_prss_any_bound(case):
    """Reference-generated PRSS cases whose PRF bound is NOT the field order: 2 (random bits, also on GF(2^8):
    runtime.py:4138,4218), other powers of two below and above the order, runtime._convert's
    (1 << (k+l)) // comb(m,t) + 1 and foreign field orders (runtime.py:735-739,758-760)."""
    mod, bound, m, t, n = int(case['modulus'], 16), int(case['bound'], 16), case['m'], case['t'], case['n']
    F = fakefield.make_gf256(mod) if case['field'] == 'gf' else fakefield.make_prime_field(mod)
    uci = bytes.fromhex(case['uci'])
    keys = {tuple(int(x) for x in k.split(',')): bytes.fromhex(v) for k, v in case['keys'].items()}
    for party in case['parties']:
        i = party['i']
        prfs = {S: thresha.PRF(k, bound) for S, k in keys.items() if i in S}
        a_np = thresha.np_pseudorandom_share(F, m, i, prfs, uci, n)
        assert isinstance(a_np, F.array) and [int(v) for v in a_np.value] == unhex(party['share_np'])
        assert [int(x.value) for x in thresha.pseudorandom_share(F, m, i, prfs, uci, n)] == unhex(party['share_list'])
        assert [int(x.value) for x in thresha.pseudorandom_share_zero(F, m, i, prfs, uci, n)] == unhex(party['zero_list'])
        if t:
            assert [int(v) for v in thresha.np_pseudorandom_share_0(F, m, i, prfs, uci, n).value] == unhex(party['zero_np'])


@pytest.mark.parametrize('mod,binary', [(283, True), (P61, False), (P128, False), (GEN['192'], False), (P256, False)])
def test_prss_general_bound_pipeline_sizes(mod, binary):
    """General-bound PRSS at multi-chunk sizes (reduction kernel + combine kernel per pipeline chunk) against the oracle."""
    from itertools import combinations
    from math import comb
    F = fakefield.make_gf256(mod) if binary else fakefield.make_prime_field(mod)
    Fo = orc.field_of(mod, binary=binary)
    m, t, i = 5, 2, 1
    for bound, n in (((1 << 62) // comb(m, t) + 1, 20011), (P256, 3001), ((1 << 77) + 1, 777), (1 << 90, 1500), (3, 40000)):
        keys = {S: bytes([(sum(S) * 11 + 3) & 0xFF] * 16) for S in combinations(range(m), m - t) if i in S}
        prfs = {S: thresha.PRF(k, bound) for S, k in keys.items()}
        got = [int(v) for v in thresha.np_pseudorandom_share(F, m, i, prfs, b'uci-gen!', n).value]
        assert got == orc.prss_share(Fo, m, i, {S: orc.prf_values(k, bound, b'uci-gen!', n) for S, k in keys.items()}, n)
        n0 = max(n // 7, 1)
        got0 = [int(v) for v in thresha.np_pseudorandom_share_0(F, m, i, prfs, b'uci-gen0', n0).value]
        assert got0 == orc.prss_share_zero_np_order(Fo, m, i, {S: orc.prf_values(k, bound, b'uci-gen0', n0 * t) for S, k in keys.items()}, n0)


def test_prss_power_of_two_bound_and_prf():
    """bounded PRSS (runtime.py:4076: bound = power of two) and the PRF class itself."""
    key = bytes.fromhex(load('prf.json')['key'])
    for c in load('prf.json')['cases']:
        F = thresha.PRF(key, int(c['bound'], 16))
        assert F.byte_length == c['l']
        assert F(bytes.fromhex(c['s']), c['n']) == unhex(c['values'])
    p = P69
    Fld = fakefield.make_prime_field(p)
    m, t, n = 5, 2, 33
    Fo = orc.field_of(p)
    from itertools import combinations
    for bound in (1, 2, 1 << 13, 1 << 40, 1 << 64):
        for i in range(m):
            prfs = {S: thresha.PRF(bytes([sum(S) + 7] * 16), bound) for S in combinations(range(m), m - t) if i in S}
            got = thresha.np_pseudorandom_share(Fld, m, i, prfs, b'uci-0001', n).value.tolist()
            prl = {S: orc.prf_values(f.key, bound, b'uci-0001', n) for S, f in prfs.items()}
            assert got == orc.prss_share(Fo, m, i, prl, n)


def test_golden_gf256():
    f = G256['modulus']
    ctx = mpyc_b200.context_for(f, binary=True)
    tab = np.frombuffer(bytes.fromhex(G256['mul_table_hex']), dtype=np.uint8).reshape(256, 256)
    a = np.repeat(np.arange(256, dtype=np.uint8), 256)
    b = np.tile(np.arange(256, dtype=np.uint8), 256)
    A, B = DeviceArray.from_limbs(ctx, a), DeviceArray.from_limbs(ctx, b)
    assert np.array_equal((A * B).to_limbs(), tab.reshape(-1))
    assert np.array_equal((A + B).to_limbs(), a ^ b)
    assert np.array_equal((A - B).to_limbs(), a ^ b)
    # odd offsets / lengths exercise the byte tail and the unaligned path
    A3, B3 = DeviceArray.from_limbs(ctx, a[:1003]), DeviceArray.from_limbs(ctx, b[:1003])
    assert np.array_equal((A3 * B3).to_limbs(), tab.reshape(-1)[:1003])
    assert np.array_equal((A3 * 0x53).to_limbs(), tab[a[:1003], 0x53])
    nzv = np.arange(1, 256, dtype=np.uint8)
    assert DeviceArray.from_limbs(ctx, nzv).reciprocal().to_limbs().tolist() == G256['inv'][1:]
    with pytest.raises(ZeroDivisionError):
        DeviceArray.from_limbs(ctx, np.arange(0, 9, dtype=np.uint8)).reciprocal()
    F = fakefield.make_gf256(f)
    for case in G256['split']:
        m, t = case['m'], case['t']
        s, stream = unhex(case['secrets']), unhex(case['stream'])
        with inject(stream):
            sh = thresha.np_random_split(F, np.array([fakefield.Poly(x) for x in s], dtype=object), t, m)
        assert [[int(v) for v in row] for row in sh] == unhex(case['shares_np'])
        with inject(stream):
            sl = thresha.random_split(F, [F(x) for x in s], t, m)
        assert [[int(v) for v in row] for row in sl] == unhex(case['shares_list'])
        xs = case['xs']
        assert [int(v) for v in thresha._recombination_vector(F, tuple(xs), 0)] == unhex(case['lambda0'])
        y = thresha.np_recombine(F, [(x, sh[x - 1]) for x in xs])
        assert [int(v) for v in y.value] == unhex(case['y0'])


# ---- seeded random parity against the oracle ----------------------------------------------------------

PARITY_PRIMES = [P61, P64, P64G, P69, GEN['96'], P127, P128, GEN['128'], GEN['192'], 2**192 - 237, GEN['250'], P256, GEN['256'], 101, 65537]


@pytest.mark.parametrize('p', PARITY_PRIMES, ids=lambda p: f'p{p.bit_length()}_{p & 0xffff:x}')
@pytest.mark.parametrize('n', [0, 1, 2, 3, 7, 64, 1001, 4096 + 5])
def test_split_recombine_vs_oracle(p, n):
    ctx = mpyc_b200.context_for(p)
    F = orc.field_of(p)
    rnd = random.Random(n * 7919 + p % 10007)
    for (m, t) in ((1, 0), (3, 1), (5, 2), (7, 3), (4, 3), (13, 5), (17, 8), (12, 9), (24, 11)):
        if n > 100 and (m, t) in ((12, 9), (24, 11), (13, 5)):
            continue
        s = (orc.edge_block(p) + orc.synth_elements(p, max(n - 8, 0), 11 * m + t))[:n]
        C = [orc.synth_elements(p, n, 1000 + 31 * j + m, stream=5) for j in range(t)]
        want = orc.split_np_order(F, s, C, m)
        S = DeviceArray.from_ints(ctx, s)
        CM = DeviceMatrix.from_ints(ctx, C) if t else None
        sh = dev.shamir_split(ctx, S, CM, t, m)
        assert [r.tolist() for r in sh.to_ints()] == want
        if n == 0:
            continue
        k = rnd.choice([t + 1, min(m, 2 * t + 1), m])
        xs = sorted(rnd.sample(range(1, m + 1), k))
        rows = [sh.row(x - 1) for x in xs]
        got = dev.shamir_recombine(ctx, xs, rows)
        assert got.to_ints().tolist() == orc.recombine(F, xs, [want[x - 1] for x in xs]) == s
        x_rs = [0, m + 1, xs[0]]
        gw = dev.shamir_recombine(ctx, xs, rows, x_rs)
        assert [r.tolist() for r in gw.to_ints()] == orc.recombine(F, xs, [want[x - 1] for x in xs], x_rs)


@pytest.mark.parametrize('p', PARITY_PRIMES, ids=lambda p: f'p{p.bit_length()}_{p & 0xffff:x}')
def test_elementwise_vs_oracle(p):
    ctx = mpyc_b200.context_for(p)
    for n in (1, 2, 5, 255, 256, 257, 10007):
        a = (orc.edge_block(p) + orc.synth_elements(p, n, 5))[:n]
        b = (list(reversed(orc.edge_block(p))) + orc.synth_elements(p, n, 6))[:n]
        A, B = DeviceArray.from_ints(ctx, a), DeviceArray.from_ints(ctx, b)
        assert (A * B).to_ints().tolist() == orc.ff_mul(p, a, b)
        assert (A + B).to_ints().tolist() == orc.ff_add(p, a, b)
        assert (A - B).to_ints().tolist() == orc.ff_sub(p, a, b)
        assert (-A).to_ints().tolist() == orc.ff_neg(p, a)
        assert (A * (p - 1)).to_ints().tolist() == orc.ff_mul(p, a, [p - 1] * n)


def test_device_fill_random_matches_oracle_recipe():
    for p in PARITY_PRIMES:
        ctx = mpyc_b200.context_for(p)
        got = DeviceArray.random(ctx, 300, seed=20260923, stream_id=3).to_ints().tolist()
        assert got == orc.synth_elements(p, 300, 20260923, stream=3)


def test_host_buffer_abi_large_chunked():
    """The host-buffer entry points (what the drop-in uses) across several pipeline chunks."""
    p = P128
    ctx = mpyc_b200.context_for(p)
    F = fakefield.make_prime_field(p)
    n, m, t = 3_000_001, 5, 2       # > one 32 MiB chunk, odd
    rng = np.random.default_rng(1)
    sec = rng.integers(0, 2**63, size=(n, 2), dtype=np.uint64)
    sec[:, 1] >>= 1
    C = rng.integers(0, 2**63, size=(t, n, 2), dtype=np.uint64)
    shares = thresha._split_limbs(ctx, sec, C, t, m)
    out = thresha._recombine_limbs(ctx, [2, 4, 5], [shares[1], shares[3], shares[4]], [0])
    assert np.array_equal(out[0], sec)
    idx = [0, 1, n // 2, n - 1]
    s_int = codec.limbs_to_ints(sec[idx], ctx).tolist()
    C_int = [codec.limbs_to_ints(C[j][idx], ctx).tolist() for j in range(t)]
    want = orc.split_np_order(orc.field_of(p), s_int, C_int, m)
    assert [codec.limbs_to_ints(shares[i][idx], ctx).tolist() for i in range(m)] == want


# ---- size-independent properties at full benchmark sizes ---------------------------------------------

@pytest.mark.parametrize('p,m,t,n', [(P128, 5, 2, 100_000_000), (P64, 3, 1, 20_000_000), (P128, 5, 2, 10_000_000), (P256, 7, 3, 2_000_000),
                                      (P64G, 3, 1, 10_000_000), (GEN['128'], 5, 2, 4_000_000), (P61, 3, 1, 10_000_001)])
def test_full_size_roundtrip_and_linearity(p, m, t, n):
    ctx = mpyc_b200.context_for(p)
    S = DeviceArray.random(ctx, n, seed=1, stream_id=1)
    S2 = DeviceArray.random(ctx, n, seed=2, stream_id=2)
    C = DeviceMatrix.empty(ctx, t, n)
    C2 = DeviceMatrix.empty(ctx, t, n)
    for j in range(t):
        C.t[j].copy_(DeviceArray.random(ctx, n, seed=10 + j, stream_id=3).t)
        C2.t[j].copy_(DeviceArray.random(ctx, n, seed=20 + j, stream_id=4).t)
    sh = dev.shamir_split(ctx, S, C, t, m)
    sh2 = dev.shamir_split(ctx, S2, C2, t, m) if n < 50_000_000 else None
    # encode -> erase -> decode: any t+1 shares return the secrets
    for xs in ([1 + i for i in range(t + 1)], [m - i for i in range(t + 1)]):
        rec = dev.shamir_recombine(ctx, xs, [sh.row(x - 1) for x in xs])
        assert rec.count_mismatch(S) == 0
    # all m shares (degree t < m) as well
    rec = dev.shamir_recombine(ctx, list(range(1, m + 1)), [sh.row(i) for i in range(m)])
    assert rec.count_mismatch(S) == 0
    if sh2 is not None:   # (skipped at the BASELINE full size to bound memory: the checks around it remain)
        # linearity: shares of (S + S2) with coefficients (C + C2) are the sums of the shares
        Ssum = S + S2
        Csum = DeviceMatrix.empty(ctx, t, n)
        for j in range(t):
            Csum.t[j].copy_((C.row(j) + C2.row(j)).t)
        shsum = dev.shamir_split(ctx, Ssum, Csum, t, m)
        for i in range(m):
            assert shsum.row(i).count_mismatch(sh.row(i) + sh2.row(i)) == 0
    # recombining at a party's own point returns that party's share
    xs = list(range(1, t + 2))
    own = dev.shamir_recombine(ctx, xs, [sh.row(x - 1) for x in xs], [m])
    assert own.row(0).count_mismatch(sh.row(m - 1)) == 0
    # spot-check against the oracle at a few positions
    idx = torch.tensor([0, 1, n // 3, n - 2, n - 1], device=S.t.device)
    pick = lambda arr: codec.limbs_to_ints(arr.t.index_select(0, idx).cpu().numpy().view(np.uint64), ctx).tolist()   # noqa: E731
    want = orc.split_np_order(orc.field_of(p), pick(S), [pick(C.row(j)) for j in range(t)], m)
    assert [pick(sh.row(i)) for i in range(m)] == want


def test_error_behaviour():
    ctx = mpyc_b200.context_for(P61)
    S = DeviceArray.from_ints(ctx, [1, 2, 3])
    with pytest.raises(ValueError):
        dev.shamir_split(ctx, S, None, 3, 3)        # t >= m
    with pytest.raises(ZeroDivisionError):
        dev.shamir_recombine(ctx, [1, 1], [S, S])   # repeated x-coordinate
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        mpyc_b200.context_for(2**300 + 157)
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        mpyc_b200.context_for(2)
    assert mpyc_b200.launch_count() > 0


# ---- generate mode (coefficients from a ChaCha20 keystream inside the kernel) ---------------------------

def _chacha20_block(key, counter, nonce0, nonce1):
    """Reference ChaCha20 block function (RFC 8439 section 2.3 arithmetic; 64-bit counter layout)."""
    def rotl(v, c):
        return ((v << c) & 0xffffffff) | (v >> (32 - c))

    def qr(x, a, b, c, d):
        x[a] = (x[a] + x[b]) & 0xffffffff; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] = (x[c] + x[d]) & 0xffffffff; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] = (x[a] + x[b]) & 0xffffffff; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] = (x[c] + x[d]) & 0xffffffff; x[b] = rotl(x[b] ^ x[c], 7)
    init = [0x61707865, 0x3320646e, 0x79622d32, 0x6b206574] + [int.from_bytes(key[4 * i:4 * i + 4], 'little') for i in range(8)] \
        + [counter & 0xffffffff, counter >> 32, nonce0, nonce1]
    x = list(init)
    for _ in range(10):
        qr(x, 0, 4, 8, 12); qr(x, 1, 5, 9, 13); qr(x, 2, 6, 10, 14); qr(x, 3, 7, 11, 15)
        qr(x, 0, 5, 10, 15); qr(x, 1, 6, 11, 12); qr(x, 2, 7, 8, 13); qr(x, 3, 4, 9, 14)
    return [(a + b) & 0xffffffff for a, b in zip(x, init)]


def test_chacha_reference_block_matches_rfc8439():
    key = bytes(range(32))
    # RFC 8439 2.3.2: counter = 1, nonce = 00:00:00:09:00:00:00:4a:00:00:00:00
    out = _chacha20_block(key, 1 | (0x09000000 << 32), 0x4a000000, 0)
    assert out[:4] == [0xe4e7f110, 0x15593bd1, 0x1fdd0f50, 0xc47120a3]
    assert out[12:] == [0xd19c12b5, 0xb94e16de, 0xe883d0cb, 0x4e3c50a2]


@pytest.mark.parametrize('p', [P64, P61, P128, P69, P256, P64G, GEN['128'], 2**192 - 237], ids=lambda p: f'p{p.bit_length()}_{p & 0xffff:x}')
def test_generate_mode_uses_chacha20_keystream(p):
    """Known-answer: with t=1 the coefficient of X is share_2 - share_1; it must equal the ChaCha20
    keystream words (64 bits wider than p) reduced mod p, for the documented counter layout."""
    ctx = mpyc_b200.context_for(p)
    L = ctx.nlimbs
    n = 37
    key = bytes((7 * i + 3) & 0xFF for i in range(32))
    nonce = 0x1234567_89ABCDEF
    s = (orc.edge_block(p) + orc.synth_elements(p, n, 3))[:n]
    S = DeviceArray.from_ints(ctx, s)
    sh = dev.shamir_split_generate(ctx, S, 1, 3, key=key, nonce=nonce).to_ints()
    coef = [(int(b) - int(a)) % p for a, b in zip(sh[0], sh[1])]
    words = 2 * L + 2
    slot = 4 if words <= 4 else (8 if words <= 8 else 16)
    per_block = 16 // slot
    E = {1: 4, 2: 2, 3: 1, 4: 1}[L]   # elements per 32-byte vector item (L == 3: scalar path)
    bpi = (E + per_block - 1) // per_block
    keep = (1 << (p.bit_length() + 64)) - 1
    n_items = n // E
    for h in range(n):
        if h < n_items * E:
            it, c = divmod(h, E)
            blk = _chacha20_block(key, it * bpi + c // per_block, nonce & 0xffffffff, (nonce >> 32) & 0x7fffffff)
            off = (c % per_block) * slot
        else:   # scalar tail: disjoint keystream (top nonce bit set), one element per item
            blk = _chacha20_block(key, h * ((1 + per_block - 1) // per_block), nonce & 0xffffffff, ((nonce >> 32) & 0x7fffffff) | 0x80000000)
            off = 0
        x = sum(w << (32 * i) for i, w in enumerate(blk[off:off + words]))
        assert coef[h] == (x & keep) % p, h
    # shares are a valid degree-1 sharing of the secrets
    F = orc.field_of(p)
    assert orc.recombine(F, [2, 3], [[int(v) for v in sh[1]], [int(v) for v in sh[2]]]) == s


@pytest.mark.parametrize('p,m,t,n', [(P64, 3, 1, 1_000_003), (P128, 5, 2, 500_000), (P256, 7, 3, 100_001), (P64G, 5, 2, 200_000), (P69, 9, 4, 50_001)])
def test_generate_mode_properties(p, m, t, n):
    ctx = mpyc_b200.context_for(p)
    S = DeviceArray.random(ctx, n, seed=5, stream_id=9)
    key = bytes(range(32))
    sh = dev.shamir_split_generate(ctx, S, t, m, key=key, nonce=1)
    for xs in ([1 + i for i in range(t + 1)], [m - i for i in range(t + 1)]):
        assert dev.shamir_recombine(ctx, xs, [sh.row(x - 1) for x in xs]).count_mismatch(S) == 0
    sh_same = dev.shamir_split_generate(ctx, S, t, m, key=key, nonce=1)
    sh_other = dev.shamir_split_generate(ctx, S, t, m, key=key, nonce=2)
    sh_fresh = dev.shamir_split_generate(ctx, S, t, m)      # OS randomness
    assert all(sh.row(i).count_mismatch(sh_same.row(i)) == 0 for i in range(m))
    assert sh.row(0).count_mismatch(sh_other.row(0)) > n - 10
    assert sh.row(0).count_mismatch(sh_fresh.row(0)) > n - 10
    # fewer than t+1 shares do not determine the secrets: recombining t shares gives something else
    if t >= 1:
        xs = list(range(1, t + 1))
        assert dev.shamir_recombine(ctx, xs, [sh.row(x - 1) for x in xs]).count_mismatch(S) > n - 10
    with pytest.raises(mpyc_b200.UnsupportedFieldError):
        dev.shamir_split_generate(ctx, S, 5, 11)


# ---- modular matmul (finfields.py:1126-1146) -----------------------------------------------------------

@pytest.mark.parametrize('case', FF['cases'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_{c['p'][-4:]}")
def test_golden_matmul(case):
    p = int(case['p'], 16)
    ctx = mpyc_b200.context_for(p)
    a, b = unhex(case['a']), unhex(case['b'])
    A, B = DeviceArray.from_ints(ctx, a[:12]), DeviceArray.from_ints(ctx, b[:20])
    got = dev.matmul(ctx, A, B, 3, 4, 5).to_ints().tolist()
    want = unhex(case['matmul_3x4_4x5'])
    assert got == [v for row in want for v in row]


@pytest.mark.parametrize('p', [P61, P64, P64G, P69, P128, GEN['128'], 2**192 - 237, P256, GEN['256'], 101], ids=lambda p: f'p{p.bit_length()}_{p & 0xffff:x}')
@pytest.mark.parametrize('shape', [(1, 1, 1), (1, 3136, 300), (5, 70, 257), (9, 64, 3), (2, 129, 600), (4, 0, 3), (3, 1000, 257), (5, 513, 70),
                                   (7, 257, 9)])   # k >= 256 with few output tiles: split-k form
def test_matmul_vs_oracle(p, shape):
    r, k, c = shape
    ctx = mpyc_b200.context_for(p)
    a = (orc.edge_block(p) * (r * k // 8 + 1))[:r * k // 2] + orc.synth_elements(p, r * k - r * k // 2, 21)
    b = orc.synth_elements(p, k * c - min(k * c, 8), 22) + orc.edge_block(p)[:min(k * c, 8)]
    A = DeviceArray.from_ints(ctx, a) if a else DeviceArray.empty(ctx, 0)
    B = DeviceArray.from_ints(ctx, b) if b else DeviceArray.empty(ctx, 0)
    got = dev.matmul(ctx, A, B, r, k, c).to_ints().tolist()
    Am = [a[i * k:(i + 1) * k] for i in range(r)]
    Bm = [b[l * c:(l + 1) * c] for l in range(k)]
    want = [[sum(Am[i][l] * Bm[l][j] for l in range(k)) % p for j in range(c)] for i in range(r)]
    assert got == [v for row in want for v in row]


def test_gf256_matmul():
    f = G256['modulus']
    ctx = mpyc_b200.context_for(f, binary=True)
    tab = np.frombuffer(bytes.fromhex(G256['mul_table_hex']), dtype=np.uint8).reshape(256, 256)
    rng = np.random.default_rng(3)
    r, k, c = 4, 16, 33
    a = rng.integers(0, 256, size=(r, k), dtype=np.uint8)
    b = rng.integers(0, 256, size=(k, c), dtype=np.uint8)
    want = np.zeros((r, c), dtype=np.uint8)
    for l in range(k):
        want ^= tab[a[:, l][:, None], b[l][None, :]]
    got = dev.matmul(ctx, DeviceArray.from_limbs(ctx, a.reshape(-1)), DeviceArray.from_limbs(ctx, b.reshape(-1)), r, k, c)
    assert np.array_equal(got.to_limbs().reshape(r, c), want)


def test_finfields_batched_hooks():
    """mpyc_b200.finfields: value-array in / value-array out replacements of PrimeFieldArray's classmethods."""
    from mpyc_b200 import finfields as ff
    for p in (P61, P128, P256, P64G):
        F = fakefield.make_prime_field(p)
        cls = F.array
        a = np.array(orc.synth_elements(p, 600, 31), dtype=object).reshape(20, 30)
        nz = np.where(a == 0, 1, a)
        assert ff.reciprocal(cls, nz).tolist() == np.array(orc.ff_inv(p, nz.reshape(-1).tolist()), dtype=object).reshape(20, 30).tolist()
        assert ff.power(cls, a, 7).reshape(-1).tolist() == orc.ff_pow(p, a.reshape(-1).tolist(), 7)
        assert ff.power(cls, nz, -2).reshape(-1).tolist() == orc.ff_pow(p, nz.reshape(-1).tolist(), -2)
        assert ff.is_sqr(cls, a).reshape(-1).tolist() == orc.ff_is_sqr(p, a.reshape(-1).tolist())
        if p & 3 == 3:
            assert ff.sqrt(cls, a).reshape(-1).tolist() == orc.ff_sqrt(p, a.reshape(-1).tolist())
            assert ff.sqrt(cls, nz, INV=True).reshape(-1).tolist() == orc.ff_sqrt(p, nz.reshape(-1).tolist(), INV=True)
        with pytest.raises(ZeroDivisionError):
            ff.reciprocal(cls, np.array([3, 0, 5], dtype=object))
        A, B = a[:4, :6], a[:6, :5]
        want = orc.ff_matmul(p, A.tolist(), B.tolist())
        assert ff.matmul(cls, A, B).tolist() == want
        assert ff.matmul(cls, A[0], B).tolist() == want[0]
        assert ff.matmul(cls, A, B[:, 0]).tolist() == [row[0] for row in want]


@pytest.mark.parametrize('p', [2**61 - 1, 2**64 - 189, 2**69 - 93, 2**128 - 173, 2**192 - 237, 2**256 - 189,
                               9409569905028393239, 0x800000000000000000000000000000fb, 101],
                         ids=lambda p: f'p{p.bit_length()}')
@pytest.mark.parametrize('batch', [1, 2, 7, 32])
def test_batched_inverse_montgomery_trick(p, batch, monkeypatch):
    """k_inv_batch (Montgomery's trick, one Fermat exponentiation per `batch` elements) equals the oracle's
    per-element inverse for every batch length, ragged sizes, and reports zeros like gmpy2.invert."""
    monkeypatch.setenv('MPYC_B200_INV_BATCH', str(batch))
    ctx = mpyc_b200.context_for(p)
    rnd = random.Random(p % 977 + batch)
    for n in (1, 2, 31, 257, 1000):
        a = [1, p - 1][:n] + [rnd.randrange(1, p) for _ in range(max(0, n - 2))]
        assert DeviceArray.from_ints(ctx, a).reciprocal().to_ints().tolist() == orc.ff_inv(p, a)
    z = [rnd.randrange(1, p) for _ in range(100)]
    z[37] = 0
    with pytest.raises(ZeroDivisionError):
        DeviceArray.from_ints(ctx, z).reciprocal()


def test_batched_inverse_large_property():
    """n = 2^21 (the launcher picks batch 8 on a 132-SM H100): a * a^-1 == 1 everywhere, checked on the device."""
    for p in (2**128 - 173, 9409569905028393239):
        ctx = mpyc_b200.context_for(p)
        n = (1 << 21) + 5
        A = DeviceArray.random(ctx, n, seed=5, stream_id=3)     # a zero among 2^21 random residues: probability ~0
        limbs = (A * A.reciprocal()).to_limbs()
        assert (limbs[:, 0] == 1).all() and (limbs[:, 1:] == 0).all()


@pytest.mark.parametrize('m,t', [(3, 1), (1, 0), (5, 2), (7, 3), (9, 4), (13, 5), (255, 1)])
@pytest.mark.parametrize('n', [16, 48, 1000, 4096, 4096 + 7, 100003])
def test_gf256_vector_kernels_vs_oracle(m, t, n):
    """GF(2^8) bulk path (k_gf_split_vec: Horner in the point, 16 bytes per access; k_gf_recombine_vec) equals
    the oracle for every t the vector form covers (<= 4), the ladder/generic form (t = 5), ragged tails and
    the largest party count the byte encoding of the points allows."""
    if m == 255 and n > 5000:
        pytest.skip('oracle too slow')
    f = 283
    ctx = mpyc_b200.context_for(f, binary=True)
    Fo = orc.field_of(f, binary=True)
    rnd = random.Random(n * 31 + m)
    s = [rnd.randrange(256) for _ in range(n)]
    C = [[rnd.randrange(256) for _ in range(n)] for _ in range(t)]
    S = DeviceArray.from_limbs(ctx, np.array(s, dtype=np.uint8))
    CM = DeviceMatrix.from_ints(ctx, C) if t else None
    sh = dev.shamir_split(ctx, S, CM, t, m)
    want = orc.split_np_order(Fo, s, C, m)
    got = sh.to_ints()
    assert [[int(v) for v in row] for row in got] == want
    xs = list(range(m - t, m + 1))
    rec = dev.shamir_recombine(ctx, xs, [sh.row(x - 1) for x in xs])
    assert [int(v) for v in rec.to_ints()] == s
    if m >= 2 * t + 1 and m < 255:
        xs = list(range(1, 2 * t + 2))
        rec = dev.shamir_recombine(ctx, xs, [sh.row(x - 1) for x in xs])
        assert [int(v) for v in rec.to_ints()] == s


@pytest.mark.parametrize('p,m,t', [(2**256 - 189, 7, 3), (2**69 - 93, 3, 1), (9409569905028393239, 5, 2), (2**61 - 1, 3, 1),
                                   (2**128 - 173, 5, 2), (2**127 - 1, 3, 1), (2**192 - 237, 3, 1)],
                         ids=['p256_m7t3', 'p69_m3t1', 'generic64_m5t2', 'p61_m3t1', 'p128_m5t2', 'p127_m3t1', 'p192_m3t1'])
def test_prss_pipeline_in_library(p, m, t, monkeypatch):
    """mpyc_b200_prss_host (SHAKE128 sponges on host threads -> pinned chunks -> tiled combine kernel with TMA-staged
    byte tiles): equal to the oracle on a multi-chunk call, and independent of the thread count and of the kernel
    form (tiled / untiled) on a call of np_cnnmnist's largest size (n = 213,248, SURVEY 8a)."""
    F = fakefield.make_prime_field(p)
    Fo = orc.field_of(p)
    subsets = list(itertools.combinations(range(m), m - t))
    keys = {S: bytes([17 * (a + 1) % 256 for a in S] + [0] * (16 - len(S))) for S in subsets}
    i = 1
    mine = {S: keys[S] for S in subsets if i in S}
    uci = b'\x05\x00\x00\x00\x07'

    def prfs(bound):
        return {S: thresha.PRF(k, bound) for S, k in mine.items()}

    n = 20_011                                   # several 256-element tiles, ragged tail, > 1 pipeline chunk for 48-byte chunks
    got = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, n).value.tolist()
    assert got == orc.prss_share(Fo, m, i, {S: orc.prf_values(k, p, uci, n) for S, k in mine.items()}, n)
    got0 = thresha.np_pseudorandom_share_0(F, m, i, prfs(p), uci, 3001).value.tolist()
    assert got0 == orc.prss_share_zero_np_order(Fo, m, i, {S: orc.prf_values(k, p, uci, 3001 * t) for S, k in mine.items()}, 3001)
    big = 213_248
    ref = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, big).value
    monkeypatch.setattr(thresha, 'prss_threads', 1)
    one = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, big).value
    monkeypatch.setenv('MPYC_B200_PRSS_UNTILED', '1')
    flat = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, big).value
    monkeypatch.setenv('MPYC_B200_PRSS_FULL', '1')       # full products with f_S(i) instead of the small-integer form
    flat_full = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, big).value
    monkeypatch.delenv('MPYC_B200_PRSS_UNTILED')
    tiled_full = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, big).value
    zero_full = thresha.np_pseudorandom_share_0(F, m, i, prfs(p), uci, 3001).value.tolist()
    monkeypatch.delenv('MPYC_B200_PRSS_FULL')
    monkeypatch.setenv('MPYC_B200_PRSS_NO_SIMPLE', '1')  # general small form instead of the compile-time plain-share variant
    general = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, big).value
    monkeypatch.delenv('MPYC_B200_PRSS_NO_SIMPLE')
    monkeypatch.setenv('MPYC_B200_PRSS_CHUNK', '2048')   # ~100 pipeline chunks: slot reuse, events, producer hand-off
    monkeypatch.setattr(thresha, 'prss_threads', 3)      # several sponges per thread: the AVX-512 lock-step form where available
    many = thresha.np_pseudorandom_share(F, m, i, prfs(p), uci, big).value
    monkeypatch.setenv('MPYC_B200_NO_AVX512', '1')       # (read once per process: only effective if set before the first PRSS call)
    monkeypatch.delenv('MPYC_B200_PRSS_CHUNK')
    monkeypatch.delenv('MPYC_B200_NO_AVX512')
    monkeypatch.setattr(thresha, 'prss_threads', 0)
    assert many.tolist() == ref.tolist()
    assert general.tolist() == ref.tolist()
    assert zero_full == got0
    assert ref.tolist() == one.tolist() == flat.tolist() == flat_full.tolist() == tiled_full.tolist()
    assert ref[:n].tolist() == got               # a longer call extends the same streams (XOF prefix property)


@pytest.mark.parametrize('p,m,t,k', [(P128, 5, 2, 3), (P64, 3, 1, 3), (P256, 7, 3, 7), (GEN['128'], 5, 2, 5)], ids=['p128', 'p64', 'p256', 'generic128'])
def test_reshare_step_host_equals_the_two_calls(p, m, t, k):
    """mpyc_b200_shamir_reshare_step_host (recombine batch j while dealing batch j+1, chunks of both jobs interleaved on
    two stream sets) gives exactly what mpyc_b200_shamir_split_host and mpyc_b200_shamir_recombine_host give, for
    multi-chunk and ragged sizes and with either job empty; the recombined values are checked against the oracle."""
    import ctypes
    from mpyc_b200 import _cabi
    from mpyc_b200._cabi import lib, check
    ctx = mpyc_b200.context_for(p)
    L = ctx.nlimbs
    Fo = orc.field_of(p)
    xs = list(range(1, k + 1))
    def rand_limbs(n, seed):
        """n canonical residues as a host limb array (generated on the device: no Python-int loops)."""
        if n == 0:
            return np.zeros((0, L), np.uint64)
        return np.ascontiguousarray(DeviceArray.random(ctx, n, seed=seed, stream_id=4).to_limbs())

    for n_split, n_rec in ((1_000_003, 700_001), (5, 3), (0, 1000), (4099, 0), (300_000, 2_000_000)):
        sec = rand_limbs(n_split, 5)
        C = np.stack([rand_limbs(n_split, 6 + j) for j in range(t)]) if n_split else np.zeros((t, 0, L), np.uint64)
        rows = [rand_limbs(n_rec, 20 + i) for i in range(k)]
        sh_a, out_a = np.zeros((m, n_split, L), np.uint64), np.zeros((1, n_rec, L), np.uint64)
        sh_b, out_b = np.zeros((m, n_split, L), np.uint64), np.zeros((1, n_rec, L), np.uint64)
        rowp = _cabi.ptr_array([r.ctypes.data for r in rows])
        xs_c, xr_c = _cabi.i64_array(xs), _cabi.i64_array([0])
        ptr = lambda a: ctypes.c_void_p(a.ctypes.data)   # noqa: E731
        check(lib.mpyc_b200_shamir_split_host(ctx.handle, ptr(sec), ptr(C), n_split, ptr(sh_a), n_split, n_split, t, m, 0))
        check(lib.mpyc_b200_shamir_recombine_host(ctx.handle, rowp, xs_c, k, xr_c, 1, ptr(out_a), n_rec, n_rec, 0))
        check(lib.mpyc_b200_shamir_reshare_step_host(ctx.handle, ptr(sec), ptr(C), n_split, ptr(sh_b), n_split, n_split, t, m,
                                                     rowp, xs_c, k, xr_c, 1, ptr(out_b), n_rec, n_rec, 0))
        assert np.array_equal(sh_a, sh_b) and np.array_equal(out_a, out_b)
        if 0 < n_rec <= 1000:
            want = orc.recombine(Fo, xs, [[int(v) for v in codec.limbs_to_ints(r, ctx)] for r in rows], [0])[0]
            assert [int(v) for v in codec.limbs_to_ints(out_b[0], ctx)] == want
