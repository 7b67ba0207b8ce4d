"""Pin the CPU oracle (oracle/shamir_oracle.py) against fixtures produced by the real reference.

Every function of the oracle is replayed on the inputs stored in tests/golden/*.json and must
reproduce the reference's outputs bit for bit.  Runs on CPU (no GPU, no reference needed).
"""
from collections import defaultdict

import pytest

import random_instances as ri
from oracle import shamir_oracle as orc
from golden_util import digest, load, unhex

SPLIT = load('split_recombine.json')
PRF = load('prf.json')
PRSS = load('prss.json')
FF = load('finfields.json')
G256 = load('gf256.json')
RANDOM = load('random_instances.json')   # digests of the reference's results on tests/random_instances.py's instances


def test_default_primes_match_reference_find_prime_root():
    d = {k: int(v, 16) for k, v in SPLIT['meta']['default_primes'].items()}
    assert d == {'61': 2**61 - 1, '64': 2**64 - 189, '69': 2**69 - 93, '128': 2**128 - 173, '256': 2**256 - 189}


@pytest.mark.parametrize('case', SPLIT['cases'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_{c['p'][-4:]}_m{c['m']}t{c['t']}")
def test_split_and_recombine(case):
    p, m, t = int(case['p'], 16), case['m'], case['t']
    F = orc.field_of(p)
    s, stream = unhex(case['secrets']), unhex(case['stream'])
    n = len(s)
    sh_np = orc.split_np_order(F, s, orc.np_stream_to_C(stream, t, n), m)
    assert sh_np == unhex(case['shares_np'])
    sh_li = orc.split_list_order(F, s, orc.list_stream_to_c(stream, t, n), m)
    assert sh_li == unhex(case['shares_list'])
    for rec in case['recombine']:
        xs = rec['xs']
        rows = [sh_np[x - 1] for x in xs]
        assert orc.recombination_vector(F, xs, 0) == unhex(rec['lambda0'])
        assert orc.recombine(F, xs, rows) == unhex(rec['y0'])
        assert orc.recombine(F, xs, rows, rec['x_rs']) == unhex(rec['yw'])
    # recombining t+1 shares returns the secrets
    assert orc.recombine(F, list(range(1, t + 2)), sh_np[:t + 1]) == s


def test_survey_golden_vectors():
    """SURVEY.md 8c vectors (1)-(3), verified there against the reference."""
    p = 2**61 - 1
    F = orc.field_of(p)
    s, t, m = [5, 7, 11], 2, 5
    stream = list(range(100, 100 + t * len(s)))
    sh = orc.split_np_order(F, s, orc.np_stream_to_C(stream, t, 3), m)
    assert sh[0] == [208, 212, 218] and sh[4] == [3080, 3112, 3146]
    sl = orc.split_list_order(F, s, orc.list_stream_to_c(stream, t, 3), m)
    assert sl[0] == [206, 212, 220] and sl[4] == [3010, 3072, 3136]
    assert orc.recombination_vector(F, [1, 2, 3], 0) == [3, p - 3, 1]
    key = bytes.fromhex(PRF['key'])
    assert orc.prf_byte_length(key, p) == 24
    assert orc.prf_values(key, p, b'test uci', 3) == [1046088318803487675, 1073978524010014604, 482091145522698244]


@pytest.mark.parametrize('case', PRF['cases'], ids=lambda c: f"b{int(c['bound'],16).bit_length()}_n{c['n']}")
def test_prf(case):
    key = bytes.fromhex(PRF['key'])
    bound = int(case['bound'], 16)
    assert orc.prf_byte_length(key, bound) == case['l']
    assert orc.prf_values(key, bound, bytes.fromhex(case['s']), case['n']) == unhex(case['values'])


@pytest.mark.parametrize('case', PRSS['cases'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_m{c['m']}t{c['t']}")
def test_prss(case):
    p, m, t, n = int(case['p'], 16), case['m'], case['t'], case['n']
    F = orc.field_of(p)
    uci = bytes.fromhex(case['uci'])
    keys = {tuple(int(x) for x in k.split(',')): bytes.fromhex(v) for k, v in case['keys'].items()}
    zero_rows = []
    for party in case['parties']:
        i = party['i']
        mine = {S: k for S, k in keys.items() if i in S}
        for S in mine:
            assert orc.f_S_i(F, m, i, S) % p == int(party['f_S_i'][','.join(map(str, S))], 16) % p
        prl = {S: orc.prf_values(k, p, uci, n) for S, k in mine.items()}
        assert orc.prss_share(F, m, i, prl, n) == unhex(party['share_np']) == unhex(party['share_list'])
        d = t
        prl0 = {S: orc.prf_values(k, p, uci, n * d) for S, k in mine.items()}
        assert orc.prss_share_zero_list_order(F, m, i, prl0, n) == unhex(party['zero_list'])
        if t:
            assert orc.prss_share_zero_np_order(F, m, i, prl0, n) == unhex(party['zero_np'])
            zero_rows.append(unhex(party['zero_np']))
    if t:   # degree-2t sharing of zero: all m shares recombine to 0
        assert orc.recombine(F, list(range(1, m + 1)), zero_rows) == [0] * n


@pytest.mark.parametrize('case', FF['cases'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_{c['p'][-4:]}")
def test_finfields_ops(case):
    p = int(case['p'], 16)
    a, b, nz = unhex(case['a']), unhex(case['b']), unhex(case['nz'])
    assert orc.ff_add(p, a, b) == unhex(case['add'])
    assert orc.ff_sub(p, a, b) == unhex(case['sub'])
    assert orc.ff_mul(p, a, b) == unhex(case['mul'])
    assert orc.ff_neg(p, a) == unhex(case['neg'])
    assert orc.ff_inv(p, nz) == unhex(case['inv_nz'])
    assert orc.ff_div(p, a, nz) == unhex(case['div'])
    assert orc.ff_lshift(p, a, 7) == unhex(case['lshift7'])
    assert orc.ff_rshift(p, a, 7) == unhex(case['rshift7'])
    assert orc.ff_pow(p, a, 5) == unhex(case['pow5'])
    assert orc.ff_pow(p, nz, -3) == unhex(case['powm3_nz'])
    assert orc.ff_pow(p, a, (p - 1) // 2 + 3) == unhex(case['pow_big'])
    assert orc.ff_is_sqr(p, a) == case['is_sqr']
    assert orc.ff_signed(p, a) == [int(x) for x in case['signed']]
    assert orc.ff_mul(p, a, [12345678901234567890123] * len(a)) == unhex(case['mul_scalar'])
    assert orc.ff_add(p, a, [p - 5] * len(a)) == unhex(case['add_scalar'])
    if 'sqrt_a' in case:
        assert orc.ff_sqrt(p, a) == unhex(case['sqrt_a'])
        assert orc.ff_sqrt(p, orc.ff_mul(p, a, a)) == unhex(case['sqrt_of_sq'])
        assert orc.ff_sqrt(p, orc.ff_mul(p, nz, nz), INV=True) == unhex(case['invsqrt_of_nzsq'])
    A = [a[0:4], a[4:8], a[8:12]]
    B = [b[0:5], b[5:10], b[10:15], b[15:20]]
    assert orc.ff_matmul(p, A, B) == unhex(case['matmul_3x4_4x5'])
    with pytest.raises(ZeroDivisionError):
        orc.ff_inv(p, [1, 0])


def test_gf256_tables_and_known_answers():
    f = G256['modulus']
    tab = bytes.fromhex(G256['mul_table_hex'])
    for a in range(256):
        for b in range(0, 256, 1):
            assert orc.gf2x_mod(orc.gf2x_mul(a, b), f) == tab[a * 256 + b]
    assert [0] + orc.bf_inv(f, list(range(1, 256))) == G256['inv']
    # reference tests/test_finfields.py:94-99
    assert orc.bf_mul(f, [16, 57], [16, 67]) == [27, 137]
    assert orc.bf_mul(f, [137], [orc.gf2x_invert(57, f)]) == [67]


@pytest.mark.parametrize('case', G256['split'], ids=lambda c: f"m{c['m']}t{c['t']}")
def test_gf256_split_recombine(case):
    F = orc.field_of(G256['modulus'], binary=True)
    m, t = case['m'], case['t']
    s, stream = unhex(case['secrets']), unhex(case['stream'])
    n = len(s)
    sh = orc.split_np_order(F, s, orc.np_stream_to_C(stream, t, n), m)
    assert sh == unhex(case['shares_np'])
    assert orc.split_list_order(F, s, orc.list_stream_to_c(stream, t, n), m) == unhex(case['shares_list'])
    xs = case['xs']
    assert orc.recombination_vector(F, xs, 0) == unhex(case['lambda0'])
    assert orc.recombine(F, xs, [sh[x - 1] for x in xs]) == unhex(case['y0'])


def test_numpy_object_variants_agree_with_scalar_oracle():
    import numpy as np
    p = 2**128 - 173
    m, t, n = 5, 2, 40
    s = orc.edge_block(p) + orc.synth_elements(p, n - 8, 7)
    C = orc.np_stream_to_C(orc.synth_elements(p, t * n, 8), t, n)
    ref = orc.split_np_order(orc.field_of(p), s, C, m)
    got = orc.np_split(p, np.array(s, dtype=object), np.array(C, dtype=object), m)
    assert got.tolist() == ref
    rec = orc.np_recombine(p, (1, 2, 3), got[:3])
    assert rec.tolist() == s


BOUNDS = load('prss_bounds.json')


def _bound_id(c):
    return f"{c['field']}{int(c['modulus'], 16).bit_length()}_b{int(c['bound'], 16).bit_length()}_m{c['m']}t{c['t']}"


@pytest.mark.parametrize('case', BOUNDS['cases'], ids=_bound_id)
def test_prss_with_any_prf_bound(case):
    """PRF bounds other than the field order (thresha.py:257-261 reduces chunk % bound for any bound; callers
    runtime.py:735-739,758-760,4138,4218), prime fields and GF(2^8), reference-generated."""
    mod, bound, m, t, n = int(case['modulus'], 16), int(case['bound'], 16), case['m'], case['t'], case['n']
    F = orc.field_of(mod, binary=case['field'] == 'gf')
    uci = bytes.fromhex(case['uci'])
    keys = {tuple(int(x) for x in k.split(',')): bytes.fromhex(v) for k, v in case['keys'].items()}
    for party in case['parties']:
        i = party['i']
        mine = {S: k for S, k in keys.items() if i in S}
        prl = {S: orc.prf_values(k, bound, uci, n) for S, k in mine.items()}
        assert orc.prss_share(F, m, i, prl, n) == unhex(party['share_np']) == unhex(party['share_list'])
        prl0 = {S: orc.prf_values(k, bound, uci, n * t) for S, k in mine.items()}
        assert orc.prss_share_zero_list_order(F, m, i, prl0, n) == unhex(party['zero_list'])
        if t:
            assert orc.prss_share_zero_np_order(F, m, i, prl0, n) == unhex(party['zero_np'])


# ---- protocol-local algebra (SURVEY 8f N3 / N4): oracle vs the reference's own expressions -----------------------

LOCAL = load('local.json')


@pytest.mark.parametrize('case', LOCAL['algebra'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_{c['p'][-4:]}")
def test_local_algebra(case):
    p = int(case['p'], 16)
    a, b, c = unhex(case['a']), unhex(case['b']), unhex(case['c'])
    assert orc.local_fma(p, a, a, c) == unhex(case['square_add'])
    assert orc.local_fma(p, a, b, c) == unhex(case['mul_add'])
    assert orc.local_nonzero(a) == case['nonzero']
    for f in (0, 6):
        s = ((p + 1) >> 1 << f) % p
        assert orc.local_axpb(p, a, s, s) == unhex(case[f'bits_tail_f{f}'])
    assert orc.local_axpb(p, a, 2, -1) == unhex(case['s_sign'])
    for key in case:
        if key.startswith('low_bits_'):
            assert orc.local_low_bits(c, int(key[9:])) == unhex(case[key])
    for comp in case['compose']:
        bits = unhex(comp['bits'])
        assert orc.local_bits_compose(p, bits, comp['n'], comp['f']) == unhex(comp['ascending'])
        assert orc.local_bits_compose(p, bits, comp['n'], comp['f'], descending=True) == unhex(comp['descending'])
    for dec in case['decompose']:
        assert orc.local_bits_decompose(c, dec['l']) == unhex(dec['ascending'])
        assert orc.local_bits_decompose(c, dec['l'], descending=True) == unhex(dec['descending'])


@pytest.mark.parametrize('case', LOCAL['conv'], ids=lambda c: f"p{int(c['p'],16).bit_length()}_{'x'.join(map(str, c['shape']))}")
def test_local_conv2d(case):
    p = int(case['p'], 16)
    k, r, m, n, v, s = case['shape']
    assert orc.local_conv2d(p, unhex(case['X']), unhex(case['W']), unhex(case['B']), k, r, m, n, v, s) == unhex(case['Y'])


def _check_random(test, p, results):
    want = dict(zip(ri.KINDS[test], RANDOM[test][ri.PRIMES.index(p)]))
    assert {k: digest(results[k]) for k in want} == want


@pytest.mark.parametrize('p', ri.PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_split_recombine_prss_random_instances(p):
    Fo = orc.field_of(p)
    got = defaultdict(list)
    for c in ri.split_instances(p):
        m, t, n, s, stream, xs, i, keys, uci = (c[k] for k in ('m', 't', 'n', 's', 'stream', 'xs', 'i', 'keys', 'uci'))
        sh_np = orc.split_np_order(Fo, s, orc.np_stream_to_C(stream, t, n), m)
        rec = orc.recombine(Fo, xs, [sh_np[x - 1] for x in xs])
        assert rec == s
        got['shares_np'].append(sh_np)
        got['shares_list'].append(orc.split_list_order(Fo, s, orc.list_stream_to_c(stream, t, n), m))
        got['recombination_vectors'].append([orc.recombination_vector(Fo, xs, x_r) for x_r in (0, m + 1)])
        got['recombined'].append(rec)
        got['f_S_i'].append([orc.f_S_i(Fo, m, i, S) % p for S in keys])
        got['prss'].append(orc.prss_share(Fo, m, i, {S: orc.prf_values(k, p, uci, n) for S, k in keys.items()}, n))
        if t:
            prl = {S: orc.prf_values(k, p, uci, n * t) for S, k in keys.items()}
            got['prss_zero_np'].append(orc.prss_share_zero_np_order(Fo, m, i, prl, n))
            got['prss_zero_list'].append(orc.prss_share_zero_list_order(Fo, m, i, prl, n))
    _check_random('split', p, got)


@pytest.mark.parametrize('p', ri.PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_field_array_operators_random_instances(p):
    a, b = ri.operator_instance(p)
    got = {'add': orc.ff_add(p, a, b), 'sub': orc.ff_sub(p, a, b), 'mul': orc.ff_mul(p, a, b), 'neg': orc.ff_neg(p, a),
           'inv': orc.ff_inv(p, b), 'div': orc.ff_div(p, a, b), 'lshift5': orc.ff_lshift(p, a, 5),
           'rshift5': orc.ff_rshift(p, a, 5), 'pow7': orc.ff_pow(p, a, 7)}
    _check_random('operators', p, got)


@pytest.mark.parametrize('p', ri.PRIMES, ids=lambda p: f'p{p.bit_length()}')
def test_local_algebra_random_instances(p):
    """oracle.local_* against the expressions of np_random_bits / np_trunc / np_sgn / np_to_bits (mpyc/runtime.py:860,
    870, 3646-3660, 4252-4271, 4415) evaluated on the reference's field arrays, random sizes and bit counts."""
    got = defaultdict(list)
    for c in ri.local_instances(p):
        n, f, a, b, cc, bits, ln = (c[k] for k in ('n', 'f', 'a', 'b', 'c', 'bits', 'l'))
        got['square_add'].append(orc.local_fma(p, a, a, cc))
        got['mul_add'].append(orc.local_fma(p, a, b, cc))
        got['axpb'].append(orc.local_axpb(p, a, c['s'], c['t']))
        got['low_bits'].append(orc.local_low_bits(cc, c['nb']))
        got['nonzero'].append(orc.local_nonzero(a))
        got['compose_ascending'].append(orc.local_bits_compose(p, bits, n, f))
        got['compose_descending'].append(orc.local_bits_compose(p, bits, n, f, descending=True))
        got['decompose_descending'].append(orc.local_bits_decompose(cc, ln, descending=True))
        got['decompose_ascending'].append(orc.local_bits_decompose(cc, ln))
    _check_random('local', p, got)
