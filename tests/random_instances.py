"""Seeded random instances for tests/test_oracle_golden.py, and the generator of the reference's results on them:

    MPYC_REFERENCE=<checkout of lschoe/mpyc> python tests/random_instances.py    # writes tests/golden/random_instances.json

The inputs are regenerated from these recipes (random.Random's integer streams are the same in every Python 3 version),
so the fixture holds only, per test and prime (order of PRIMES), one short SHA-256 digest per result kind (order of
KINDS) over the reference's results on all instances, with secrets.randbelow replaced by the instance's stream."""
import itertools
import json
import os
import random
import sys
from collections import defaultdict

PRIMES = [2**61 - 1, 2**64 - 189, 2**69 - 93, 2**128 - 173, 2**256 - 189, 9409569905028393239, 101, 2**89 - 1]
KINDS = {'split': ('shares_np', 'shares_list', 'recombination_vectors', 'recombined', 'f_S_i', 'prss', 'prss_zero_np',
                   'prss_zero_list'),
         'operators': ('add', 'sub', 'mul', 'neg', 'inv', 'div', 'lshift5', 'rshift5', 'pow7'),
         'local': ('square_add', 'mul_add', 'axpb', 'low_bits', 'nonzero', 'compose_ascending', 'compose_descending',
                   'decompose_descending', 'decompose_ascending')}


def split_instances(p):
    """Split / recombination / PRSS instances: secrets s, the coefficient stream that stands in for secrets.randbelow,
    the recombining parties xs, and one party i's PRF keys for PRSS."""
    rnd = random.Random(p % 10007)
    for m, t in ((1, 0), (3, 1), (4, 1), (5, 2), (7, 3), (6, 5)):
        n = rnd.randrange(1, 9)
        s = [rnd.randrange(p) for _ in range(n)]
        stream = [rnd.randrange(p) for _ in range(t * n)]
        xs = sorted(rnd.sample(range(1, m + 1), min(m, t + 1)))
        i = rnd.randrange(m)
        subsets = [S for S in itertools.combinations(range(m), m - t) if i in S]
        keys = {S: bytes(rnd.randrange(256) for _ in range(16)) for S in subsets}
        uci = bytes(rnd.randrange(256) for _ in range(5))
        yield dict(m=m, t=t, n=n, s=s, stream=stream, xs=xs, i=i, keys=keys, uci=uci)


def operator_instance(p):
    rnd = random.Random(p % 7919)
    a = [rnd.randrange(p) for _ in range(12)]
    b = [rnd.randrange(1, p) for _ in range(12)]
    return a, b


def local_instances(p):
    """Operands of the protocols' raw-value algebra: n elements, f bits per composed element, a public s, t, a bit
    count nb for the low bits and a length l for the bit decomposition."""
    rnd = random.Random(p % 9973)
    for _ in range(6):
        n, f = rnd.randrange(1, 7), rnd.randrange(1, 75)
        a, b, c = ([rnd.randrange(p) for _ in range(n)] for _ in range(3))
        s, t = rnd.randrange(p), rnd.randrange(p)
        nb = rnd.randrange(0, p.bit_length() + 3)
        bits = [rnd.randrange(p) for _ in range(n * f)]
        l = rnd.randrange(1, p.bit_length() + 1)   # noqa: E741
        yield dict(n=n, f=f, a=a, b=b, c=c, s=s, t=t, nb=nb, bits=bits, l=l)


class injected:
    def __init__(self, stream):
        self.it = iter(stream)

    def __enter__(self):
        self.orig = thresha.secrets.randbelow
        thresha.secrets.randbelow = lambda order: next(self.it)

    def __exit__(self, *exc):
        thresha.secrets.randbelow = self.orig


def split_cases(p):
    F = finfields.GF(p)
    out = defaultdict(list)
    for c in split_instances(p):
        m, t, n, s, xs, i = c['m'], c['t'], c['n'], c['s'], c['xs'], c['i']
        with injected(c['stream']):
            sh_np = thresha.np_random_split(F, F.array(np.array(s, dtype=object)), t, m)
        with injected(c['stream']):
            sh_li = thresha.random_split(F, [F(x) for x in s], t, m)
        prfs = {S: thresha.PRF(k, p) for S, k in c['keys'].items()}
        out['shares_np'].append(sh_np)
        out['shares_list'].append([[int(v) for v in row] for row in sh_li])
        out['recombination_vectors'].append([[int(v) % p for v in thresha._recombination_vector(F, tuple(xs), x_r)]
                                             for x_r in (0, m + 1)])
        out['recombined'].append(thresha.np_recombine(F, [(x, sh_np[x - 1]) for x in xs]).value)
        out['f_S_i'].append([int(thresha._f_S_i(F, m, i, S)) % p for S in c['keys']])
        out['prss'].append(thresha.np_pseudorandom_share(F, m, i, prfs, c['uci'], n).value)
        if t:
            out['prss_zero_np'].append(thresha.np_pseudorandom_share_0(F, m, i, prfs, c['uci'], n).value)
            out['prss_zero_list'].append([a.value for a in thresha.pseudorandom_share_zero(F, m, i, prfs, c['uci'], n)])
    return [digest(out[k]) for k in KINDS['split']]


def operator_case(p):
    F = finfields.GF(p)
    a, b = operator_instance(p)
    A, B = F.array(np.array(a, dtype=object)), F.array(np.array(b, dtype=object))
    results = {'add': (A + B).value, 'sub': (A - B).value, 'mul': (A * B).value, 'neg': (-A).value,
               'inv': B.reciprocal().value, 'div': (A / B).value, 'lshift5': (A << 5).value, 'rshift5': (A >> 5).value,
               'pow7': (A ** 7).value}
    return [digest(results[k]) for k in KINDS['operators']]


def local_cases(p):
    """The expressions of np_random_bits / np_trunc / np_sgn / np_to_bits (mpyc/runtime.py:860, 870, 3646-3660,
    4252-4271, 4415) on the reference's field arrays."""
    Zp = finfields.GF(p)
    arr = lambda v: Zp.array(np.array(v, dtype=object))   # noqa: E731
    out = defaultdict(list)
    for c in local_instances(p):
        n, f, ln = c['n'], c['f'], c['l']
        A, B, C, R = arr(c['a']), arr(c['b']), arr(c['c']), arr(c['bits'])
        for k, v in (('square_add', Zp.array(A.value**2 + C.value).value),
                     ('mul_add', Zp.array(A.value * B.value + C.value).value),
                     ('axpb', Zp.array(A.value * c['s'] + c['t']).value),
                     ('low_bits', C.value & ((1 << c['nb']) - 1)),
                     ('nonzero', A.value != 0),
                     ('compose_ascending', Zp.array(np.sum(R.value.reshape((n, f)) << np.arange(f), axis=1)).value),
                     ('compose_descending', Zp.array(np.sum(R.value.reshape((n, f)) << np.arange(f - 1, -1, -1), axis=1)).value),
                     ('decompose_descending', np.right_shift.outer(C.value, np.arange(ln - 1, -1, -1)).T & 1),
                     ('decompose_ascending', np.right_shift.outer(C.value, np.arange(ln)).T & 1)):
            out[k].append(v)
    return [digest(out[k]) for k in KINDS['local']]


def main():
    global thresha, finfields, np, digest   # used by the case functions above
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path[:0] = [os.path.dirname(here), here]
    sys.dont_write_bytecode = True
    from golden_util import digest
    from oracle import reference
    if reference.path() is None:
        raise SystemExit('set MPYC_REFERENCE to a checkout of the reference')
    sys.path.insert(0, reference.path())
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']   # mpyc parses sys.argv at import
    from mpyc import thresha, finfields
    import numpy as np
    sys.argv = argv
    obj = {'meta': {'reference': 'lschoe/mpyc v0.11.2 (unmodified, gmpy2 stubs=mpyc.gmpy)'},
           'split': [split_cases(p) for p in PRIMES],
           'operators': [operator_case(p) for p in PRIMES],
           'local': [local_cases(p) for p in PRIMES]}
    path = os.path.join(here, 'golden', 'random_instances.json')
    with open(path, 'w') as fh:
        json.dump(obj, fh, separators=(',', ':'))
    print('random_instances.json', os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
